"""Host twins of the diverse-list kernels (csrc/diverse.cu) against brute forces written from the contract, and the
input checks of recommend_diverse, without a GPU.

* item_union_host / cocount_host: co-rating counts as Python set intersections of the columns, with empty columns, a
  user who rated every union item and a union of one;
* item_cosine_host: bit for bit c / math.sqrt(d_a * d_b) rounded to fp32;
* diverse_select_host: the greedy selection as a literal loop over sorted keys, with ties, +-0, NaN, -inf, padding
  and short pools; penalty 0 gives the pool's prefix;
* every input check: k > pool, pool > 256, a pool that does not fit the merge, penalty negative, infinite or NaN."""
import math

import numpy as np
import pytest

from igmc_b200 import recommend as rc
from tests import support


def _graph(rows, num_items):
    rp, ci = support.rows_csr([sorted(r) for r in rows])
    cols = [set() for _ in range(num_items)]
    for u, r in enumerate(rows):
        for v in r:
            cols[v].add(u)
    cp = np.concatenate([[0], np.cumsum([len(c) for c in cols])]).astype(np.int32)
    return rp, ci, cp, cols


def _random_rows(seed, nu=40, ni=30, empty=(3, 17)):
    rng = np.random.default_rng(seed)
    rows = []
    for u in range(nu):
        n = int(rng.integers(0, 12))
        r = set(int(v) for v in rng.choice(ni, n, replace=False)) - set(empty)
        rows.append(sorted(r))
    rows[5] = [v for v in range(ni) if v not in empty]            # a user who rated every item that has raters
    rows[6] = []
    return rows


def _sim(cols, a, b):
    """the contract: |col(a) & col(b)| / sqrt(d_a d_b), rounded once to fp32, 0 without raters"""
    da, db = len(cols[a]), len(cols[b])
    if da * db == 0:
        return np.float32(0.0)
    return np.float32(len(cols[a] & cols[b]) / math.sqrt(da * db))


# ---- union and co-counts ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_union_and_cocounts_match_set_intersections(seed):
    ni = 30
    rows = _random_rows(seed, ni=ni)
    rp, ci, cp, cols = _graph(rows, ni)
    rng = np.random.default_rng(seed + 10)
    pools = rng.integers(-1, ni, (4, 9))
    pools[0, :3] = [3, 17, 3]                                      # empty columns, repeated
    mp, lst, bad = rc.item_union_host(pools, ni)
    want = sorted(set(int(v) for v in pools.reshape(-1) if v >= 0))
    assert not bad and lst.tolist() == want
    assert [int(mp[v]) for v in range(ni)] == [want.index(v) if v in want else -1 for v in range(ni)]
    table = rc.cocount_host(rp, ci, len(rows), ni, lst)
    nu = len(lst)
    assert table.dtype == np.uint32 and len(table) == nu * (nu - 1) // 2
    t = 0
    for i in range(nu):
        for j in range(i + 1, nu):
            assert table[t] == len(cols[lst[i]] & cols[lst[j]]), (i, j)
            assert rc._tri_at(i, j, nu) == t
            t += 1


def test_union_of_one_and_bad_ids():
    rows = _random_rows(4)
    rp, ci, cp, cols = _graph(rows, 30)
    mp, lst, bad = rc.item_union_host([[-1, 7, 7, -1]], 30)
    assert lst.tolist() == [7] and mp[7] == 0 and (np.delete(mp, 7) == -1).all() and not bad
    assert len(rc.cocount_host(rp, ci, len(rows), 30, lst)) == 0
    mp, lst, bad = rc.item_union_host([[2, 30, -2, 5]], 30)
    assert bad and lst.tolist() == [2, 5]


# ---- cosine -----------------------------------------------------------------------------------------------------------
def test_cosine_bit_for_bit():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        da, db = (int(x) for x in rng.integers(0, 5000, 2))
        c = int(rng.integers(0, min(da, db) + 1))
        got = rc.item_cosine_host(c, da, db)
        want = np.float32(0.0) if da * db == 0 else np.float32(c / math.sqrt(da * db))
        assert got.dtype == np.float32 and got.view(np.uint32) == want.view(np.uint32)
        if da * db:     # the same value through numpy's fp64
            alt = np.float32(np.float64(c) / np.sqrt(np.float64(da) * np.float64(db)))
            assert got.view(np.uint32) == alt.view(np.uint32)
    for d in (1, 2, 3, 7, 1000, 4095, 65537):
        assert rc.item_cosine_host(d, d, d) == np.float32(1.0)
    assert rc.item_cosine_host(0, 0, 5) == 0 and rc.item_cosine_host(0, 5, 0) == 0


def test_item_similarity_host_matches_contract():
    rows = _random_rows(7)
    rp, ci, cp, cols = _graph(rows, 30)
    items = [3, 0, 9, 9, 17, 29, 1]
    got = rc.item_similarity_host(rp, ci, cp, len(rows), 30, items)
    want = np.array([[_sim(cols, a, b) for b in items] for a in items], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ---- greedy selection -------------------------------------------------------------------------------------------------
def _brute_select(cols, pool_i, pool_s, k, penalty):
    """the contract as a literal loop: per step the keys of the unchosen real entries, sorted by (NaN last, key
    descending, pool position)"""
    pen = np.float32(penalty)
    Q, P = np.shape(pool_i)
    out_i = np.full((Q, k), -1, np.int64)
    out_s = np.full((Q, k), -np.inf, np.float32)
    out_k = np.full((Q, k), -np.inf, np.float32)
    for q in range(Q):
        chosen = []
        for s in range(k):
            keys = []
            for j in range(P):
                v = int(pool_i[q][j])
                if v < 0 or j in chosen:
                    continue
                m = max([_sim(cols, v, int(pool_i[q][c])) for c in chosen], default=np.float32(0.0))
                key = np.float32(np.float32(pool_s[q][j]) - np.float32(pen * np.float32(m)))
                keys.append((bool(np.isnan(key)), 0.0 if np.isnan(key) else -float(key), j, key))
            if not keys:
                break
            keys.sort(key=lambda t: t[:3])
            j, key = keys[0][2], keys[0][3]
            chosen.append(j)
            out_i[q, s], out_s[q, s], out_k[q, s] = pool_i[q][j], pool_s[q][j], key
    return out_i, out_s, out_k


def _select(rows, ni, pool_i, pool_s, k, penalty):
    rp, ci, cp, cols = _graph(rows, ni)
    mp, lst, bad = rc.item_union_host(pool_i, ni)
    table = rc.cocount_host(rp, ci, len(rows), ni, lst)
    got = rc.diverse_select_host(cp, pool_i, pool_s, k, penalty, mp, table, len(lst))
    return got, _brute_select(cols, pool_i, pool_s, k, penalty)


@pytest.mark.parametrize("penalty", [0.0, 0.25, 1.0, 3.0, 1e6])
def test_selection_matches_literal_loop(penalty):
    ni = 30
    rows = _random_rows(11, ni=ni)
    rng = np.random.default_rng(int(penalty * 7) + 1)
    Q, P, k = 6, 12, 7
    pool_i = np.full((Q, P), -1, np.int64)
    pool_s = np.full((Q, P), -np.inf, np.float32)
    for q in range(Q):
        n = [P, P, 9, 4, 1, 0][q]                                   # short pools and an empty one: padding past them
        pool_i[q, :n] = rng.choice(ni, n, replace=False)
        pool_s[q, :n] = np.round(rng.uniform(1, 5, n) * 4) / 4      # many ties
    pool_s[0, 2:5] = [0.0, -0.0, 0.0]                               # +-0 compare equal: ties by position
    pool_s[1, 3], pool_s[1, 7] = np.nan, np.nan                     # NaN after every number
    pool_s[1, 0], pool_s[2, 1] = -np.inf, np.inf
    pool_i[0, 5], pool_i[0, 6] = 3, 17                              # items without raters: sim 0
    (gi, gs, gk, bad), (wi, ws, wk) = _select(rows, ni, pool_i, pool_s, k, penalty)
    assert not bad.any()
    assert np.array_equal(gi, wi) and support.same(gs, ws) and support.same(gk, wk)
    assert (gi[3, 4:] == -1).all() and (gs[4, 1:] == -np.inf).all() and (gk[5] == -np.inf).all()


def test_selection_flags_bad_pools_as_padding():
    rows = _random_rows(3)
    rp, ci, cp, cols = _graph(rows, 30)
    pool_i = np.array([[4, 5, 6], [4, 31, 6], [4, -3, 6], [8, 9, -1]], np.int64)
    pool_s = np.ones((4, 3), np.float32)
    mp, lst, bad = rc.item_union_host(pool_i, 30)
    assert bad
    table = rc.cocount_host(rp, ci, len(rows), 30, lst)
    gi, gs, gk, bad = rc.diverse_select_host(cp, pool_i, pool_s, 2, 1.0, mp, table, len(lst))
    assert bad.tolist() == [False, True, True, False]
    assert (gi[1:3] == -1).all() and (gs[1:3] == -np.inf).all() and (gk[1:3] == -np.inf).all()
    mp[9] = -1                                                      # an item the union does not hold
    gi, _, _, bad = rc.diverse_select_host(cp, pool_i, pool_s, 2, 1.0, mp, table, len(lst))
    assert bad.tolist() == [False, True, True, True] and (gi[3] == -1).all()


def test_penalty_zero_is_the_pool_prefix():
    ni = 30
    rows = _random_rows(5, ni=ni)
    rng = np.random.default_rng(2)
    scores = np.round(rng.uniform(1, 5, (5, ni)) * 2) / 2
    scores[0, :4] = [np.nan, -0.0, 0.0, -np.inf]
    pools = [rc.rank_host(scores[q], np.arange(ni), 20) for q in range(5)]
    pool_s = np.stack([p[0] for p in pools])
    pool_i = np.stack([p[1] for p in pools])
    pool_i[4, 12:], pool_s[4, 12:] = -1, -np.inf                    # a short pool
    for k in (1, 8, 20):
        (gi, gs, gk, _), _ = _select(rows, ni, pool_i, pool_s, k, 0.0)
        assert np.array_equal(gi, pool_i[:, :k]) and support.same(gs, pool_s[:, :k]) and support.same(gk, gs)


def test_recommend_diverse_host_composes_the_twins():
    ni = 30
    rows = _random_rows(9, ni=ni)
    rp, ci, cp, cols = _graph(rows, ni)
    rng = np.random.default_rng(3)
    table = rng.uniform(1, 5, (len(rows), ni)).astype(np.float32)

    def pooler(users, pool):
        out = [rc.rank_host(table[u][np.setdiff1d(np.arange(ni), rows[u])], np.setdiff1d(np.arange(ni), rows[u]), pool)
               for u in users]
        return np.stack([o[1] for o in out]), np.stack([o[0] for o in out])

    users = [0, 5, 6, 11]
    gi, gs, gk = rc.recommend_diverse_host(rp, ci, cp, len(rows), ni, users, 5, 0.5, pooler, pool=15)
    pi, ps = pooler(users, 15)
    wi, ws, wk = _brute_select(cols, pi, ps, 5, 0.5)
    assert np.array_equal(gi, wi) and support.same(gs, ws) and support.same(gk, wk)
    assert sorted(gi[1, :2].tolist()) == [3, 17] and (gi[1, 2:] == -1).all()   # user 5: only the unrated items
    hi, hs, _ = rc.recommend_diverse_host(rp, ci, cp, len(rows), ni, users, 5, 0.0, pooler, pool=15)
    assert np.array_equal(hi, pi[:, :5]) and support.same(hs, ps[:, :5])


# ---- input checks -----------------------------------------------------------------------------------------------------
def test_input_checks():
    ok = dict(k=5, penalty=0.5, pool=50, batch_size=256)
    assert rc._diverse_inputs(**ok) == (5, 50, 0.5)
    assert rc._diverse_inputs(5, -0.0, 50, 256)[2] == 0.0 and math.copysign(1, rc._diverse_inputs(5, -0.0, 50, 256)[2]) > 0
    for bad, err in ((dict(k=51), ValueError), (dict(k=0), ValueError), (dict(pool=0), ValueError),
                     (dict(pool=257, k=5), NotImplementedError), (dict(penalty=-0.1), ValueError),
                     (dict(penalty=float("inf")), ValueError), (dict(penalty=float("nan")), ValueError),
                     (dict(penalty=1e39), ValueError), (dict(pool=256, batch_size=19200), ValueError)):
        args = dict(ok, **bad)
        with pytest.raises(err):
            rc._diverse_inputs(**args)
        with pytest.raises(err):    # the public function checks before it touches the model or the graph
            rc.recommend_diverse(None, None, [0], args["k"], args["penalty"], pool=args["pool"],
                                 batch_size=args["batch_size"])
