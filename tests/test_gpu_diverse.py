"""Diversified lists and item similarity on the GPU (recommend_diverse, item_similarity,
InferenceEngine.start_recommend_diverse; csrc/diverse.cu).

* igmc_item_union, igmc_cocount, igmc_diverse_select and igmc_item_cosine byte for byte against their host twins
  (tests/test_diverse_host.py), with sentinel-filled outputs and guard entries past them, a rating row longer than the
  count kernel's shared-memory tile, and bad ids setting the error word;
* item_similarity against the twin on ml_1m* and the flixster split;
* every diversified list bit for bit (items, scores, keys) recommend_diverse_host over ``recommend`` pools from the
  same engine, on plans 2 / 4 / 0 (R = 13) / L2, rgcn="pyg-2", DGCNN_RS and three checkpoints, with items lists,
  per-user rows, retrieve= and exclude_rated=False;
* penalty 0 is recommend(k); a tiny workspace bound (users in chunks) gives the same lists; a user's list does not
  depend on the other users; two runs are bit-identical; the diverse stage makes at most one host sync per chunk; a
  graph.update between runs is served and one during a run raises."""
import ctypes as C
import tempfile
import warnings

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.util_functions import RatingGraph, _stream_ptr
from tests import support

pytestmark = pytest.mark.gpu

SENT32, SENTF = -77, -7.5
GUARD = 16


def _users(g, n, seed):
    rng = np.random.default_rng(seed)
    deg = np.diff(g.host["row_ptr"])[:g.num_users]
    return np.sort(rng.choice(np.flatnonzero(deg >= 3), n, replace=False)).astype(np.int64)


# ---- 1. the kernels against their twins --------------------------------------------------------------------------------
def _toy_graph(long_row=2500, ni=3000, nu=300, seed=0):
    """a graph whose user 7 rated ``long_row`` items (beyond the count kernel's tile of 1 024 row entries), with
    unrated items and an empty user"""
    rng = np.random.default_rng(seed)
    rows = [np.sort(rng.choice(ni - 10, int(rng.integers(0, 60)), replace=False)) for _ in range(nu)]
    rows[7] = np.sort(rng.choice(ni - 10, long_row, replace=False))
    rows[8] = np.zeros(0, np.int64)
    u = np.concatenate([np.full(len(r), j) for j, r in enumerate(rows)])
    v = np.concatenate(rows)
    A = ssp.csr_matrix((np.ones(len(u)), (u, v)), shape=(nu, ni))
    return RatingGraph(A)


def _union(items, ni):
    items = support.dev(items, torch.int64)
    bitmap = torch.full(((ni + 31) // 32,), SENT32, dtype=torch.int32, device="cuda")
    mp = torch.full((ni + GUARD,), SENT32, dtype=torch.int32, device="cuda")
    lst = torch.full((ni + GUARD,), SENT32, dtype=torch.int32, device="cuda")
    nu = torch.full((1 + GUARD,), SENT32, dtype=torch.int32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    code = _lib.load().igmc_item_union(items.data_ptr(), items.numel(), ni, bitmap.data_ptr(), mp.data_ptr(),
                                       lst.data_ptr(), nu.data_ptr(), err.data_ptr(), _stream_ptr())
    torch.cuda.synchronize()
    return code, int(err.item()), mp, lst, nu


def _cocount(g, mp, Nu, cap=None):
    need = Nu * (Nu - 1) // 2
    table = torch.full((max(need, 1) + GUARD,), SENT32, dtype=torch.int32, device="cuda")
    code = _lib.load().igmc_cocount(C.byref(g._c), mp.data_ptr(), Nu, table.data_ptr(),
                                    need if cap is None else cap, _stream_ptr())
    torch.cuda.synchronize()
    return code, table


@pytest.mark.parametrize("n_pool", [1, 40, 2000])
def test_union_and_cocount_kernels_match_twins(n_pool):
    g = _toy_graph()
    ni, hp = g.num_items, g.host
    rng = np.random.default_rng(n_pool)
    items = rng.integers(-1, ni, n_pool) if n_pool > 1 else np.array([5])
    items[:min(3, n_pool)] = items[0]                                            # repeats
    code, err, mp, lst, nu = _union(items, ni)
    assert code == 0 and err == 0
    want_mp, want_lst, _ = rc.item_union_host(items, ni)
    Nu = len(want_lst)
    assert int(nu[0]) == Nu and (nu[1:].cpu().numpy() == SENT32).all()
    got_mp, got_lst = mp.cpu().numpy(), lst.cpu().numpy()
    assert np.array_equal(got_mp[:ni], want_mp) and (got_mp[ni:] == SENT32).all()
    assert np.array_equal(got_lst[:Nu], want_lst) and (got_lst[Nu:] == SENT32).all()
    code, table = _cocount(g, mp, Nu)
    assert code == 0
    want = rc.cocount_host(hp["row_ptr"], hp["col_idx"], g.num_users, ni, want_lst)
    got = table.cpu().numpy().view(np.uint32)
    need = len(want)
    assert np.array_equal(got[:need], want) and (got[max(need, 1):].view(np.int32) == SENT32).all()
    if n_pool == 2000:
        r7 = hp["col_idx"][hp["row_ptr"][7]:hp["row_ptr"][8]]
        assert np.isin(r7, want_lst).sum() > 1024                                # the long row spans several tiles
        assert _lib.load().igmc_cocount(C.byref(g._c), mp.data_ptr(), Nu, table.data_ptr(), need - 1, None) == -2


def test_union_kernel_flags_bad_ids():
    ni = 3000
    items = np.array([4, -1, 3000, 9, -2, 4], np.int64)
    code, err, mp, lst, nu = _union(items, ni)
    assert code == 0 and err == 7                                                 # IGMC_ERR_CANDIDATES
    assert int(nu[0]) == 2 and lst[:2].cpu().tolist() == [4, 9]


def _select(g, pool_i, pool_s, k, penalty, mp, Nu, table):
    Q, P = pool_i.shape
    oi = torch.full((Q * k + GUARD,), SENT32, dtype=torch.int64, device="cuda")
    os_ = torch.full((Q * k + GUARD,), SENTF, dtype=torch.float32, device="cuda")
    ok = torch.full((Q * k + GUARD,), SENTF, dtype=torch.float32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    di, ds = support.dev(pool_i, torch.int64), support.dev(pool_s, torch.float32)
    code = _lib.load().igmc_diverse_select(C.byref(g._c), di.data_ptr(), ds.data_ptr(), Q, P, k, penalty,
                                           mp.data_ptr(), Nu, table.data_ptr(), oi.data_ptr(), os_.data_ptr(),
                                           ok.data_ptr(), err.data_ptr(), _stream_ptr())
    torch.cuda.synchronize()
    return code, int(err.item()), oi.cpu().numpy(), os_.cpu().numpy(), ok.cpu().numpy()


@pytest.mark.parametrize("P,k,penalty", [(12, 7, 0.0), (12, 12, 0.75), (256, 40, 2.0), (33, 1, 1e6)])
def test_select_kernel_matches_twin(P, k, penalty):
    g = _toy_graph(seed=1)
    ni, hp = g.num_items, g.host
    rng = np.random.default_rng(P + k)
    Q = 7
    pool_i = np.full((Q, P), -1, np.int64)
    pool_s = np.full((Q, P), -np.inf, np.float32)
    cols = np.flatnonzero(np.diff(hp["col_ptr"]) >= 2)
    for q in range(Q):
        n = [P, P, P // 2, 3, 1, 0, P][q]
        pool_i[q, :n] = rng.choice(cols if q < 6 else ni, n, replace=False)
        pool_s[q, :n] = np.round(rng.uniform(1, 5, n) * 4) / 4                    # ties
    pool_s[0, :3] = [0.0, -0.0, 0.0]
    pool_s[1, 2], pool_s[1, 5], pool_s[2, 0] = np.nan, -np.inf, np.inf
    pool_i[6, :2] = [ni - 1, ni - 2]                                              # items without raters
    mp, lst, _ = rc.item_union_host(pool_i, ni)
    Nu = len(lst)
    table = rc.cocount_host(hp["row_ptr"], hp["col_idx"], g.num_users, ni, lst)
    want = rc.diverse_select_host(hp["col_ptr"], pool_i, pool_s, k, penalty, mp, table, Nu)
    dt = support.dev(table.view(np.int32)) if Nu > 1 else torch.zeros(1, dtype=torch.int32, device="cuda")
    code, err, gi, gs, gk = _select(g, pool_i, pool_s, k, penalty, support.dev(mp), Nu, dt)
    assert code == 0 and err == 0
    n = Q * k
    assert np.array_equal(gi[:n], want[0].reshape(-1)) and (gi[n:] == SENT32).all()
    assert support.same(gs[:n], want[1].reshape(-1)) and (gs[n:] == SENTF).all()
    assert support.same(gk[:n], want[2].reshape(-1)) and (gk[n:] == SENTF).all()


def test_select_kernel_flags_bad_pools():
    g = _toy_graph(seed=2)
    ni, hp = g.num_items, g.host
    pool_i = np.array([[4, 5, 6], [4, ni, 6], [4, -3, 6], [8, 9, -1]], np.int64)
    pool_s = np.ones((4, 3), np.float32)
    mp, lst, _ = rc.item_union_host(pool_i, ni)
    mp[9] = -1                                                                    # an item the map does not hold
    table = rc.cocount_host(hp["row_ptr"], hp["col_idx"], g.num_users, ni, lst)
    want = rc.diverse_select_host(hp["col_ptr"], pool_i, pool_s, 2, 1.0, mp, table, len(lst))
    assert want[3].tolist() == [False, True, True, True]
    code, err, gi, gs, gk = _select(g, pool_i, pool_s, 2, 1.0, support.dev(mp), len(lst),
                                    support.dev(table.view(np.int32)))
    assert code == 0 and err == 7
    assert np.array_equal(gi[:8], want[0].reshape(-1)) and support.same(gs[:8], want[1].reshape(-1))
    assert support.same(gk[:8], want[2].reshape(-1))
    lib, p = _lib.load(), support.dev(mp).data_ptr()
    for P, k, pen in ((3, 4, 1.0), (257, 2, 1.0), (3, 2, -1.0), (3, 2, float("inf")), (3, 2, float("nan"))):
        assert lib.igmc_diverse_select(C.byref(g._c), p, p, 1, P, k, pen, p, 3, p, p, p, p, None, None) == -1


def test_item_similarity_kernel_and_public_matches_twin_toy():
    g = _toy_graph(seed=3)
    hp = g.host
    items = np.array([7, 7, 2999, 0, 15, 2, 7, 100, 2999], np.int64)
    got = rc.item_similarity(g, items).cpu().numpy()
    want = rc.item_similarity_host(hp["row_ptr"], hp["col_idx"], hp["col_ptr"], g.num_users, g.num_items, items)
    assert support.same(got, want)
    with pytest.raises(IndexError):
        rc.item_similarity(g, [1, g.num_items])
    assert rc.item_similarity(g, []).shape == (0, 0)


@pytest.mark.parametrize("name", ["ml_1m", "flixster"])
def test_item_similarity_matches_twin(name):
    g = RatingGraph(support.adj(name))
    hp = g.host
    rng = np.random.default_rng(0)
    items = rng.choice(g.num_items, 400)                                         # repeats included
    items[:5] = np.argsort(-np.diff(hp["col_ptr"]))[:5]                          # the most rated items
    got = rc.item_similarity(g, items).cpu().numpy()
    want = rc.item_similarity_host(hp["row_ptr"], hp["col_idx"], hp["col_ptr"], g.num_users, g.num_items, items)
    assert support.same(got, want)
    d = np.diff(hp["col_ptr"])[items]
    assert (np.diag(got)[d > 0] == 1).all() and (np.diag(got)[d == 0] == 0).all()


# ---- 2. the lists are the host composition over recommend pools --------------------------------------------------------
CASES = {
    # name: (dataset, mnph, model kwargs, forced kernel plan, checkpoints)
    "plan 2 ml_1m": ("ml_1m", 100, {}, 2, 0),
    "plan 4 ml_100k": ("ml_100k", 200, {}, 4, 0),
    "plan 0 R=13": ("r13", 50, {}, "auto", 0),
    "L2 plan ml_100k uncapped": ("ml_100k", None, {}, "auto", 0),
    "pyg-2": ("ml_1m", 100, dict(rgcn="pyg-2"), "auto", 0),
    "DGCNN_RS": ("ml_1m", 100, dict(dgcnn=True), "auto", 0),
    "K=3 checkpoints": ("ml_1m", 100, {}, "auto", 3),
}


def _check_lists(eng, g, users, k, penalty, pool, **kw):
    got = eng.recommend_diverse(users, k, penalty, pool, **kw)
    hp = g.host

    def pooler(us, p):
        ti, ts = eng.recommend(us, p, **kw)
        return ti.cpu().numpy(), ts.cpu().numpy()
    want = rc.recommend_diverse_host(hp["row_ptr"], hp["col_idx"], hp["col_ptr"], g.num_users, g.num_items, users, k,
                                     penalty, pooler, pool)
    assert np.array_equal(got.items.cpu().numpy(), want[0]), (k, penalty, pool, kw.keys())
    assert support.same(got.scores.cpu().numpy(), want[1]) and support.same(got.keys.cpu().numpy(), want[2])
    return got


@pytest.mark.parametrize("name", list(CASES))
def test_lists_equal_host_composition(name):
    dsn, mnph, kw, plan, K = CASES[name]
    g = RatingGraph(support.adj(dsn))
    m = support.model(13 if dsn == "r13" else 5, **kw)
    m.kernel_plan = plan
    try:
        with tempfile.TemporaryDirectory() as d:
            ck = support.checkpoints(m, K, d) if K else None
            eng = rc.InferenceEngine(m, g, max_nodes_per_hop=mnph, batch_size=64, checkpoints=ck, sample_seed=3)
            try:
                ni = g.num_items
                users = _users(g, 8, len(name))
                rng = np.random.default_rng(1)
                shared = rng.choice(ni, 120, replace=False)
                rows = np.full((len(users), 70), -1, np.int64)
                for j in range(len(users)):
                    rows[j, :60] = rng.choice(ni, 60)                             # duplicates and -1 slots
                runs = [dict(), dict(items=shared), dict(items=rows), dict(items=shared, exclude_rated=False),
                        dict(retrieve=80), dict(exclude_rated=False)]
                for j, extra in enumerate(runs):
                    pen = (0.5, 2.0, 0.25, 1.0, 4.0, 0.75)[j]
                    _check_lists(eng, g, users, 10, pen, 50 if j % 2 == 0 else 30, **extra)
            finally:
                eng.close()
    finally:
        m.kernel_plan = "auto"


# ---- 3. penalty 0, chunks, independence, syncs and updates ---------------------------------------------------------------
def test_penalty_zero_is_recommend_and_chunks_change_nothing():
    g = RatingGraph(support.adj("ml_1m"))
    m = support.model(5)
    users = _users(g, 24, 5)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=256)
    try:
        ti, ts = eng.recommend(users, 10)
        got = eng.recommend_diverse(users, 10, 0.0, pool=60)
        assert torch.equal(got.items, ti) and support.same(got.scores.cpu().numpy(), ts.cpu().numpy())
        assert support.same(got.keys.cpu().numpy(), got.scores.cpu().numpy())
        pub = rc.recommend_diverse(m, g, users, 10, 0.0, pool=60, max_nodes_per_hop=100)
        assert torch.equal(pub.items, ti)
        base = eng.recommend_diverse(users, 10, 1.5, pool=60)
        assert not torch.equal(base.items, ti)                                    # the penalty moves items
        eng.diverse_ws_bytes = 4 * (130 * 129 // 2)                               # two users' pools at most
        nbytes, chunk = C.c_int64(0), C.c_int(0)
        assert eng.lib.igmc_diverse_ws_bytes(len(users), 60, g.num_items, eng.diverse_ws_bytes, C.byref(nbytes),
                                             C.byref(chunk)) == 0
        assert chunk.value == 2
        small = eng.recommend_diverse(users, 10, 1.5, pool=60)
        for a, b in zip(small, base):
            assert support.same(a.cpu().numpy(), b.cpu().numpy())
        eng.diverse_ws_bytes = 1                                                  # one user per chunk
        one = eng.recommend_diverse(users, 10, 1.5, pool=60)
        for a, b in zip(one, base):
            assert support.same(a.cpu().numpy(), b.cpu().numpy())
    finally:
        eng.close()


def _stage_syncs(eng, pi, ps):
    """the host syncs of the diverse stage over finished pools, counted by torch's sync debug mode"""
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = eng._diverse(pi, ps, 10, 1.0)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, sum("called a synchronizing" in str(x.message) for x in w)


def test_independent_deterministic_sync_count():
    g = RatingGraph(support.adj("ml_1m"))
    m = support.model(5)
    users = _users(g, 12, 9)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=128)
    try:
        a = eng.recommend_diverse(users, 10, 1.0)
        b = eng.recommend_diverse(users, 10, 1.0)
        for x, y in zip(a, b):
            assert support.same(x.cpu().numpy(), y.cpu().numpy())
        more = np.r_[_users(g, 5, 77), users]
        c = eng.recommend_diverse(more, 10, 1.0)
        pos = [int(np.flatnonzero(more == u)[0]) for u in users]
        for x, y in zip(c, a):
            assert support.same(x.cpu().numpy()[pos], y.cpu().numpy())
        pi, ps = eng.recommend(users, 50)
        got, one = _stage_syncs(eng, pi, ps)
        assert one == 1                                                           # one chunk: one sync
        eng.diverse_ws_bytes = 1
        again, per_user = _stage_syncs(eng, pi, ps)
        assert 1 <= per_user <= len(users)                                        # at most one per chunk
        for x, y in zip(got, again):
            assert support.same(x.cpu().numpy(), y.cpu().numpy())
    finally:
        eng.close()


def test_served_across_updates():
    g = RatingGraph(support.adj("ml_100k"), reserve_nnz=50)
    m = support.model(5)
    users = np.array([1, 2, 40, 41], np.int64)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=64)
    try:
        first = eng.recommend_diverse(users, 5, 1.0, pool=20)
        top = int(first.items[0, 0])
        g.update([1, 2, 3, 4], [top, top, top, top], [4, 4, 4, 4])                 # user 1 rates its top item
        got = _check_lists(eng, g, users, 5, 1.0, 20)
        assert top not in got.items.cpu().numpy()[0]
        eng.start_recommend_diverse(users, 5, 1.0, pool=20)
        g.update([2], [int(first.items[1, 1])], [3])
        with pytest.raises(RuntimeError, match="updated during this run"):
            eng.finish()
        _check_lists(eng, g, users, 5, 1.0, 20)
    finally:
        eng.close()
