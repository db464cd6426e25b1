"""Host twins of the counterfactual kernels (csrc/counterfactual.cu) and the greedy search they run.

* counterfactual_pairs_host against brute-force enumeration of the trials of a pass;
* counterfactual_select_host against the selection order restated with Python's sort;
* the greedy search composed of the two twins, driven by a toy scorer, against counterfactual_host (the contract
  restated as a plain loop): ties, NaN scores, flips by a tie and every stop rule;
* the argument checks of ``counterfactual``."""
import types

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import recommend as rc


def _graph(seed, nu=9, ni=14, density=0.35, R=5):
    """a small rating matrix as (row_ptr, col_idx, rating) with user 0's row empty"""
    rng = np.random.default_rng(seed)
    A = (rng.random((nu, ni)) < density) * rng.integers(1, R + 1, (nu, ni))
    A[0] = 0
    A = ssp.csr_matrix(A.astype(np.float32))
    A.sort_indices()
    return A, A.indptr.astype(np.int64), A.indices.astype(np.int32), (A.data - 1).astype(np.uint8)


def _state(Q, M):
    return dict(removed=np.zeros((Q, M), np.int32), size=np.zeros(Q, np.int32), count=np.ones(Q, np.int32),
                found=np.zeros(Q, bool), items=np.full((Q, M), -1, np.int32), ratings=np.full((Q, M), -1, np.int32),
                score=np.full((Q, M + 1), np.nan, np.float32), rival_score=np.full((Q, M + 1), np.nan, np.float32))


# ---- the pairs / rows twin ------------------------------------------------------------------------------------------
def _brute_trials(rp, ci, users, removed, size, count, step):
    """every trial of a pass in order: (q, set of removed row positions)"""
    out = []
    for q, u in enumerate(users):
        deg = int(rp[u + 1] - rp[u])
        R = set(int(x) for x in removed[q][:size[q]])
        if step == 0:
            out += [(q, R)] * int(count[q])
            continue
        free = [p for p in range(deg) if p not in R]
        assert count[q] in (0, len(free))                             # a query done, or one trial per free position
        out += [(q, R | {p}) for p in free] if count[q] else []
    return out


@pytest.mark.parametrize("B", [1, 2, 5, 7, 64])
@pytest.mark.parametrize("step", [0, 1, 3])
def test_pairs_twin_matches_enumeration(B, step):
    A, rp, ci, rt = _graph(1)
    ni = A.shape[1]
    users = np.array([3, 0, 5, 3, 8, 2], np.int64)                # a zero-degree user, a duplicated query
    items = np.array([1, 4, 2, 1, 0, 13], np.int64)
    rivals = np.array([2, 5, 3, 2, 7, 12], np.int64)
    Q, M = len(users), 4
    rng = np.random.default_rng(step)
    st = _state(Q, M)
    deg = rp[users + 1] - rp[users]
    for q in range(Q):
        t = min(step - 1, int(deg[q])) if step > 0 else 0
        st["size"][q] = t
        st["removed"][q, :t] = np.sort(rng.choice(int(deg[q]), t, replace=False)) if t else []
        st["count"][q] = (deg[q] - t if deg[q] - t > 0 and q != 4 else 0) if step > 0 else 1
    offsets = rc.explain_offsets_host(st["count"])
    trials = _brute_trials(rp, ci, users, st["removed"], st["size"], st["count"], step)
    P2 = 2 * len(trials)
    assert P2 == 2 * offsets[-1] and P2 > 0
    for pos in list(range(0, P2, B)) + [P2 + 3]:                    # the last start is an all-padding batch
        out, (ru, rptr, rcol, rrat) = rc.counterfactual_pairs_host(rp, ci, rt, ni, users, items, rivals, st["removed"],
                                                                   st["size"], offsets, step, pos, B)
        assert rptr[0] == 0 and len(rptr) == B + 1
        for i in range(B):
            p = min(pos + i, P2 - 1)
            q, R = trials[p >> 1]
            u = int(users[q])
            v = int(rivals[q] if p & 1 else items[q])
            assert tuple(out[:, i]) == (u, v, u * ni + v, pos + i if pos + i < P2 else -1)
            assert ru[i] == u
            keep = [k for k in range(int(rp[u + 1] - rp[u])) if k not in R]
            assert list(rcol[rptr[i]:rptr[i + 1]]) == list(ci[rp[u] + np.array(keep, np.int64)]) if keep else \
                rptr[i + 1] == rptr[i]
            assert list(rrat[rptr[i]:rptr[i + 1]]) == list(rt[rp[u] + np.array(keep, np.int64)]) if keep else True


# ---- the select twin ------------------------------------------------------------------------------------------------
def _ahead(a_s, a_i, b_s, b_i):
    """recommend's order restated: the non-NaN score first, the larger score first, then the smaller item"""
    an, bn = np.isnan(a_s), np.isnan(b_s)
    if an != bn:
        return bn
    if not an and a_s != b_s:
        return a_s > b_s
    return a_i < b_i


@pytest.mark.parametrize("seed", range(6))
def test_select_twin_matches_sorted_order(seed):
    A, rp, ci, rt = _graph(seed + 10)
    rng = np.random.default_rng(seed)
    users = np.array([1, 2, 0, 4, 6, 1], np.int64)
    items = np.array([0, 3, 1, 5, 2, 9], np.int64)
    rivals = np.array([1, 2, 4, 6, 8, 0], np.int64)
    Q, M = len(users), 3
    st = _state(Q, M)
    deg = rp[users + 1] - rp[users]
    for q in range(Q):
        t = min(1, int(deg[q]))
        st["size"][q] = t
        st["removed"][q, :t] = rng.choice(int(deg[q]), t, replace=False) if t else []
        st["count"][q] = deg[q] - t
    st["count"][5] = 0                                                  # a query already done
    offsets = rc.explain_offsets_host(st["count"])
    T = int(offsets[-1])
    # few distinct values: ties in score and margin, NaN in both
    scores = rng.choice(np.array([0.5, 1.0, 1.5, np.nan], np.float32), 2 * T)
    before = {k: v.copy() for k, v in st.items()}
    rc.counterfactual_select_host(rp, ci, rt, users, items, rivals, offsets, scores, 1, st)
    for q in range(Q):
        n = int(offsets[q + 1] - offsets[q])
        if n == 0:
            assert st["count"][q] == 0 and st["size"][q] == before["size"][q]
            continue
        u, X, Y, t = int(users[q]), int(items[q]), int(rivals[q]), int(before["size"][q])
        free = [p for p in range(int(deg[q])) if p not in set(before["removed"][q, :t])]
        trials = []
        for c, pos in enumerate(free):
            sx, sy = scores[2 * (offsets[q] + c)], scores[2 * (offsets[q] + c) + 1]
            m = np.float32(sx - sy)
            trials.append(((not _ahead(sy, Y, sx, X)), bool(np.isnan(m)), 0.0 if np.isnan(m) else float(m),
                           int(ci[rp[u] + pos]), pos, sx, sy, _ahead(sy, Y, sx, X)))
        best = sorted(trials)[0]
        assert st["items"][q, t] == best[3] and st["ratings"][q, t] == rt[rp[u] + best[4]]
        assert list(st["removed"][q, :t + 1]) == sorted(list(before["removed"][q, :t]) + [best[4]])
        assert np.array_equal(st["score"][q, t + 1:t + 2], np.float32([best[5]]), equal_nan=True)
        assert np.array_equal(st["rival_score"][q, t + 1:t + 2], np.float32([best[6]]), equal_nan=True)
        assert st["found"][q] == best[7] and st["size"][q] == t + 1
        done = best[7] or t + 1 == M or deg[q] == t + 1
        assert st["count"][q] == (0 if done else deg[q] - t - 1)


# ---- the greedy search ----------------------------------------------------------------------------------------------
def _toy_scorer(seed, levels=4, nan_items=()):
    """score(u, deleted, v) = base(u, v) - sum of w(u, i, v) over deleted i, on a coarse grid (many ties); deleting an
    item of ``nan_items`` makes the score NaN"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, levels, (64, 64)).astype(np.float32)
    w = rng.integers(0, 2, (64, 64, 64)).astype(np.float32) * np.float32(0.5)

    def one(u, deleted, v):
        if any(int(i) in nan_items for i in deleted):
            return np.float32(np.nan)
        s = base[u, v]
        for i in deleted:
            s = np.float32(s - w[u, int(i), v])
        return s

    def batch(users, deleted, targets):
        return np.array([one(int(u), d, int(v)) for u, d, v in zip(users, deleted, targets)], np.float32)
    return one, batch


def _greedy_by_twins(rp, ci, rt, ni, users, items, rivals, M, score_one, B):
    """the engine's pass loop on the twins: offsets, the pairs of every batch, their scores by tag, the selection"""
    Q = len(users)
    st = _state(Q, M)
    step = 0
    while True:
        offsets = rc.explain_offsets_host(st["count"])
        P2 = 2 * int(offsets[-1])
        if P2 == 0:
            break
        scores = np.full(P2, -7.0, np.float32)
        for pos in range(0, P2, B):
            out, (ru, rptr, rcol, _) = rc.counterfactual_pairs_host(rp, ci, rt, ni, users, items, rivals,
                                                                    st["removed"], st["size"], offsets, step, pos, B)
            for g in range(B):
                if out[3, g] < 0:
                    continue
                u = int(out[0, g])
                deleted = sorted(set(ci[rp[u]:rp[u + 1]]) - set(rcol[rptr[g]:rptr[g + 1]]))
                scores[out[3, g]] = score_one(u, deleted, int(out[1, g]))
        rc.counterfactual_select_host(rp, ci, rt, users, items, rivals, offsets, scores, step, st)
        step += 1
        assert step <= M + 1
    return st


def _same(st, cf):
    assert np.array_equal(st["found"], cf.found) and np.array_equal(st["size"], cf.size)
    assert np.array_equal(st["items"], cf.items) and np.array_equal(st["ratings"], cf.ratings)
    assert np.array_equal(st["score"], cf.score, equal_nan=True)
    assert np.array_equal(st["rival_score"], cf.rival_score, equal_nan=True)


@pytest.mark.parametrize("seed,M,B,nan_items", [(0, 3, 1, ()), (1, 5, 3, ()), (2, 10, 7, (2, 5)), (3, 2, 50, (0,)),
                                                 (4, 14, 4, ())])
def test_greedy_twins_match_restated_contract(seed, M, B, nan_items):
    A, rp, ci, rt = _graph(seed + 20, density=0.5)
    nu, ni = A.shape
    rng = np.random.default_rng(seed)
    Q = 12
    users = np.r_[[0], rng.integers(1, nu, Q - 1)]
    items = rng.integers(0, ni, Q)
    rivals = (items + rng.integers(1, ni, Q)) % ni
    users[5], items[5], rivals[5] = users[4], items[4], rivals[4]      # a duplicated query
    one, batch = _toy_scorer(seed, nan_items=set(nan_items))
    want = rc.counterfactual_host(rp, ci, rt, users, items, rivals, M, batch)
    _same(_greedy_by_twins(rp, ci, rt, ni, users, items, rivals, M, one, B), want)
    deg = rp[users + 1] - rp[users]
    # the stop rules, restated on the result
    for q in range(Q):
        t = int(want.size[q])
        behind = not _ahead(want.score[q, t], items[q], want.rival_score[q, t], rivals[q])
        assert bool(want.found[q]) == behind
        assert want.found[q] or t == M or t == deg[q]
        assert (want.items[q, t:] == -1).all() and np.isnan(want.score[q, t + 1:]).all()
        assert len(set(want.items[q, :t])) == t and set(want.items[q, :t]) <= set(ci[rp[users[q]]:rp[users[q] + 1]])


def test_ties_nan_and_flip_by_tie():
    """one user rating items 1, 2, 3, 4 with hand-set scores"""
    A = ssp.csr_matrix(np.array([[0, 1, 2, 3, 4, 0, 0]], np.float32))
    rp, ci, rt = A.indptr.astype(np.int64), A.indices.astype(np.int32), (A.data - 1).astype(np.uint8)

    def scorer_of(table):
        def batch(users, deleted, targets):
            return np.array([table(frozenset(int(i) for i in d), int(v)) for d, v in zip(deleted, targets)],
                            np.float32)
        return batch

    # X = 5, Y = 6: X ahead at 3.0 vs 2.0.  Step 1: removing 2 or 3 gives the least margin, 0.5 (item 2 wins the
    # tie); step 2: removing 1 as well makes s(X) NaN, which ranks X behind Y
    def table(R, v):
        if v == 6:
            return 2.0
        if 1 in R and len(R) >= 2:
            return np.nan
        return 3.0 - 0.5 * len(R & {2, 3}) - 0.5 * (4 in R) * (len(R) > 1)
    cf = rc.counterfactual_host(rp, ci, rt, [0], [5], [6], 4, scorer_of(table))
    assert list(cf.items[0]) == [2, 1, -1, -1] and list(cf.ratings[0]) == [1, 0, -1, -1]
    assert cf.found[0] and cf.size[0] == 2
    assert list(cf.score[0, :2]) == [3.0, 2.5] and np.isnan(cf.score[0, 2]) and cf.rival_score[0, 2] == 2.0
    # a flip by a tie: equal scores, X = 6 > Y = 5, so X is behind Y under the tie
    cf = rc.counterfactual_host(rp, ci, rt, [0], [6], [5], 4,
                                scorer_of(lambda R, v: 1.0 if v == 5 else 2.0 - 1.0 * (3 in R)))
    assert list(cf.items[0]) == [3, -1, -1, -1] and cf.found[0] and cf.score[0, 1] == cf.rival_score[0, 1]
    # already behind at step 0: size 0, found
    cf = rc.counterfactual_host(rp, ci, rt, [0], [5], [6], 4, scorer_of(lambda R, v: float(v == 6)))
    assert cf.found[0] and cf.size[0] == 0 and (cf.items[0] == -1).all() and np.isnan(cf.score[0, 1:]).all()
    # never behind: stops at max_removals, then at the end of the row
    for M, size in ((2, 2), (6, 4)):
        cf = rc.counterfactual_host(rp, ci, rt, [0], [5], [6], M, scorer_of(lambda R, v: float(v == 5)))
        assert not cf.found[0] and cf.size[0] == size and list(cf.items[0, :size]) == [1, 2, 3, 4][:size]
    # the twins agree on all of it
    for X, Y, tab, M in ((5, 6, table, 4), (6, 5, lambda R, v: 1.0 if v == 5 else 2.0 - (3 in R), 4),
                         (5, 6, lambda R, v: float(v == 5), 6)):
        def one(u, deleted, v, tab=tab):
            return np.float32(tab(frozenset(int(i) for i in deleted), v))
        _same(_greedy_by_twins(rp, ci, rt, 7, np.array([0]), np.array([X]), np.array([Y]), M, one, 3),
              rc.counterfactual_host(rp, ci, rt, [0], [X], [Y], M, scorer_of(tab)))


# ---- argument checks ------------------------------------------------------------------------------------------------
def test_argument_checks():
    A = ssp.csr_matrix(np.eye(5, 6, dtype=np.float32))
    model = types.SimpleNamespace(flat_params=torch.zeros(1))
    with pytest.raises(IndexError):
        rc.counterfactual(model, A, [5], [0], [1])
    with pytest.raises(IndexError):
        rc.counterfactual(model, A, [0], [6], [1])
    with pytest.raises(IndexError):
        rc.counterfactual(model, A, [0], [0], [-1])
    with pytest.raises(ValueError):
        rc.counterfactual(model, A, [0, 1], [0], [1])
    with pytest.raises(ValueError):
        rc.counterfactual(model, A, [0], [0], [1, 2])
    with pytest.raises(ValueError):
        rc.counterfactual(model, A, [0, 1], [2, 3], [1, 3])
    with pytest.raises(ValueError):
        rc.counterfactual(model, A, [0], [0], [1], max_removals=0)
    with pytest.raises(NotImplementedError):
        rc.counterfactual(model, A, [0], [0], [1], max_removals=257)
    with pytest.raises(TypeError):
        rc.counterfactual(model, A, [0], [0.5], [1])
    cf = rc.counterfactual(model, A, [], [], [], max_removals=7)
    assert cf.found.shape == (0,) and cf.items.shape == (0, 7) and cf.score.shape == (0, 8)
    assert cf.found.dtype == torch.bool and cf.size.dtype == torch.int32 and cf.score.dtype == torch.float32
