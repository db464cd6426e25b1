"""The cache repair of RecommendationCache on the host (igmc_b200/recommend.py, csrc/recommend_cache.cu), no GPU:

* the affected-set rule is sound: every pair whose canonical h = 1 subgraph (oracle/extract_np.py) differs before and
  after an update is in rescore_plan_host's plan, under max_nodes_per_hop None / 1 / 3 and sample_ratio 1 / 0.5, and
  the plan is strictly smaller than every pair;
* rescore_plan_host against a brute-force loop over pairs and edits, with a shared list and exclude_rated on and off;
* invalidate -> merge -> settle against brute-force sorts of every candidate: each settled prefix is the slot's exact
  ranking, and a slot falls back exactly when it keeps fewer than k entries - ties at the threshold, NaN, +-0, +-inf,
  incomplete prefixes, every item rescored and slots without candidates."""
import numpy as np
import pytest
import scipy.sparse as ssp

from igmc_b200 import recommend as rc
from oracle import extract_np


def _graph(rng, nu, ni, n):
    """a random rating matrix with empty rows and columns (the last user and item never rate)"""
    A = np.zeros((nu, ni), np.int64)
    for _ in range(n):
        A[rng.integers(nu - 1), rng.integers(ni - 1)] = rng.integers(1, 6)
    return A


def _apply(A, users, items, values):
    """RatingGraph.update on a dense matrix: the last occurrence of a pair wins, 0 deletes, new users grow the rows"""
    nu = max(A.shape[0], int(max(users)) + 1 if len(users) else 0)
    B = np.zeros((nu, A.shape[1]), np.int64)
    B[:A.shape[0]] = A
    for u, v, x in zip(users, items, values):
        B[u, v] = x
    return B


def _edits(rng, A, kind):
    nu, ni = A.shape
    rated = np.argwhere(A > 0)
    pick = rated[rng.integers(len(rated), size=2)]
    if kind == "insert":
        return [int(rng.integers(nu))] * 2, [int(rng.integers(ni)), int(rng.integers(ni))], [3, 4]
    if kind == "overwrite":
        return list(pick[:, 0]), list(pick[:, 1]), [5, 1]
    if kind == "delete":
        return list(pick[:, 0]), list(pick[:, 1]), [0, 0]
    if kind == "absent":                                   # deleting ratings that are not there
        z = np.argwhere(A == 0)[:2]
        return list(z[:, 0]), list(z[:, 1]), [0, 0]
    if kind == "repeat":                                   # the same pair twice, the last wins
        return [int(pick[0, 0])] * 2, [int(pick[0, 1])] * 2, [2, 0]
    return [nu, nu, nu + 1], [int(pick[0, 1]), int(pick[1, 1]), int(rng.integers(ni))], [2, 3, 1]   # new users


def _csr(A):
    S = ssp.csr_matrix(A)
    S.sort_indices()
    return S.indptr.astype(np.int64), S.indices.astype(np.int64)


@pytest.mark.parametrize("mnph,ratio", [(None, 1.0), (1, 1.0), (3, 1.0), (None, 0.5), (3, 0.5)])
@pytest.mark.parametrize("kind", ["insert", "overwrite", "delete", "absent", "repeat", "new_users"])
def test_affected_set_is_sound(mnph, ratio, kind):
    rng = np.random.default_rng([len(kind), ord(kind[0]), mnph or 0, int(ratio * 2)])
    for trial in range(3):
        A = _graph(rng, 9, 8, 22)
        eu, ev, ex = _edits(rng, A, kind)
        B = _apply(A, eu, ev, ex)
        nu, ni = A.shape
        old, new = extract_np.RatingCSR(ssp.csr_matrix(A)), extract_np.RatingCSR(ssp.csr_matrix(B))
        rp, ci = _csr(B)
        user_off, items, _, _ = rc.rescore_plan_host(rp, ci, ni, np.arange(nu), eu, ev, exclude_rated=False)
        plan = {(u, int(v)) for u in range(nu) for v in items[user_off[u]:user_off[u + 1]]}
        assert len(plan) < nu * ni
        for u in range(nu):
            for v in range(ni):
                kw = dict(h=1, sample_ratio=ratio, max_nodes_per_hop=mnph, seed=0, pair_id=u * ni + v)
                s0, s1 = extract_np.extract_subgraph(old, u, v, **kw), extract_np.extract_subgraph(new, u, v, **kw)
                if any(not np.array_equal(s0[key], s1[key]) for key in s0):
                    assert (u, v) in plan, (kind, trial, u, v)


@pytest.mark.parametrize("exclude_rated", [True, False])
@pytest.mark.parametrize("shared", [False, True])
def test_rescore_plan_twin_against_brute_force(exclude_rated, shared):
    rng = np.random.default_rng(7)
    for trial in range(6):
        A = _graph(rng, 12, 10, 30)
        eu, ev, ex = _edits(rng, A, ["insert", "overwrite", "delete", "new_users"][trial % 4])
        B = _apply(A, eu, ev, ex)
        rp, ci = _csr(B)
        ni = B.shape[1]
        cand = np.sort(rng.choice(ni, 6, replace=False)) if shared else None
        users = np.array([0, 3, 3, 11, int(eu[0]) if eu[0] < 12 else 1, 5])
        user_off, items, full, total = rc.rescore_plan_host(rp, ci, ni, users, eu, ev, cand, exclude_rated)
        want_total = 0
        for j, u in enumerate(users):
            cands = [v for v in range(ni) if (cand is None or v in cand) and not (exclude_rated and B[u, v] > 0)]
            want = [v for v in cands
                    if any(u == a or v == b or (B[u, b] > 0 and B[a, v] > 0) for a, b in zip(eu, ev))]
            assert list(items[user_off[j]:user_off[j + 1]]) == want
            assert full[j] == (len(want) == len(cands))
            want_total += len(cands)
        assert total == want_total


_POOL = np.array([-np.inf, -1.0, -0.0, 0.0, 0.5, 1.0, np.inf, np.nan], np.float32)


def _slot_case(rng, ni, D, k):
    """one slot: candidates, old and new scores, a cached exact prefix, its complete flag and the rescored items"""
    cands = np.sort(rng.choice(ni, int(rng.integers(0, ni + 1)), replace=False))
    old = _POOL[rng.integers(len(_POOL), size=ni)]
    top_s, top_i = rc.rank_host(old[cands], cands, D)
    nc = len(cands)
    n = int(rng.integers(min(k, nc), min(D, nc) + 1)) if nc else 0      # an exact prefix of k..D entries
    top_s[n:], top_i[n:] = -np.inf, -1
    complete = n == nc and (n < D or rng.random() < 0.5)
    mode = rng.integers(4)
    resc = cands if mode == 0 else cands[rng.random(nc) < (0.2 if mode == 1 else 0.7)]
    new = old.copy()
    new[resc] = _POOL[rng.integers(len(_POOL), size=len(resc))]
    return cands, new, top_s, top_i, complete, resc


@pytest.mark.parametrize("D,k", [(1, 1), (4, 1), (6, 3), (10, 10)])
def test_invalidate_merge_settle_against_brute_force(D, k):
    rng = np.random.default_rng(D * 31 + k)
    for trial in range(40):
        U, ni = 6, 12
        cases = [_slot_case(rng, ni, D, k) for _ in range(U)]
        top_s = np.stack([c[2] for c in cases])
        top_i = np.stack([c[3] for c in cases])
        complete = np.array([c[4] for c in cases], np.uint8)
        full = np.array([len(c[5]) == len(c[0]) for c in cases], np.uint8)
        user_off = np.concatenate([[0], np.cumsum([len(c[5]) for c in cases])]).astype(np.int64)
        resc = np.concatenate([c[5] for c in cases]).astype(np.int32)
        s, i, thr_s, thr_i = rc.cache_invalidate_host(user_off, resc, full, complete, top_s, top_i)
        for j, c in enumerate(cases):
            kept = [x for x in top_i[j] if x >= 0 and x not in c[5]]
            assert list(i[j][i[j] >= 0]) == kept
            s[j], i[j] = rc.topk_merge_host(s[j], i[j], c[1][c[5]], c[5])
        s, i, comp, redo = rc.cache_settle_host(thr_s, thr_i, s, i, k)
        for j, (cands, new, _, _, _, _) in enumerate(cases):
            d = int((i[j] >= 0).sum())
            want_s, want_i = rc.rank_host(new[cands], cands, D)
            assert np.array_equal(i[j][:d], want_i[:d]) and np.array_equal(s[j][:d], want_s[:d], equal_nan=True)
            assert (j in redo) == (d < min(k, len(cands))), (trial, j, d)
            if comp[j]:
                assert d == len(cands)
