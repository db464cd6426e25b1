"""Host twins of the retriever (csrc/retrieve.cu) and of the per-user candidate lists (csrc/recommend.cu) against brute
force, and the input validation of the new arguments.

The retriever's twin is B B^T B without the u' = u term; brute force here counts the 3-paths u - i - u' - v one by one.
tests/test_gpu_retrieve.py holds the kernels to the twins byte for byte."""
import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import recommend as rc
from tests import support


def _brute_paths(A, u, exclude):
    nu, ni = A.shape
    R = [set(A.indices[A.indptr[x]:A.indptr[x + 1]].tolist()) for x in range(nu)]
    p = np.zeros(ni, np.int64)
    for v in range(ni):
        if exclude and v in R[u]:
            continue
        for u2 in range(nu):
            if u2 == u or v not in R[u2]:
                continue
            for i in R[u]:
                p[v] += i in R[u2]
    return p


def _brute_top(p, m):
    order = sorted((v for v in range(len(p)) if p[v] > 0), key=lambda v: (-p[v], v))[:m]
    items = np.full(m, -1, np.int32)
    paths = np.zeros(m, np.int32)
    items[:len(order)] = order
    paths[:len(order)] = p[order]
    return items, paths


@pytest.mark.parametrize("exclude", [True, False])
@pytest.mark.parametrize("m", [1, 3, 12, 25, 40])
@pytest.mark.parametrize("seed", range(3))
def test_corated_twin_matches_brute_force(seed, m, exclude):
    """users without ratings, items with one rater, m beyond the reachable set, m = 1 and m >= num_items"""
    nu, ni = 14, 25
    A = support.random_csr(nu, ni, 0.2 + 0.1 * seed, seed, empty_rows=(3,), single_cols=(4, 9))
    m = min(m, ni)
    users = np.array([0, 3, 5, 5, 13, 1], np.int64)
    rp, ci = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    items, paths = rc.corated_host(rp, ci, nu, ni, users, m, exclude)
    assert items.shape == (len(users), m) and items.dtype == np.int32 and paths.dtype == np.int32
    for j, u in enumerate(users):
        wi, wp = _brute_top(_brute_paths(A, int(u), exclude), m)
        assert np.array_equal(items[j], wi), (j, items[j], wi)
        assert np.array_equal(paths[j], wp), (j, paths[j], wp)
    assert (items[1] == -1).all() and (paths[1] == 0).all()          # no ratings: no bridge
    if exclude:
        for j, u in enumerate(users):
            assert not np.isin(items[j], ci[rp[u]:rp[u + 1]]).any()


def test_corated_twin_reachability_and_ties():
    """a path graph: only the items two hops away are reachable; equal counts in ascending item order"""
    # u0 - i0 - u1 - i1, u1 - i2, u2 - i0, u2 - i3
    A = ssp.csr_matrix((np.ones(6, np.float32), ([0, 1, 1, 1, 2, 2], [0, 0, 1, 2, 0, 3])), shape=(4, 5))
    A.sort_indices()
    items, paths = rc.corated_host(A.indptr, A.indices, 4, 5, [0, 3], 5, True)
    assert items[0].tolist() == [1, 2, 3, -1, -1] and paths[0].tolist() == [1, 1, 1, 0, 0]
    assert (items[1] == -1).all()
    items, paths = rc.corated_host(A.indptr, A.indices, 4, 5, [0], 5, False)
    assert items[0].tolist() == [0, 1, 2, 3, -1] and paths[0].tolist() == [2, 1, 1, 1, 0]


@pytest.mark.parametrize("exclude", [True, False])
def test_candidate_lists_twin(exclude):
    """dedupe, -1 slots, rated removal, a row of only empty slots, a user without ratings"""
    A = support.random_csr(6, 20, 0.3, 7, empty_rows=(2,))
    rp, ci = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    users = np.array([0, 2, 4, 0], np.int64)
    row0 = ci[rp[0]:rp[1]]
    rows = np.full((4, 8), -1, np.int64)
    rows[0, :5] = [7, 3, 7, -1, 19][:5]
    rows[1, :4] = [5, 5, 5, 0]
    rows[2, :] = -1
    rows[3, :len(row0[:4])] = row0[:4]
    rows[3, 6] = 11
    off, lists = rc.candidate_lists_host(rp, ci, 20, users, rows, exclude)
    assert off.dtype == np.int64 and len(off) == 5 and lists.dtype == np.int32
    for j, u in enumerate(users):
        rated = set(ci[rp[u]:rp[u + 1]].tolist())
        want = sorted({int(x) for x in rows[j] if x >= 0 and not (exclude and x in rated)})
        assert lists[off[j]:off[j + 1]].tolist() == want, j
    assert off[3] - off[2] == 0


def _fake_model():
    m = type("M", (), {})()
    m.flat_params = torch.zeros(1)
    return m


def test_validation_of_rows_and_retrieve():
    nu, ni = 5, 7
    A = support.random_csr(nu, ni, 0.4, 3)
    m = _fake_model()
    with pytest.raises(ValueError):            # row count != len(users)
        rc.recommend(m, A, [0, 1], 3, items=np.zeros((3, 2), np.int64))
    with pytest.raises(IndexError):            # ids outside [-1, num_items)
        rc.recommend(m, A, [0], 3, items=np.array([[0, ni]]))
    with pytest.raises(IndexError):
        rc.recommend(m, A, [0], 3, items=np.array([[-2, 1]]))
    with pytest.raises(TypeError):
        rc.recommend(m, A, [0], 3, items=np.array([[0.5, 1.0]]))
    with pytest.raises(ValueError):            # retrieve= with items=
        rc.recommend(m, A, [0], 3, items=[1, 2], retrieve=3)
    with pytest.raises(ValueError):
        rc.recommend(m, A, [0], 3, retrieve=0)
    with pytest.raises(ValueError):
        rc.recommend(m, A, [0], 3, retrieve=ni + 1)
    with pytest.raises(IndexError):            # users are still checked with per-user lists
        rc.recommend(m, A, [nu], 3, items=np.array([[0, 1]]))
    # -1 slots are valid; no query user: nothing to run
    ti, ts = rc.recommend(m, A, np.zeros(0, np.int64), 4, items=np.zeros((0, 3), np.int64))
    assert ti.shape == (0, 4) and ts.shape == (0, 4)
    ti, ts = rc.recommend(m, A, np.zeros(0, np.int64), 4, retrieve=2)
    assert ti.shape == (0, 4)
    assert rc._is_rows(np.zeros((2, 3))) and not rc._is_rows([1, 2]) and not rc._is_rows(None)
    rows = rc._user_rows([[0, -1, 6], [1, 1, 1]], 2, ni)
    assert rows.dtype == np.int32 and rows.tolist() == [[0, -1, 6], [1, 1, 1]]
