"""Host twins of the item-side retriever (igmc_corated_users) and of the item-side pair post-pass
(igmc_item_query_pairs) against brute force, the symmetry with the user-side retriever, and the input validation of
recommend_users / corated_users.

The item-side count is C[u][v] = (B B^T B)[u][v] - deg(u) B[u][v]: brute force here counts the 3-paths u - i - u' - v
with u' != u one by one.  tests/test_gpu_recommend_users.py holds the kernels to the twins byte for byte."""
import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import recommend as rc
from tests import support


def _brute_counts(A, v, exclude):
    """per user u the 3-paths u - i - u' - v with u' != u, one by one"""
    nu = A.shape[0]
    R = [set(A.indices[A.indptr[x]:A.indptr[x + 1]].tolist()) for x in range(nu)]
    c = np.zeros(nu, np.int64)
    for u in range(nu):
        if exclude and v in R[u]:
            continue
        for u2 in range(nu):
            if u2 == u or v not in R[u2]:
                continue
            for i in R[u]:
                c[u] += i in R[u2]
    return c


def _brute_top(c, m):
    order = sorted((u for u in range(len(c)) if c[u] > 0), key=lambda u: (-c[u], u))[:m]
    users = np.full(m, -1, np.int32)
    paths = np.zeros(m, np.int32)
    users[:len(order)] = order
    paths[:len(order)] = c[order]
    return users, paths


@pytest.mark.parametrize("exclude", [True, False])
@pytest.mark.parametrize("m", [1, 2, 5, 13, 30])
@pytest.mark.parametrize("seed", range(3))
def test_corated_users_twin_matches_brute_force(seed, m, exclude):
    """empty rows and columns (users and items without ratings), m = 1, m beyond the reachable users, m = num_users"""
    nu, ni = 16, 11
    A = support.random_csr(nu, ni, 0.25 + 0.1 * seed, seed, empty_rows=(2, 9), empty_cols=(4,))
    m = min(m, nu)
    items = np.array([0, 4, 3, 3, 10, 7], np.int64)
    rp, ci = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    users, paths = rc.corated_users_host(rp, ci, nu, ni, items, m, exclude)
    assert users.shape == (len(items), m) and users.dtype == np.int32 and paths.dtype == np.int32
    for j, v in enumerate(items):
        wu, wp = _brute_top(_brute_counts(A, int(v), exclude), m)
        assert np.array_equal(users[j], wu), (j, users[j], wu)
        assert np.array_equal(paths[j], wp), (j, paths[j], wp)
    assert (users[1] == -1).all() and (paths[1] == 0).all()          # nobody rated item 4: no bridge
    assert not np.isin(users, [2, 9]).any()                          # users without ratings have no bridge
    if exclude:
        for j, v in enumerate(items):
            raters = np.flatnonzero(A[:, int(v)].toarray().ravel())
            assert not np.isin(users[j], raters).any()


def test_corated_users_twin_ties_at_the_mth_place():
    """a star of equal counts: the m-th place is a tie, broken towards the lower user id"""
    # users 1..4 each rated items 0 and 1; user 0 rated item 0 only: every u in 1..4 reaches item 1 through the other
    # three raters of item 1 and both items it shares with each (6 paths); user 0 through item 0 and four raters (4)
    rows = [0, 1, 1, 2, 2, 3, 3, 4, 4]
    cols = [0, 0, 1, 0, 1, 0, 1, 0, 1]
    A = ssp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(5, 2))
    A.sort_indices()
    users, paths = rc.corated_users_host(A.indptr, A.indices, 5, 2, [1], 3, False)
    assert users[0].tolist() == [1, 2, 3] and paths[0].tolist() == [6, 6, 6]
    users, paths = rc.corated_users_host(A.indptr, A.indices, 5, 2, [1], 5, False)
    assert users[0].tolist() == [1, 2, 3, 4, 0] and paths[0].tolist() == [6, 6, 6, 6, 4]
    users, paths = rc.corated_users_host(A.indptr, A.indices, 5, 2, [1], 2, True)
    assert users[0].tolist() == [0, -1] and paths[0].tolist() == [4, 0]
    for j, v in enumerate([1]):
        for excl in (True, False):
            for m in (1, 2, 3, 4, 5):
                wu, wp = _brute_top(_brute_counts(A, v, excl), m)
                got = rc.corated_users_host(A.indptr, A.indices, 5, 2, [v], m, excl)
                assert np.array_equal(got[0][0], wu) and np.array_equal(got[1][0], wp), (excl, m)


def _dense_counts(ids, paths, n):
    """the [rows, n] count matrix of a retriever result that kept every id (m = n)"""
    D = np.zeros((ids.shape[0], n), np.int64)
    for j in range(ids.shape[0]):
        keep = ids[j] >= 0
        D[j, ids[j][keep]] = paths[j][keep]
    return D


@pytest.mark.parametrize("exclude", [True, False])
@pytest.mark.parametrize("seed", range(4))
def test_item_side_counts_are_the_user_side_counts(seed, exclude):
    """corated_users_host(items)[v][u] == corated_host(users)[u][v] for every pair: one count seen from either side"""
    nu, ni = 21, 17
    A = support.random_csr(nu, ni, 0.15 + 0.08 * seed, 10 + seed, empty_rows=(0,), empty_cols=(5,))
    rp, ci = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    iu, ip = rc.corated_host(rp, ci, nu, ni, np.arange(nu), ni, exclude)
    uu, up = rc.corated_users_host(rp, ci, nu, ni, np.arange(ni), nu, exclude)
    by_user, by_item = _dense_counts(iu, ip, ni), _dense_counts(uu, up, nu)
    assert np.array_equal(by_user, by_item.T)
    assert by_user.sum() > 0


def _transposed_host(A):
    """the transposed view's arrays: rows are items (G's columns), columns users"""
    C = A.tocsc()
    C.sort_indices()
    return C.indptr.astype(np.int64), C.indices.astype(np.int64)


@pytest.mark.parametrize("exclude", [True, False])
@pytest.mark.parametrize("which", ["all", "list"])
def test_item_query_pairs_twin_enumerates_the_item_side_pairs(which, exclude):
    """the candidate kernels' twins run on the transposed arrays, then item_query_pairs_host: per query item, in query
    order, its candidate users ascending as (user, item) pairs with pair id u * num_items + v; the tail repeats the
    last pair with tag -1"""
    nu, ni = 13, 9
    A = support.random_csr(nu, ni, 0.3, 5, empty_rows=(4,), empty_cols=(2,))
    trp, tci = _transposed_host(A)
    items = np.array([1, 2, 8, 1, 0], np.int64)
    cand = None if which == "all" else np.array([0, 3, 4, 7, 11, 12], np.int64)
    plan = rc.candidate_plan_host(trp, tci, nu, items, cand, exclude)
    P = int(plan[0][-1])
    want = []
    for j, v in enumerate(items):
        raters = set(A[:, int(v)].nonzero()[0].tolist())
        for u in (range(nu) if cand is None else cand):
            if not (exclude and u in raters):
                want.append((u, v, u * ni + v, j))
    assert P == len(want) > 0
    want = np.array(want, np.int64).T
    B = 7
    got = []
    for pos in range(0, P + B, B):
        lu, lv, pid, tag = rc.candidate_pairs_host(trp, tci, nu, items, cand, exclude, plan, pos, B)
        assert np.array_equal(pid, lu * nu + lv)                    # the transposed pair id before the post-pass
        u, v, pid2 = rc.item_query_pairs_host(ni, lu, lv)
        got.append(np.stack([u, v, pid2, tag]))
    got = np.concatenate(got, 1)
    real = got[3] >= 0
    assert real.sum() == P and real[:P].all()
    assert np.array_equal(got[:, :P], want)
    assert (got[:3, P:] == want[:3, -1:]).all()                     # the tail: the last pair, swapped like the rest


def test_item_query_pairs_twin_int64_pair_ids():
    u, v, pid = rc.item_query_pairs_host(3_000_000, [2_999_999, 0], [1_000, 999_999])
    assert u.tolist() == [1_000, 999_999] and v.tolist() == [2_999_999, 0]
    assert pid.dtype == np.int64 and pid.tolist() == [1_000 * 3_000_000 + 2_999_999, 999_999 * 3_000_000]


def _fake_model():
    m = type("M", (), {})()
    m.flat_params = torch.zeros(1)
    return m


def test_validation_of_recommend_users():
    nu, ni = 6, 5
    A = support.random_csr(nu, ni, 0.4, 3)
    m = _fake_model()
    for k in (0, 257):
        with pytest.raises((ValueError, NotImplementedError)):
            rc.recommend_users(m, A, [0], k)
    with pytest.raises(IndexError):            # item id out of range
        rc.recommend_users(m, A, [ni], 3)
    with pytest.raises(IndexError):
        rc.recommend_users(m, A, [-1], 3)
    with pytest.raises(IndexError):            # a candidate user out of range
        rc.recommend_users(m, A, [0], 3, users=[0, nu])
    with pytest.raises(ValueError):            # per-item rows: one per query item
        rc.recommend_users(m, A, [0, 1], 3, users=np.zeros((3, 2), np.int64))
    with pytest.raises(IndexError, match="users"):
        rc.recommend_users(m, A, [0], 3, users=np.array([[0, nu]]))
    with pytest.raises(TypeError):
        rc.recommend_users(m, A, [0], 3, users=np.array([[0.5, 1.0]]))
    with pytest.raises(ValueError, match="without users="):
        rc.recommend_users(m, A, [0], 3, users=[1, 2], retrieve=3)
    for M in (0, nu + 1):                     # retrieve= counts users: 1 <= M <= num_users
        with pytest.raises(ValueError):
            rc.recommend_users(m, A, [0], 3, retrieve=M)
    with pytest.raises(ValueError, match="top-k merge"):     # k + batch_size beyond one CTA's shared memory
        rc.recommend_users(m, A, [0], 256, batch_size=19369 - 255)
    # no query item: nothing to run
    tu, ts = rc.recommend_users(m, A, np.zeros(0, np.int64), 4)
    assert tu.shape == (0, 4) and tu.dtype == torch.int64 and ts.shape == (0, 4) and ts.dtype == torch.float32
    tu, ts = rc.recommend_users(m, A, np.zeros(0, np.int64), 4, users=np.zeros((0, 3), np.int64))
    assert tu.shape == (0, 4)


def test_validation_of_corated_users():
    nu, ni = 6, 5
    A = support.random_csr(nu, ni, 0.4, 3)
    for M in (0, nu + 1):                     # 1 <= m <= num_users
        with pytest.raises(ValueError):
            rc.corated_users(A, [0], M)
    with pytest.raises(IndexError):
        rc.corated_users(A, [ni], 2)
    with pytest.raises(TypeError):
        rc.corated_users(A, [0.5], 2)
