"""Host twins of the inference kernels (csrc/recommend.cu) against brute force, and the API's input validation.

The twins restate the kernels' integer arithmetic: per-user candidate counts and offsets, the rated positions in a
candidate list, the position -> (user, item) mapping by two binary searches (tail-batch padding included), and the
rank-counting merge of a batch segment into a running top-k list.  tests/test_gpu_recommend.py holds the kernels to
the twins bit for bit."""
import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import recommend as rc
from tests import support


def _brute(A, users, cand, exclude):
    """per query user the ascending candidate items"""
    ni = A.shape[1]
    base = np.arange(ni) if cand is None else np.unique(cand)
    out = []
    for u in users:
        rated = set(A.indices[A.indptr[u]:A.indptr[u + 1]].tolist())
        out.append([int(v) for v in base if not (exclude and v in rated)])
    return out


CASES = [
    # (label, candidate list builder)
    ("all items", lambda A, rng: None),
    ("list hitting no row", lambda A, rng: np.array([A.shape[1] - 1])),
    ("random list", lambda A, rng: rng.choice(A.shape[1], A.shape[1] // 3, replace=False)),
    ("list = a whole row", lambda A, rng: A.indices[A.indptr[2]:A.indptr[3]].copy()),
    ("list with duplicates", lambda A, rng: rng.integers(0, A.shape[1], 40)),
]


@pytest.mark.parametrize("exclude", [True, False])
@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("B", [1, 7, 64])
def test_candidate_plan_and_pairs_match_brute_force(case, exclude, B):
    A = support.random_csr(12, 30, 0.3, seed=case, full_rows=(0,), empty_rows=(1,))
    A = ssp.csr_matrix(A)
    A.data[A.indices == A.shape[1] - 1] = 0       # the last item has no rating: a list of it hits no row
    A.eliminate_zeros()
    rng = np.random.default_rng(10 + case)
    cand = CASES[case][1](A, rng)
    cand = None if cand is None else np.unique(cand)
    users = np.array([0, 1, 2, 5, 2, 11, 7, 1], np.int64)          # rated every item, no rating, repeated users
    rp, ci, ni = A.indptr.astype(np.int64), A.indices.astype(np.int64), A.shape[1]
    plan = rc.candidate_plan_host(rp, ci, ni, users, cand, exclude)
    want = _brute(A, users, cand, exclude)
    assert np.array_equal(np.diff(plan[0]), [len(w) for w in want])
    if exclude and cand is not None:
        for j, u in enumerate(users):       # positions in the list of the user's rated items, ascending
            pos = plan[2][plan[1][j]:plan[1][j + 1]]
            rated = set(A.indices[A.indptr[u]:A.indptr[u + 1]].tolist())
            assert pos.tolist() == [p for p, v in enumerate(cand) if v in rated]
    P = int(plan[0][-1])
    flat = [(j, int(users[j]), v) for j in range(len(users)) for v in want[j]]
    assert len(flat) == P
    if P == 0:
        return
    for pos in range(0, P + B, B):          # one batch past the end: all padding
        got = rc.candidate_pairs_host(rp, ci, ni, users, cand, exclude, plan, pos, B)
        for i in range(B):
            g = pos + i
            j, u, v = flat[min(g, P - 1)]
            assert got[0, i] == u and got[1, i] == v and got[2, i] == u * ni + v
            assert got[3, i] == (j if g < P else -1)


def test_rated_everything_and_unrated_nothing():
    A = support.random_csr(4, 9, 0.0, 0, full_rows=(0, 3))
    rp, ci = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    for users in ([0, 3], [0], [3, 0, 3]):
        plan = rc.candidate_plan_host(rp, ci, 9, np.array(users), None, True)
        assert int(plan[0][-1]) == 0
    plan = rc.candidate_plan_host(rp, ci, 9, np.array([0, 1]), None, True)
    assert np.array_equal(plan[0], [0, 0, 9])
    got = rc.candidate_pairs_host(rp, ci, 9, np.array([0, 1]), None, True, plan, 0, 12)
    assert got[1, :9].tolist() == list(range(9)) and set(got[0, :9].tolist()) == {1}
    assert (got[3, 9:] == -1).all() and (got[1, 9:] == 8).all()


def _stream(scores, items, k, cuts):
    """the running list after merging the candidates in segments cut at ``cuts``"""
    ts, ti = np.full(k, -np.inf, np.float32), np.full(k, -1, np.int64)
    bounds = [0] + sorted(cuts) + [len(scores)]
    for a, b in zip(bounds[:-1], bounds[1:]):
        if b > a:
            ts, ti = rc.topk_merge_host(ts, ti, scores[a:b], items[a:b])
    return ts, ti


def _sorted_key(s, v):
    return (2, 0.0, v) if np.isnan(s) else (0, -float(s), v)


@pytest.mark.parametrize("k", [1, 3, 10, 40])
@pytest.mark.parametrize("seed", range(4))
def test_streaming_topk_order(k, seed):
    """ties (scores drawn from 5 values), NaN, +-inf, k above the candidate count; the list does not depend on where
    the segments are cut"""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 30))
    items = np.sort(rng.choice(200, n, replace=False)).astype(np.int64)
    scores = rng.choice(np.array([0.5, 1.0, -2.0, np.nan, np.inf, -np.inf, 0.0, -0.0], np.float32), n)
    ref = sorted(zip(scores.tolist(), items.tolist()), key=lambda t: _sorted_key(*t))[:k]
    want_s, want_i = rc.rank_host(scores, items, k)
    assert want_i[:len(ref)].tolist() == [v for _, v in ref]
    assert (want_i[len(ref):] == -1).all() and np.isneginf(want_s[len(ref):]).all()
    for trial in range(5):
        cuts = rng.choice(np.arange(1, n + 1), int(rng.integers(0, n + 1)), replace=False).tolist() if n > 1 else []
        got_s, got_i = _stream(scores, items, k, cuts)
        assert np.array_equal(got_i, want_i), (cuts, got_i, want_i)
        assert np.array_equal(got_s, want_s, equal_nan=True)


def test_validation_errors():
    nu, ni = 5, 7
    A = support.random_csr(nu, ni, 0.4, 3)
    m = type("M", (), {})()
    m.flat_params = torch.zeros(1)
    with pytest.raises(ValueError):
        rc.recommend(m, A, [0], 0)
    with pytest.raises(NotImplementedError):
        rc.recommend(m, A, [0], 257)
    with pytest.raises(IndexError):
        rc.recommend(m, A, [nu], 3)
    with pytest.raises(IndexError):
        rc.recommend(m, A, [-1], 3)
    with pytest.raises(IndexError):
        rc.recommend(m, A, [0], 3, items=[ni])
    with pytest.raises(IndexError):
        rc.predict_pairs(m, A, [0, 1], [0, ni])
    with pytest.raises(IndexError):
        rc.predict_pairs(m, A, torch.tensor([0, nu]), torch.tensor([0, 1]))
    with pytest.raises(ValueError):
        rc.predict_pairs(m, A, [0, 1], [0])
    with pytest.raises(TypeError):
        rc.predict_pairs(m, A, [0.5], [0])
    ti, ts = rc.recommend(m, A, np.zeros(0, np.int64), 4)
    assert ti.shape == (0, 4) and ti.dtype == torch.int64 and ts.shape == (0, 4) and ts.dtype == torch.float32
    s = rc.predict_pairs(m, A, [], [])
    assert s.shape == (0,) and s.dtype == torch.float32


def test_candidates_struct_matches_header_layout():
    import ctypes
    from igmc_b200 import _lib
    P = ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(_lib.Candidates) == 7 * P + 8 + 16     # igmc_candidates_t
    assert _lib.TOPK_MAX == 256
