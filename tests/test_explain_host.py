"""Host twins of the explanation kernels (igmc_b200/recommend.py, csrc/explain.cu) against brute force: the offsets,
the position -> (pair, rating) mapping with its tail batch, the edge mask and the per-pair order with ties, NaN,
pairs without ratings and m larger than a pair's rating count."""
import numpy as np
import pytest

from igmc_b200 import recommend as rc


def _brute_positions(num_edges):
    """every (pair, rating) position in order"""
    return [(q, j) for q, n in enumerate(num_edges) for j in range(n)]


@pytest.mark.parametrize("num_edges", [[3, 0, 2, 0, 0, 5], [0, 4], [1], [0, 0, 2, 0]])
def test_offsets_and_positions_match_brute_force(num_edges):
    off = rc.explain_offsets_host(num_edges)
    assert off.dtype == np.int64 and off[0] == 0 and off[-1] == sum(num_edges)
    pos = _brute_positions(num_edges)
    T = len(pos)
    pu = np.arange(len(num_edges)) + 10
    pv = np.arange(len(num_edges)) * 3 + 1
    ni = 100
    for B in (1, 3, 4, T, T + 2):
        for start in range(0, T + B, B):
            got = rc.occlusion_pairs_host(off, pu, pv, ni, start, B)
            for i in range(B):
                c = start + i
                q, j = pos[min(c, T - 1)]
                assert tuple(got[:, i]) == (pu[q], pv[q], pu[q] * ni + pv[q], c if c < T else -1, j), (B, c)


def test_mask_drops_both_copies_of_one_rating():
    m = np.array([4, 0, 3, 1])
    edge_ptr = np.concatenate([[0], np.cumsum(2 * m)])
    tag = np.array([5, 7, -1, 9])
    j = np.array([2, 0, 1, 0])
    keep = rc.occlusion_mask_host(edge_ptr, tag, j)
    want = np.ones(edge_ptr[-1], np.uint8)
    for g in range(len(m)):
        if tag[g] < 0 or m[g] == 0:
            continue
        ei = np.arange(edge_ptr[g], edge_ptr[g + 1])
        # [u|v ; v|u]: the user->item copy of rating j at j, its item->user copy at m + j
        want[ei[j[g]]] = want[ei[m[g] + j[g]]] = 0
    assert np.array_equal(keep, want)
    assert int((keep == 0).sum()) == 2 * 2      # graph 1 has no ratings, graph 2 is padding


def _brute_order(delta, seg):
    """selection by repeated minimum under the explicit comparison: NaN last, |delta| descending, then j"""
    rest = list(seg)
    out = []

    def before(a, b):
        da, db = abs(float(delta[a])), abs(float(delta[b]))
        na, nb = np.isnan(da), np.isnan(db)
        if na or nb:
            return a < b if (na and nb) else nb
        return da > db or (da == db and a < b)
    while rest:
        best = rest[0]
        for x in rest[1:]:
            if before(x, best):
                best = x
        out.append(best)
        rest.remove(best)
    return out


@pytest.mark.parametrize("m", [None, 1, 3, 10])
def test_order_matches_brute_force(m):
    num_edges = [6, 0, 4, 1, 0, 7]
    off = rc.explain_offsets_host(num_edges)
    T, P = int(off[-1]), len(num_edges)
    score = np.array([1.0, 2.0, 3.5, -1.0, 0.0, 2.25], np.float32)
    q = np.repeat(np.arange(P), num_edges)
    rng = np.random.default_rng(1)
    d = rng.choice([0.5, -0.5, 0.25, 0.0, -0.0, 1.0, np.nan], T).astype(np.float32)   # ties, signed zeros, NaN
    occ = (score[q] + d).astype(np.float32)
    delta, order = rc.explain_order_host(score, occ, off, m)
    assert np.array_equal(delta, (occ - score[q]).astype(np.float32), equal_nan=True)
    want = [_brute_order(delta, range(off[p], off[p + 1])) for p in range(P)]
    if m is None:
        assert np.array_equal(order, np.concatenate(want))
    else:
        assert order.shape == (P, m)
        for p in range(P):
            n = min(m, num_edges[p])
            assert list(order[p, :n]) == want[p][:m]
            assert (order[p, n:] == -1).all()


def test_order_of_a_worked_example():
    num_edges = [5, 3]
    off = rc.explain_offsets_host(num_edges)
    score = np.array([1.0, 1.0], np.float32)
    occ = np.array([1.5, 0.5, 1.25, 0.75, 1.5, 1.0, np.nan, 0.0], np.float32)
    _, full = rc.explain_order_host(score, occ, off)
    # pair 0: |delta| 0.5 at positions 0, 1, 4 (a tie, by j), then 0.25 at 2 and 3 (a tie)
    # pair 1: |delta| 1 at 7, then 0 at 5, then NaN at 6
    assert list(full) == [0, 1, 4, 2, 3, 7, 5, 6]
    _, top = rc.explain_order_host(score, occ, off, 4)
    assert top.tolist() == [[0, 1, 4, 2], [7, 5, 6, -1]]
