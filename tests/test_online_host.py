"""The online trainer's pair draw without a GPU: the numpy twins of igmc_online_draw / igmc_online_recent_append
(igmc_b200/train_eval.py) on hand-built graphs, the draw's distribution, the argument checks of the two entry points
and of OnlineTrainer that need no device."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as ssp
import torch
from scipy import stats

from igmc_b200 import _lib
from igmc_b200.train_eval import (_draw_keys, online_draw_host, recent_append_host, recent_threshold,
                                  _splitmix64_np, OnlineTrainer)

M64 = (1 << 64) - 1


def _graph(rows, num_items):
    """host CSR arrays of {user: {item: label}}"""
    nu = max(rows) + 1 if rows else 0
    u, v, x = [], [], []
    for a, r in rows.items():
        for b, lab in r.items():
            u.append(a), v.append(b), x.append(lab + 1)
    A = ssp.csr_matrix((np.array(x, np.float32), (u, v)), shape=(nu, num_items))
    A.sort_indices()
    return A.indptr.astype(np.int64), A.indices.astype(np.int64), (A.data - 1).astype(np.uint8)


def _ring(cap, pairs=()):
    ru, rv, tot = np.zeros(cap, np.int32), np.zeros(cap, np.int32), 0
    if pairs:
        u, v = zip(*pairs)
        ru, rv, tot = recent_append_host(ru, rv, 0, u, v, np.ones(len(u), np.int64))
    return ru, rv, tot


def _draw(g, ni, ring, frac, step=3, B=64, seed=11, drop=0x1234ABCD):
    return online_draw_host(*g, ni, ring[0], ring[1], ring[2], recent_threshold(frac), step, seed, drop, B)


def _scalar_splitmix(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


# a graph with empty rows (users 0, 2, 5) and several row lengths
ROWS = {1: {0: 0, 3: 4, 7: 2}, 3: {2: 1}, 4: {0: 3, 1: 1, 5: 0, 6: 4, 8: 2}, 6: {4: 3}}
NI = 9


def test_keys_and_seeds_follow_the_counter_hash():
    """seeds and keys in plain Python integers: seeds[0] = splitmix64(sample_seed + s), the dropout seeds of steps s
    and s + 1, key = sample_state(seed, j, round, 7) of csrc/common.cuh"""
    g = _graph(ROWS, NI)
    s, ss, ds = 5, 99, 0x1234ABCD
    *_, seeds, _ = online_draw_host(*g, NI, *_ring(4), recent_threshold(0), s, ss, ds, 8)
    assert [int(a) for a in seeds] == [_scalar_splitmix(ss + s), _scalar_splitmix(ds + s), _scalar_splitmix(ds + s + 1)]
    seed = int(seeds[0])
    for rnd in (0, 1):
        want = [_scalar_splitmix(seed ^ _scalar_splitmix(j * 16 + 14 + rnd)) for j in range(8)]
        assert [int(k) for k in _draw_keys(seed, 8, rnd)] == want
    assert int(_splitmix64_np(np.uint64(M64))) == _scalar_splitmix(M64)


def test_uniform_position_is_the_high_word_of_h_times_nnz():
    """one user rating items 0..nnz-1: the uniform draw's item is floor(h * nnz / 2^64) in plain integers"""
    for nnz in (1, 2, 7, 1000, 65537):
        g = (np.array([0, nnz]), np.arange(nnz), np.zeros(nnz, np.uint8))
        u, v, *_, seeds, _ = online_draw_host(*g, nnz, *_ring(4), 0, 9, 4, 0, 300)
        h = _draw_keys(int(seeds[0]), 300, 1)
        assert (u == 0).all() and v.tolist() == [(int(x) * nnz) >> 64 for x in h], nnz


@pytest.mark.parametrize("frac", [0.0, 0.3, 1.0])
def test_draws_are_ratings_of_the_graph(frac):
    g = _graph(ROWS, NI)
    ring = _ring(8, [(1, 3), (4, 6), (3, 2)])
    u, v, lab, pid, _, win = _draw(g, NI, ring, frac, B=400)
    for j in range(400):
        assert v[j] in ROWS[u[j]] and lab[j] == ROWS[u[j]][v[j]]
        assert pid[j] == u[j] * NI + v[j]
    if frac == 0.0:
        assert not win.any()
    elif frac == 1.0:
        assert win.all()
        assert set(zip(u.tolist(), v.tolist())) <= {(1, 3), (4, 6), (3, 2)}
    else:
        assert 0 < win.sum() < 400


def test_window_labels_are_read_from_the_graph_at_draw_time():
    """a window pair whose rating changed is drawn with the new label; a deleted one falls through to the uniform
    draw, which is the draw a zero fraction gives in that slot"""
    ring = _ring(4, [(1, 3), (4, 6)])
    changed = {a: dict(r) for a, r in ROWS.items()}
    changed[1][3] = 0
    u, v, lab, _, _, win = _draw(_graph(changed, NI), NI, ring, 1.0, B=200)
    assert win.all() and all(lab[j] == changed[u[j]][v[j]] for j in range(200))
    gone = {a: dict(r) for a, r in ROWS.items()}
    del gone[1][3]
    g = _graph(gone, NI)
    u, v, lab, _, _, win = _draw(g, NI, ring, 1.0, B=200)
    u0, v0, lab0, _, _, _ = _draw(g, NI, ring, 0.0, B=200)
    fell = ~win
    assert fell.any() and win.any()
    assert set(zip(u[win].tolist(), v[win].tolist())) == {(4, 6)}
    assert np.array_equal(u[fell], u0[fell]) and np.array_equal(v[fell], v0[fell]) and np.array_equal(lab[fell], lab0[fell])
    # a window entry beyond the graph's shape (ids are only ever valid ones; still never read out of bounds)
    u, v, _, _, _, win = _draw(g, NI, _ring(2, [(50, 2), (1, 70)]), 1.0, B=50)
    assert not win.any()


def test_empty_window_and_a_single_rating():
    g = _graph(ROWS, NI)
    a = _draw(g, NI, _ring(16), 1.0, B=100)
    b = _draw(g, NI, _ring(16), 0.0, B=100)
    assert not a[5].any() and all(np.array_equal(x, y) for x, y in zip(a[:4], b[:4]))
    one = _graph({2: {5: 3}}, 7)
    u, v, lab, pid, _, _ = _draw(one, 7, _ring(4), 0.5, B=64)
    assert (u == 2).all() and (v == 5).all() and (lab == 3).all() and (pid == 2 * 7 + 5).all()


def test_ring_wraps_around_keeping_the_newest():
    cap = 4
    ru, rv, tot = np.full(cap, -1, np.int32), np.full(cap, -1, np.int32), 0
    ru, rv, tot = recent_append_host(ru, rv, tot, [1, 2, 3], [10, 20, 30], [1, 0, 5])        # value 0: not appended
    assert tot == 2 and list(ru) == [1, 3, -1, -1] and list(rv) == [10, 30, -1, -1]
    ru, rv, tot = recent_append_host(ru, rv, tot, [4, 5, 6], [40, 50, 60], [2, 2, 2])
    assert tot == 5 and list(ru) == [6, 3, 4, 5] and list(rv) == [60, 30, 40, 50]
    # more than the capacity in one call: the last `cap` of the call, each at (total + rank) % cap
    ru, rv, tot = recent_append_host(ru, rv, tot, np.arange(100, 110), np.arange(10), np.ones(10, np.int64))
    assert tot == 15
    assert sorted(ru.tolist()) == [106, 107, 108, 109]
    assert all(ru[(5 + r) % cap] == 100 + r for r in range(6, 10))
    # the draw reads the current window only: min(total, capacity) entries
    g = _graph({0: {0: 1}, 1: {1: 2}, 2: {2: 3}}, 3)
    ru, rv, tot = recent_append_host(np.zeros(8, np.int32), np.zeros(8, np.int32), 0, [2], [2], [4])
    u, v, *_ = online_draw_host(*g, 3, ru, rv, tot, recent_threshold(1.0), 0, 1, 2, 64)
    assert (u == 2).all() and (v == 2).all()


def test_empty_rows_are_never_drawn():
    g = _graph(ROWS, NI)
    seen = set()
    for step in range(50):
        u, *_ = _draw(g, NI, _ring(4), 0.0, step=step, B=256)
        seen |= set(u.tolist())
    assert seen == {1, 3, 4, 6}


def test_draw_distribution():
    """10^6 uniform draws: every rating position equally likely (chi-square); with a window, the share of window draws
    is recent_fraction (binomial, 5 sigma)"""
    rng = np.random.default_rng(3)
    rows = {}
    for a in range(40):
        k = int(rng.integers(0, 6))
        if k:
            rows[a] = {int(b): int(rng.integers(0, 5)) for b in rng.choice(30, k, replace=False)}
    g = _graph(rows, 30)
    nnz = int(g[0][-1])
    key = {(a, b): i for i, (a, b) in enumerate((a, b) for a in sorted(rows) for b in sorted(rows[a]))}
    counts = np.zeros(nnz, np.int64)
    B, n = 10000, 100
    for step in range(n):
        u, v, *_ = _draw(g, 30, _ring(4), 0.0, step=step, B=B, seed=5)
        np.add.at(counts, [key[(a, b)] for a, b in zip(u.tolist(), v.tolist())], 1)
    assert stats.chisquare(counts).pvalue > 1e-4
    ring = _ring(64, [(a, b) for a, b in list(key)[:20]])
    frac, total = 0.37, 0
    for step in range(n):
        total += int(_draw(g, 30, ring, frac, step=step, B=B, seed=6)[5].sum())
    N = B * n
    assert abs(total - frac * N) < 5 * np.sqrt(N * frac * (1 - frac)), total / N


def test_entry_point_argument_checks():
    """refused before any launch (no device needed)"""
    lib = _lib.load()
    csr = _lib.CSR(8, 8, 8, 8, 8, 3, 3)

    def draw(G=ctypes.byref(csr), cap=4, thresh=0, step=8, ahead=1, B=4, ring=8):
        return lib.igmc_online_draw(G, ring, ring, cap, 8, thresh, step, ahead, 0, 0, B, 8, 8, 8, 8, 8, 8, None)
    assert draw(G=None) == -1
    assert draw(cap=0) == -2 and draw(ring=None) == -2
    assert draw(thresh=-1) == -3 and draw(thresh=(1 << 32) + 1) == -3
    assert draw(step=None) == -4 and draw(ahead=-1) == -4
    assert draw(B=0) == -5
    assert lib.igmc_online_recent_append(8, 8, 8, -1, 8, 8, 4, 8, 8, None) == -1
    assert lib.igmc_online_recent_append(None, 8, 8, 3, 8, 8, 4, 8, 8, None) == -1
    assert lib.igmc_online_recent_append(8, 8, 8, 3, 8, 8, 0, 8, 8, None) == -2
    assert lib.igmc_online_recent_append(None, None, None, 0, 8, 8, 4, 8, 8, None) == 0     # nothing to append


def test_thresholds():
    assert recent_threshold(0) == 0 and recent_threshold(1) == 1 << 32 and recent_threshold(0.5) == 1 << 31


def test_trainer_refuses_a_model_off_cuda():
    from igmc_b200.models import FusedAdam, IGMC
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        OnlineTrainer(m, None, FusedAdam(m), batch_size=8)
    assert m.flat_params.device == torch.device("cpu")
