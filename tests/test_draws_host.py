"""Monte-Carlo-dropout draws without a GPU: the numpy twins of igmc_draws_expand / igmc_draws_mask / igmc_draws_stats
(igmc_b200/recommend.py) on hand-built cases, the masks' independence of the batch position, their rates over 10^6
draws, and the argument checks of predict_draws and the draws= rankings that need no device."""
import math

import numpy as np
import pytest
from scipy import stats

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.models import IGMC

M64 = (1 << 64) - 1


def _scalar_splitmix(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def _state(seed, pid, s, side):
    """splitmix64(sample_state(seed, pid, side, 4) + s) in plain Python integers (csrc/common.cuh, csrc/draws.cu)"""
    tag = (pid * 16 + 4 * 2 + side) & M64
    return _scalar_splitmix((_scalar_splitmix(seed ^ _scalar_splitmix(tag)) + s) & M64)


def _pairs(G):
    u = np.arange(G, dtype=np.int32) * 3 + 1
    v = np.arange(G, dtype=np.int32) * 5 + 2
    return u, v, u.astype(np.int64) * 1000 + v, np.arange(G, dtype=np.int64) + 10


# ---- expand ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,B", [(3, 8), (1, 5), (5, 5), (8, 8), (4, 17), (7, 7)])
def test_expand_layout(S, B):
    """G = B // S pairs times S consecutive draws, pair major; the tail B - G*S copies pair 0 with tag -1, draw 0"""
    G = B // S
    pu, pv, pp, pt = _pairs(G)
    u, v, pid, tag, draw = rc.draws_expand_host(S, B, pu, pv, pp, pt)
    assert u.dtype == np.int32 and v.dtype == np.int32 and pid.dtype == np.int64 and tag.dtype == np.int64
    assert draw.dtype == np.int32
    for i in range(B):
        if i < G * S:
            g, s = divmod(i, S)
            assert (u[i], v[i], pid[i], tag[i], draw[i]) == (pu[g], pv[g], pp[g], pt[g], s)
        else:
            assert (u[i], v[i], pid[i], tag[i], draw[i]) == (pu[0], pv[0], pp[0], -1, 0)


def test_expand_keeps_a_tail_pair_tag():
    """a pair the pair stream marked as tail (tag -1) stays -1 in all its draws"""
    pu, pv, pp, pt = _pairs(3)
    pt[2] = -1
    tag = rc.draws_expand_host(2, 7, pu, pv, pp, pt)[3]
    assert tag.tolist() == [10, 10, 11, 11, -1, -1, -1]


# ---- masks --------------------------------------------------------------------------------------------------------------
def test_mask_follows_the_counter_hash():
    """edge_keep and hidden_keep in plain Python integers: the keys of draw s of pair pid are the high 32 bits of
    splitmix64(state + local index), kept at or above keep_thresh(p); padding keeps everything"""
    edge_ptr = np.array([0, 6, 6, 10, 14])          # graph 1 has no edges (a cold-start pair), graph 3 is padding
    pid = np.array([7, 123456789012, 7, 5], np.int64)
    tag = np.array([0, 1, 2, -1])
    draw = np.array([0, 3, 1, 0], np.int32)
    seed, p = 0xDEADBEEF12345678, 0.2
    ek, hk = rc.draws_mask_host(edge_ptr, pid, tag, draw, p, seed)
    assert ek.dtype == np.uint8 and ek.shape == (14,) and hk.shape == (4 * 128,)
    th_e, th_h = min(int(float(np.float32(p)) * 2 ** 32), M64), 2 ** 31
    for g in range(4):
        se, sh = _state(seed, int(pid[g]), int(draw[g]), 0), _state(seed, int(pid[g]), int(draw[g]), 1)
        for e in range(edge_ptr[g], edge_ptr[g + 1]):
            want = tag[g] < 0 or (_scalar_splitmix((se + int(e - edge_ptr[g])) & M64) >> 32) >= th_e
            assert ek[e] == want, (g, e)
        for o in range(128):
            want = tag[g] < 0 or (_scalar_splitmix((sh + o) & M64) >> 32) >= th_h
            assert hk[g * 128 + o] == want, (g, o)
    assert ek[10:].all() and hk[3 * 128:].all()


def test_mask_keys_do_not_depend_on_the_batch_position():
    """the same (pair, draw) at another position, in another batch, beside other graphs: the same masks"""
    rng = np.random.default_rng(0)
    n = rng.integers(0, 40, size=12) * 2
    edge_ptr = np.concatenate([[0], np.cumsum(n)])
    pid = rng.integers(0, 2 ** 40, size=12)
    draw = rng.integers(0, 8, size=12).astype(np.int32)
    tag = np.arange(12)
    ek, hk = rc.draws_mask_host(edge_ptr, pid, tag, draw, 0.3, 99)
    perm = rng.permutation(12)
    ek2, hk2 = rc.draws_mask_host(np.concatenate([[0], np.cumsum(n[perm])]), pid[perm], tag[perm], draw[perm], 0.3, 99)
    hk, hk2 = hk.reshape(12, 128), hk2.reshape(12, 128)
    for j, g in enumerate(perm):
        e2 = np.concatenate([[0], np.cumsum(n[perm])])
        assert np.array_equal(ek[edge_ptr[g]:edge_ptr[g + 1]], ek2[e2[j]:e2[j + 1]])
        assert np.array_equal(hk[g], hk2[j])
    # the streams differ by draw, by pair, by seed, and between edges and hidden units
    one = np.array([0, 128])
    a = rc.draws_mask_host(one, [5], [0], [0], 0.5, 1)
    for other in (rc.draws_mask_host(one, [5], [0], [1], 0.5, 1), rc.draws_mask_host(one, [6], [0], [0], 0.5, 1),
                  rc.draws_mask_host(one, [5], [0], [0], 0.5, 2)):
        assert not np.array_equal(a[0], other[0]) and not np.array_equal(a[1], other[1])
    assert not np.array_equal(a[0], a[1])


def test_mask_streams_do_not_share_a_tag_with_extraction_or_the_online_draw():
    """sample_state's tag pid * 16 + hop * 2 + side: the draws use hop 4, extraction hops 1..IGMC_MAX_HOP, the online
    trainer's draw hop 7"""
    assert rc.DRAWS_HOP_TAG not in range(1, _lib.MAX_HOP + 1) and rc.DRAWS_HOP_TAG != 7 and rc.DRAWS_HOP_TAG < 8


def test_mask_rates_over_a_million_draws():
    """dropped-edge rate within a chi-square bound of adj_dropout, hidden keep rate near 0.5, and the agreement of two
    draws' masks near p^2 + (1 - p)^2"""
    rng = np.random.default_rng(1)
    p = 0.2
    n, E = 4096, 256                                   # 4096 graphs of 256 directed edges: 1 048 576 edge draws
    edge_ptr = np.arange(n + 1) * E
    pid = rng.integers(0, 2 ** 40, size=n)
    tag = np.arange(n)
    ek0, hk0 = rc.draws_mask_host(edge_ptr, pid, tag, np.zeros(n, np.int32), p, 5)
    ek1, hk1 = rc.draws_mask_host(edge_ptr, pid, tag, np.ones(n, np.int32), p, 5)
    N = ek0.size
    for ek in (ek0, ek1):
        dropped = int(N - ek.sum())
        chi = (dropped - N * p) ** 2 / (N * p) + (N - dropped - N * (1 - p)) ** 2 / (N * (1 - p))
        assert chi < stats.chi2.ppf(0.999, 1), (dropped / N, chi)
    H = hk0.size                                       # 524 288 hidden draws per mask, two masks
    rate = (int(hk0.sum()) + int(hk1.sum())) / (2 * H)
    assert abs(rate - 0.5) < 4 * math.sqrt(0.25 / (2 * H)), rate
    agree = float((ek0 == ek1).mean())
    want = p * p + (1 - p) * (1 - p)
    assert abs(agree - want) < 4 * math.sqrt(want * (1 - want) / N), (agree, want)
    agree_h = float((hk0 == hk1).mean())
    assert abs(agree_h - 0.5) < 4 * math.sqrt(0.25 / H), agree_h


# ---- statistics ---------------------------------------------------------------------------------------------------------
def test_stats_by_hand():
    """fp64 in draw order, unbiased std, each rounded once; S = 1 has std 0; the tail is not a pair"""
    preds = np.array([1.0, 2.0, 4.0, 3.0, 3.0, 3.0, 9.0], np.float32)    # S = 3: G = 2, position 6 is padding
    x, mean, sd, key = rc.draws_stats_host(preds, 1, 7, 3, beta=2.0)
    assert x.shape == (2, 3) and np.array_equal(x[0], [1, 2, 4])
    assert mean[0] == np.float32(7 / 3) and sd[0] == np.float32(math.sqrt(((1 - 7 / 3) ** 2 + (2 - 7 / 3) ** 2 +
                                                                             (4 - 7 / 3) ** 2) / 2))
    assert key[0] == np.float32(7 / 3 + 2 * math.sqrt(((1 - 7 / 3) ** 2 + (2 - 7 / 3) ** 2 + (4 - 7 / 3) ** 2) / 2))
    assert mean[1] == 3 and sd[1] == 0 and key[1] == 3
    x, mean, sd, key = rc.draws_stats_host(np.array([5.0, -1.5], np.float32), 1, 2, 1, beta=-3.0)   # S = 1
    assert mean.tolist() == [5.0, -1.5] and sd.tolist() == [0.0, 0.0] and key.tolist() == [5.0, -1.5]
    x, mean, sd, key = rc.draws_stats_host(np.arange(6, dtype=np.float32), 1, 6, 6, beta=1.0)     # S = B, G = 1
    assert mean.tolist() == [2.5] and sd[0] == np.float32(math.sqrt(3.5))


def test_stats_checkpoint_mean_and_nan():
    """a draw is the fp32 checkpoint mean (sum in checkpoint order / K); a NaN draw makes mean, std and key NaN"""
    rng = np.random.default_rng(2)
    preds = rng.normal(size=(3, 8)).astype(np.float32)
    x = rc.draws_stats_host(preds, 3, 8, 4)[0]
    want = (((preds[0] + preds[1]).astype(np.float32) + preds[2]).astype(np.float32) / np.float32(3)).astype(np.float32)
    assert np.array_equal(x.reshape(-1), want)
    preds = np.array([1.0, np.nan, 2.0, 2.0, np.inf, 1.0], np.float32)
    _, mean, sd, key = rc.draws_stats_host(preds, 1, 6, 2, beta=0.5)
    assert np.isnan([mean[0], sd[0], key[0]]).all() and mean[1] == 2 and sd[1] == 0
    assert mean[2] == np.inf and np.isnan(sd[2]) and np.isnan(key[2])


def test_stats_are_fp64_not_fp32():
    """values whose fp32 sum loses bits: the mean is the fp64 one, rounded once"""
    preds = np.array([16777216.0, 1.0, 1.0, 1.0], np.float32)
    mean = rc.draws_stats_host(preds, 1, 4, 4)[1]
    assert mean[0] == np.float32(16777219.0 / 4)


# ---- argument checks ---------------------------------------------------------------------------------------------------
def test_draw_inputs():
    assert rc._draw_inputs(None, 0.0, 0, 256) is None
    assert rc._draw_inputs(8, -1.5, 2 ** 64 - 1, 256) == dict(S=8, beta=-1.5, draw_seed=2 ** 64 - 1)
    assert rc._draw_inputs(1, 0, np.uint64(3), 1)["S"] == 1
    assert rc._draw_inputs(_lib.DRAWS_MAX, 0, 0, 512)["S"] == _lib.DRAWS_MAX
    assert _lib.DRAWS_MAX >= 64
    for bad in (0, -1):
        with pytest.raises(ValueError):
            rc._draw_inputs(bad, 0.0, 0, 256)
    with pytest.raises(ValueError):
        rc._draw_inputs(9, 0.0, 0, 8)                  # more draws than a batch holds
    with pytest.raises(NotImplementedError):
        rc._draw_inputs(_lib.DRAWS_MAX + 1, 0.0, 0, 4096)
    for beta in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError):
            rc._draw_inputs(4, beta, 0, 256)
    with pytest.raises(ValueError):
        rc._draw_inputs(None, 1.0, 0, 256)             # beta ranks by draws
    for seed in (-1, 2 ** 64):
        with pytest.raises(ValueError):
            rc._draw_inputs(4, 0.0, seed, 256)
    with pytest.raises(TypeError):
        rc._draw_inputs(4, 0.0, 1.5, 256)


def _cpu_model():
    return IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True)


class _Shape(object):
    shape = (10, 12)


def test_public_entry_points_check_before_the_device():
    """the argument checks of predict_draws and the draws= rankings run before any device work"""
    m, g = _cpu_model(), _Shape()
    with pytest.raises(ValueError):
        rc.predict_draws(m, g, [0], [0], 0)
    with pytest.raises(ValueError):
        rc.predict_draws(m, g, [0], [0], 9, batch_size=8)
    with pytest.raises(NotImplementedError):
        rc.predict_draws(m, g, [0], [0], _lib.DRAWS_MAX + 1, batch_size=4096)
    with pytest.raises(ValueError):
        rc.predict_draws(m, g, [0], [0], 4, draw_seed=-1)
    with pytest.raises(IndexError):
        rc.predict_draws(m, g, [10], [0], 4)
    with pytest.raises(ValueError):
        rc.predict_draws(m, g, [0, 1], [0], 4)
    for fn, first in ((rc.recommend, [0]), (rc.recommend_users, [0])):
        with pytest.raises(ValueError):
            fn(m, g, first, 5, draws=0)
        with pytest.raises(ValueError):
            fn(m, g, first, 5, draws=4, beta=float("nan"))
        with pytest.raises(ValueError):
            fn(m, g, first, 5, beta=1.0)
        with pytest.raises(ValueError):
            fn(m, g, first, 5, draws=4, draw_seed=2 ** 64)
        with pytest.raises(NotImplementedError):
            fn(m, g, first, 5, draws=_lib.DRAWS_MAX + 1, batch_size=4096)
        with pytest.raises(ValueError):
            fn(m, g, first, 5, draws=16, batch_size=8)
    with pytest.raises(ValueError):
        rc.recommend_sessions(m, None, 5, draws=0)
    # no pairs: empty results of the documented shapes, on the model's device
    d = rc.predict_draws(m, g, [], [], 4)
    assert d.value.shape == (0, 4) and d.mean.shape == (0,) and d.std.shape == (0,)
    top_i, top_s = rc.recommend(m, g, [], 3, draws=4, beta=1.0)
    assert top_i.shape == (0, 3) and top_s.shape == (0, 3)
