"""Per-pair gradients and influence without a GPU (igmc_b200/recommend.py pair_gradients / influence / self_influence).

* the per-pair loss l_i = (f_i - y_i)^2 in fp64 on the restated models (oracle/pyg_restated.py, tests/pyg2_oracle.py):
  its gradients summed over a batch, divided by B, plus the ARR gradient, are the batch training gradient;
* the readout block's factor form equals the materialised dot product;
* the numpy twins of the proponent / opponent order and of the streaming merge against a brute-force sort;
* argument validation before anything launches."""
import functools

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from oracle import pyg_restated
from tests import pyg2_oracle


def _graph(rng, nu, ni, R, F=4):
    """one random enclosing subgraph: target user 0, target item nu, users / items otherwise; [u|v ; v|u] edges"""
    n = nu + ni
    x = torch.zeros(n, F, dtype=torch.float64)
    x[0, 0] = x[nu, 1] = 1
    x[1:nu, 2] = 1
    x[nu + 1:, 3] = 1
    m = int(rng.integers(0, nu * ni))
    pairs = rng.choice(nu * ni, m, replace=False)
    pairs = pairs[pairs != 0]                               # the target pair's own rating is not in its subgraph
    src, dst = pairs // ni, nu + pairs % ni
    et = rng.integers(0, R, len(pairs))
    ei = torch.from_numpy(np.stack([np.concatenate([src, dst]), np.concatenate([dst, src])])).long()
    return x, ei, torch.from_numpy(np.concatenate([et, et])).long()


def _batch(graphs):
    xs, eis, ets, off = [], [], [], 0
    for x, ei, et in graphs:
        xs.append(x)
        eis.append(ei + off)
        ets.append(et)
        off += x.shape[0]
    return torch.cat(xs), torch.cat(eis, 1), torch.cat(ets)


def _flat_grad(model, loss):
    ps = list(model.parameters())
    gs = torch.autograd.grad(loss, ps, allow_unused=True)
    return torch.cat([(torch.zeros_like(p) if g is None else g).reshape(-1) for p, g in zip(ps, gs)])


@pytest.mark.parametrize("rgcn", ["pyg-1.4", "pyg-2"])
@pytest.mark.parametrize("mb", [1, 2])
def test_per_pair_gradients_sum_to_the_batch_gradient(rgcn, mb):
    torch.manual_seed(3)
    rng = np.random.default_rng(4)
    R, B, ARR = 5, 6, 0.001
    ref = pyg2_oracle.igmc_ref(rgcn, 4, (32,) * 4, R, 4, 0.0, mb).double().eval()
    graphs = [_graph(rng, int(rng.integers(1, 5)), int(rng.integers(1, 5)), R) for _ in range(B)]
    graphs[2] = (graphs[2][0], graphs[2][1][:, :0], graphs[2][2][:0])     # a subgraph without ratings
    y = torch.from_numpy(rng.integers(1, R + 1, B).astype(np.float64))
    per_pair = []
    for (x, ei, et), yi in zip(graphs, y):
        f = ref(x, ei, et)
        per_pair.append(_flat_grad(ref, ((f - yi) ** 2).sum()))
    x, ei, et = _batch(graphs)
    loss, _ = pyg_restated.train_loss(ref, dict(x=x, edge_index=ei, edge_type=et, y=y), ARR=ARR)
    want = _flat_grad(ref, loss)
    arr = _flat_grad(ref, ARR * pyg_restated.arr_regulariser(ref))
    got = torch.stack(per_pair).sum(0) / B + arr
    assert float((got - want).abs().max()) <= 1e-10 * max(float(want.abs().max()), 1.0)


def test_readout_factor_form_equals_the_materialised_dot():
    rng = np.random.default_rng(1)
    H, L = _lib.LIN1_OUT, 4
    F = 2 * 32 * L
    fac = [rng.standard_normal(2 * H + F + 1) for _ in range(2)]

    def materialise(f):
        dhid, feat, hid, dp = f[:H], f[H:H + F], f[H + F:2 * H + F], f[2 * H + F]
        return np.concatenate([np.outer(dhid, feat).reshape(-1), dhid, dp * hid, [dp]])
    a, b = materialise(fac[0]), materialise(fac[1])
    want = float(np.dot(a, b))
    assert abs(rc.readout_dot_host(fac[0], fac[1], F) - want) <= 1e-12 * abs(want) + 1e-12
    # and the self term is ||G||^2
    assert abs(rc.readout_dot_host(fac[0], fac[0], F) - float(np.dot(a, a))) <= 1e-12 * float(np.dot(a, a))


def _brute(values, k):
    """proponents: value descending, index ascending, NaN last; opponents: value ascending, same rules"""
    def cmp(sign):
        def c(i, j):
            a, b = values[i], values[j]
            an, bn = np.isnan(a), np.isnan(b)
            if an or bn:
                return (i - j) if (an and bn) else (1 if an else -1)
            a, b = sign * a, sign * b
            return -1 if a > b else 1 if a < b else i - j
        return functools.cmp_to_key(c)
    out = []
    for sign, pad in ((1, -np.inf), (-1, np.inf)):
        o = sorted(range(len(values)), key=cmp(sign))[:k]
        idx = np.full(k, -1, np.int64)
        val = np.full(k, pad, np.float32)
        idx[:len(o)] = o
        val[:len(o)] = np.asarray(values, np.float32)[o]
        out += [idx, val]
    return out


def _cases():
    rng = np.random.default_rng(7)
    v = rng.integers(-3, 4, 40).astype(np.float32)           # many ties
    v[[3, 17, 29]] = np.nan
    v[5], v[6] = 0.0, -0.0
    yield v, 10
    yield v, 64                                                # N < k: padding
    yield rng.standard_normal(300).astype(np.float32), 256
    yield np.full(5, np.nan, np.float32), 3
    yield np.zeros(0, np.float32), 4


def test_order_twin_matches_brute_force():
    for v, k in _cases():
        got = rc.influence_order_host(v, k)
        want = _brute(v, k)
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g, w)


@pytest.mark.parametrize("batch", [1, 7, 50])
def test_streaming_merge_equals_the_whole_run(batch):
    for v, k in _cases():
        n = len(v)
        pro = (np.full(k, -np.inf, np.float32), np.full(k, -1, np.int64))
        con = (np.full(k, np.inf, np.float32), np.full(k, -1, np.int64))
        for b0 in range(0, max(n, 1), batch):
            seg_i = np.arange(b0, b0 + batch)
            seg_v = np.zeros(batch, np.float32)
            real = seg_i < n
            seg_v[real] = v[seg_i[real]]
            seg_i = np.where(real, seg_i, -1)                      # the padded tail
            pro = rc.influence_merge_host(pro[0], pro[1], seg_v, seg_i, 1.0)
            con = rc.influence_merge_host(con[0], con[1], seg_v, seg_i, -1.0)
        pi, pv, ci, cv = rc.influence_order_host(v, k)
        np.testing.assert_array_equal(pro[1], pi)
        np.testing.assert_array_equal(pro[0], pv)
        np.testing.assert_array_equal(con[1], ci)
        np.testing.assert_array_equal(con[0], cv)


def test_accumulation_twin():
    """S = sum_k eta_k (<conv_b, conv_t> + readout factor form) equals the dot of the materialised gradients"""
    rng = np.random.default_rng(2)
    H, L, PC = _lib.LIN1_OUT, 2, 37
    F = 2 * 32 * L
    eta = [0.5, -1.0, 2.0]
    S = 0.0
    want = 0.0
    for e in eta:
        cb, ct = rng.standard_normal(PC), rng.standard_normal(PC)
        fb, ft = rng.standard_normal(2 * H + F + 1), rng.standard_normal(2 * H + F + 1)
        S += e * (float(np.dot(cb, ct)) + rc.readout_dot_host(fb, ft, F))

        def full(c, f):
            return np.concatenate([c, np.outer(f[:H], f[H:H + F]).reshape(-1), f[:H], f[2 * H + F] * f[H + F:2 * H + F],
                                   [f[2 * H + F]]])
        want += e * float(np.dot(full(cb, fb), full(ct, ft)))
    assert abs(S - want) <= 1e-10 * abs(want)


def _cpu_model(dgcnn=False):
    from igmc_b200.models import DGCNN_RS, IGMC
    if dgcnn:
        return DGCNN_RS(4, latent_dim=[32, 32, 32, 1], k=30, num_relations=5, num_bases=4, regression=True)
    return IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True)


def test_arguments_are_checked_before_anything_launches():
    import scipy.sparse as ssp
    A = ssp.csr_matrix(np.eye(6, 5, dtype=np.float32))
    m = _cpu_model()
    u, v, y = np.array([0, 1]), np.array([0, 1]), np.array([4.0, 5.0])
    with pytest.raises(IndexError):
        rc.pair_gradients(m, A, [0, 6], [0, 1])
    with pytest.raises(IndexError):
        rc.influence(m, A, (u, np.array([0, 5]), y), (u, v), 3)
    with pytest.raises(ValueError):
        rc.pair_gradients(m, A, [0, 1], [0])
    with pytest.raises(ValueError):
        rc.pair_gradients(m, A, u, v, [1.0])
    with pytest.raises(ValueError):
        rc.influence(m, A, (u, v, [1.0, np.nan]), (u, v), 3)
    with pytest.raises(ValueError):
        rc.self_influence(m, A, (u, v, [np.inf, 1.0]))
    with pytest.raises(ValueError):
        rc.influence(m, A, (u, v), (u, v), 3)                    # training pairs need their targets
    with pytest.raises(ValueError):
        rc.influence(m, A, (u, v, y), (u, v), 3, lrs=[1.0, 2.0])  # one eta per checkpoint (K = 1 here)
    with pytest.raises(ValueError):
        rc.influence(m, A, (u, v, y), (u, v), 0)
    with pytest.raises(NotImplementedError):
        rc.influence(m, A, (u, v, y), (u, v), _lib.TOPK_MAX + 1)
    big = np.zeros(rc.INFLUENCE_T_MAX + 1, np.int64)
    with pytest.raises(NotImplementedError):
        rc.influence(m, A, (u, v, y), (big, big), 3)
    d = _cpu_model(dgcnn=True)
    for call in (lambda: rc.pair_gradients(d, A, u, v), lambda: rc.influence(d, A, (u, v, y), (u, v), 3),
                 lambda: rc.self_influence(d, A, (u, v, y))):
        with pytest.raises(NotImplementedError):
            call()
