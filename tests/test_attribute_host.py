"""The definition behind attribute_pairs, on the CPU in fp64 (tests/edge_weight_oracle.py), and the host twins of its
scatter and order.

* the weighted restatement at w = 1 is the restated model, and at a 0/1 w it is dropout_adj with that draw, for IGMC
  and DGCNN_RS with both RGCN layers;
* the closed form the kernel evaluates (per edge, (s - segment mean) / |segment|, summed over layers) equals autograd
  d score / d w within 1e-10, with R = 1, single-edge segments, zero-edge subgraphs and h = 2;
* igmc_edge_grad_scatter's and igmc_occlusion_order's twins give the brute-force per-pair lists."""
import numpy as np
import pytest
import torch

from igmc_b200 import recommend as rc
from oracle import pyg_restated
from tests import edge_weight_oracle as ewo
from tests import pyg2_oracle


def _subgraph(rng, n_users, n_items, n_ratings, R, h):
    """one [u|v ; v|u] subgraph: node 0 the target user, node n_users the target item, the other nodes labelled by a
    hop in [1, h]; the first user rates only one item (a single-edge segment); the target pair is not rated"""
    n = n_users + n_items
    lab = np.zeros(n, np.int64)
    lab[1:n_users] = 2 * rng.integers(1, h + 1, n_users - 1)
    lab[n_users] = 1
    lab[n_users + 1:] = 2 * rng.integers(1, h + 1, n_items - 1) + 1
    pairs = set()
    if n_users > 1 and n_items > 1:
        pairs.add((1, n_users + 1))
    while len(pairs) < n_ratings:
        u, i = int(rng.integers(0, n_users)), n_users + int(rng.integers(0, n_items))
        if (u, i) != (0, n_users) and not (u == 1 and i != n_users + 1):
            pairs.add((u, i))
    pairs = sorted(pairs)
    u = np.array([p[0] for p in pairs], np.int64)
    i = np.array([p[1] for p in pairs], np.int64)
    t = rng.integers(0, R, len(pairs))
    x = np.zeros((n, 2 * h + 2))
    x[np.arange(n), lab] = 1.0
    return x, np.stack([np.concatenate([u, i]), np.concatenate([i, u])]), np.concatenate([t, t])


def _batch(seed, R, h, sizes=((6, 5, 12), (1, 1, 0), (10, 10, 80), (3, 3, 1))):
    """a batch of subgraphs (n_users, n_items, ratings); (1, 1, 0) has no edges"""
    rng = np.random.default_rng(seed)
    xs, eis, ets, bs, off = [], [], [], [], 0
    for g, (nu, ni, m) in enumerate(sizes):
        x, ei, et = _subgraph(rng, nu, ni, m, R, h)
        xs.append(x)
        eis.append(ei + off)
        ets.append(et)
        bs.append(np.full(len(x), g))
        off += len(x)
    cat = lambda a: torch.from_numpy(np.concatenate(a, -1))
    return (torch.from_numpy(np.concatenate(xs)), cat(eis), cat(ets), torch.from_numpy(np.concatenate(bs)),
            len(sizes))


def _ref(kind, rgcn, R, h, seed=0):
    torch.manual_seed(seed)
    F = 2 * h + 2
    if kind == "igmc":
        ref = pyg2_oracle.igmc_ref(rgcn, F, (32,) * 4, R, 4, 0.0)
    else:
        ref = pyg2_oracle.dgcnn_rs_ref(rgcn, F, (32, 32, 32, 1), 10, R, 4, 0.0)
    with torch.no_grad():
        for c in ref.convs:
            c.bias.uniform_(-0.3, 0.3)
    return ref.double().eval()


def _plain(ref, x, ei, et, b, B):
    if isinstance(ref, pyg_restated.DGCNN_RSRef):
        return ref(x, ei, et, b, num_graphs=B)
    return ref(x, ei, et)


def _kw(ref, b, B):
    return dict(batch=b, num_graphs=B) if isinstance(ref, pyg_restated.DGCNN_RSRef) else {}


MODELS = [(k, r) for k in ("igmc", "dgcnn_rs") for r in ("pyg-1.4", "pyg-2")]


@pytest.mark.parametrize("kind,rgcn", MODELS)
def test_unit_weights_are_the_model_and_masks_are_dropout_adj(kind, rgcn):
    R, h = 5, 1
    ref = _ref(kind, rgcn, R, h)
    x, ei, et, b, B = _batch(1, R, h)
    kw = _kw(ref, b, B)
    with torch.no_grad():
        ones = torch.ones(ei.shape[1], dtype=torch.float64)
        want = _plain(ref, x, ei, et, b, B)
        assert torch.allclose(ewo.weighted_forward(ref, x, ei, et, ones, **kw), want, rtol=0, atol=1e-12)
        keep = torch.from_numpy(np.random.default_rng(2).random(ei.shape[1]) > 0.4)
        eif, etf = pyg_restated.dropout_adj(ei, et, 0.4, True, keep)
        want = _plain(ref, x, eif, etf, b, B)
        got = ewo.weighted_forward(ref, x, ei, et, keep.double(), **kw)
        assert torch.allclose(got, want, rtol=0, atol=1e-12)


@pytest.mark.parametrize("kind,rgcn", MODELS)
@pytest.mark.parametrize("R,h", [(1, 1), (5, 1), (13, 2)])
def test_centred_formula_is_the_autograd_gradient(kind, rgcn, R, h):
    ref = _ref(kind, rgcn, R, h, seed=R)
    x, ei, et, b, B = _batch(10 + R, R, h)
    kw = _kw(ref, b, B)
    auto = ewo.autograd_edge_grad(ref, x, ei, et, **kw)
    closed = ewo.centred_edge_grad(ref, x, ei, et, **kw)
    assert float(auto.abs().max()) > 1e-6
    assert float((auto - closed).abs().max()) <= 1e-10
    # the single-edge segments of the batch add nothing: user 1 of every subgraph rates one item
    dst = ei[1]
    cnt = torch.bincount(dst, minlength=x.shape[0])
    assert (cnt[dst] == 1).any()


def test_scatter_and_order_twins_against_brute_force():
    rng = np.random.default_rng(3)
    m_per_graph = np.array([3, 0, 5, 2, 4])
    edge_ptr = np.concatenate([[0], np.cumsum(2 * m_per_graph)])
    tag = np.array([2, 0, 1, -1, 3])            # graph 3 is padding
    P = 4
    counts = np.zeros(P, np.int64)
    for g, q in enumerate(tag):
        if q >= 0:
            counts[q] = m_per_graph[g]
    offsets = rc.explain_offsets_host(counts)
    K = 3
    grads = [rng.standard_normal(edge_ptr[-1]).astype(np.float32) for _ in range(K)]
    grads[0][edge_ptr[2]] = np.nan
    grads[1][edge_ptr[4]:edge_ptr[4] + 2] = 0.0        # a tie of two zeros in one pair
    grads[2][edge_ptr[4]:edge_ptr[4] + 2] = 0.0
    grads[0][edge_ptr[4]:edge_ptr[4] + 2] = 0.0
    out = np.zeros(int(offsets[-1]), np.float32)
    for k in range(K):
        rc.edge_grad_scatter_host(edge_ptr, tag, grads[k], offsets, out, k, K)
    val, order = rc.explain_order_host(None, out, offsets)
    for g, q in enumerate(tag):
        if q < 0:
            continue
        m, e0 = int(m_per_graph[g]), int(edge_ptr[g])
        want = np.zeros(m, np.float32)
        for k in range(K):
            want = want + (grads[k][e0:e0 + m] + grads[k][e0 + m:e0 + 2 * m])
        want = want / np.float32(K)
        o = int(offsets[q])
        assert np.array_equal(out[o:o + m], want, equal_nan=True)
        brute = sorted(range(m), key=lambda j: (np.isnan(want[j]), -abs(want[j]) if not np.isnan(want[j]) else 0, j))
        assert np.array_equal(order[o:o + m] - o, brute), (q, order[o:o + m] - o, brute)
    _, top = rc.explain_order_host(None, out, offsets, m=2)
    for q in range(P):
        n = min(2, int(counts[q]))
        assert np.array_equal(top[q, :n], order[offsets[q]:offsets[q] + n]) and (top[q, n:] == -1).all()
