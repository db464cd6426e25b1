"""Host twins of the node explanation kernels (igmc_b200/recommend.py, csrc/explain.cu) against brute force
(tests/node_stream_cases.py): the per-pair node count, the node occlusion mask with its records and the node gradient
scatter over checkpoints, on nodes with one rating and with many, an isolated node, h = 2 labels, a subgraph of only
its targets and graphs past one chunk of nodes; and the public functions' argument checks."""
import types

import numpy as np
import pytest
import torch

from igmc_b200 import recommend as rc
from tests import node_stream_cases as ns


@pytest.mark.parametrize("name", list(ns.SHAPES))
def test_count_matches_brute_force(name):
    shapes, h = ns.SHAPES[name]
    bt = ns.make_batch(3, shapes, h)
    B = len(shapes)
    tag = np.arange(B)[::-1].copy()
    tag[B // 2] = -1
    got = rc.node_count_host(bt["node_ptr"], tag, np.full(B, -5, np.int64))
    for g in range(B):
        if tag[g] >= 0:
            assert got[tag[g]] == len(ns.positions(bt, g)), (name, g)
    assert list(got).count(-5) == 1


@pytest.mark.parametrize("name", list(ns.SHAPES))
def test_mask_matches_brute_force(name):
    shapes, h = ns.SHAPES[name]
    bt = ns.make_batch(4, shapes, h)
    B = len(shapes)
    for jj in (0, 1, 255, 256, 299, 10 ** 6, -1):
        j = np.array([min(jj, max(len(ns.positions(bt, g)) - 1, 0)) if jj < 10 ** 6 else jj for g in range(B)])
        tag = np.arange(B) + 7
        tag[-1] = -1
        keep, rec = rc.node_occlusion_mask_host(bt["node_ptr"], bt["edge_ptr"], bt["src"], bt["dst"], bt["node_label"],
                                                bt["node_gid"], tag, j)
        want = np.ones(int(bt["edge_ptr"][-1]), np.uint8)
        for g in range(B):
            if tag[g] < 0:
                assert (rec[:, g] == -1).all()
                continue
            drop, r = ns.mask_brute(bt, g, int(j[g]))
            want[drop] = 0
            assert tuple(rec[:, g]) == (r if r is not None else (-1, -1, -1)), (name, jj, g)
            if r is not None:
                assert len(drop) == 2 * r[2]
        assert np.array_equal(keep, want), (name, jj)


@pytest.mark.parametrize("name", list(ns.SHAPES))
@pytest.mark.parametrize("K", [1, 3])
def test_grad_scatter_matches_brute_force(name, K):
    shapes, h = ns.SHAPES[name]
    bt = ns.make_batch(5, shapes, h)
    B = len(shapes)
    npos = np.array([len(ns.positions(bt, g)) for g in range(B)])
    order = np.random.default_rng(1).permutation(B)           # pair q of graph g: offsets follow the pairs, not g
    tag = order.copy()
    counts = np.zeros(B, np.int64)
    counts[tag] = npos
    off = rc.explain_offsets_host(counts)
    T = int(off[-1])
    rng = np.random.default_rng(2)
    grads = [rng.standard_normal(int(bt["edge_ptr"][-1])).astype(np.float32) for _ in range(K)]
    out = np.full(T, np.nan, np.float32)
    for k in range(K):
        rc.node_grad_scatter_host(bt["node_ptr"], bt["edge_ptr"], bt["node_label"], bt["in_ptr"], bt["in_eid"], tag,
                                  grads[k], off, out, k, K)
    want = np.full(T, np.nan, np.float32)
    for g in range(B):
        o = int(off[tag[g]])
        acc = None
        for k in range(K):
            v, _ = ns.grad_brute(bt, g, grads[k])
            acc = v if k == 0 else (acc + v).astype(np.float32)
        if K > 1:
            acc = (acc / np.float32(K)).astype(np.float32)
        want[o:o + npos[g]] = acc
    assert np.array_equal(out.view(np.int32), want.view(np.int32)), name


def test_argument_checks():
    with pytest.raises(ValueError):
        rc._check_top(0)
    with pytest.raises(NotImplementedError):
        rc._check_top(257)
    assert rc._check_top(None) is None and rc._check_top(256) == 256
    assert set(rc.__all__) >= {"explain_nodes", "NodeExplanation", "attribute_nodes", "NodeAttribution"}
    assert rc.NodeExplanation._fields == ("score", "num_nodes", "offsets", "node", "label", "ratings", "delta")
    assert rc.NodeAttribution._fields == ("score", "num_nodes", "offsets", "node", "label", "ratings", "grad")
    model = types.SimpleNamespace(flat_params=torch.zeros(1))
    graph = types.SimpleNamespace(shape=(5, 7))
    for fn, cls in ((rc.explain_nodes, rc.NodeExplanation), (rc.attribute_nodes, rc.NodeAttribution)):
        with pytest.raises(NotImplementedError):
            fn(model, graph, [0], [0], 257)
        with pytest.raises(ValueError):
            fn(model, graph, [0], [0], 0)
        with pytest.raises(ValueError):
            fn(model, graph, [0, 1], [0])
        with pytest.raises(IndexError):
            fn(model, graph, [5], [0])
        r = fn(model, graph, [], [])          # no pairs: the empty result, nothing launched
        assert isinstance(r, cls) and r.score.shape == (0,) and r.offsets.tolist() == [0] and r[-1].shape == (0,)
        r = fn(model, graph, [], [], 4)
        assert r.node.shape == (0, 4) and r.ratings.shape == (0, 4)
