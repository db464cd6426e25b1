"""The PyG >= 1.6 RGCNConv (mean per relation) without a GPU: the oracle's ``mean_per_relation`` against naive
per-node, per-relation loops (forward and fp64 autograd gradients), the ``rgcn="pyg-2"`` model surface (names, shapes,
init, state_dict keys, refused checkpoints) and the kernel plans of the new mode."""
import math

import pytest
import torch

from oracle import pyg_restated
from tests import pyg2_oracle


def _graph(n, R, E, seed, zero_nodes=(), missing=None):
    """random directed multigraph on n nodes: no in-edge at ``zero_nodes``; node ``missing[0]`` gets no in-edge of the
    relations in ``missing[1]``; node 1 has in-edges of relation 0 only"""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (E,), generator=g)
    dst = torch.randint(0, n, (E,), generator=g)
    ty = torch.randint(0, R, (E,), generator=g)
    ok = torch.ones(E, dtype=torch.bool)
    for z in zero_nodes:
        ok &= dst != z
    if missing is not None:
        v, rels = missing
        for r in rels:
            ok &= ~((dst == v) & (ty == r))
    ty = torch.where(dst == 1, torch.zeros_like(ty), ty)
    return torch.stack([src[ok], dst[ok]]), ty[ok]


def _naive(conv, x, ei, et):
    """x'_i = x_i root + bias + sum_r 1/|N_r(i)| sum_{j in N_r(i)} x_j W_r, one node and one relation at a time"""
    R = conv.num_relations
    att, basis = (conv.comp, conv.weight) if hasattr(conv, "comp") else (conv.att, conv.basis)
    W = [sum(att[r, b] * basis[b] for b in range(conv.num_bases)) for r in range(R)]
    rows = []
    for i in range(x.shape[0]):
        o = x[i] @ conv.root + conv.bias
        for r in range(R):
            js = [int(ei[0, e]) for e in range(ei.shape[1]) if int(ei[1, e]) == i and int(et[e]) == r]
            if js:
                o = o + sum(x[j] @ W[r] for j in js) / len(js)
        rows.append(o)
    return torch.stack(rows)


@pytest.mark.parametrize("formulation", ["bmm", "transform"])
@pytest.mark.parametrize("layer", ["pyg-1.4", "pyg-2"])
def test_mean_per_relation_matches_naive_loops(formulation, layer):
    torch.manual_seed(0)
    n, R, IN, OUT = 23, 5, 6, 7
    ei, et = _graph(n, R, 140, 1, zero_nodes=(3, 17), missing=(5, (1, 3)))
    keep = torch.rand(ei.shape[1], generator=torch.Generator().manual_seed(2)) > 0.3   # injected edge drops
    ei, et = pyg_restated.dropout_adj(ei, et, 0.3, True, keep)
    if layer == "pyg-1.4":
        conv = pyg2_oracle.RGCNConvRelMeanRef(IN, OUT, R, 2, "mean_per_relation").double()
    else:
        conv = pyg2_oracle.RGCNConv2Ref(IN, OUT, R, 2).double()
    conv.formulation = formulation
    with torch.no_grad():
        conv.bias.uniform_(-0.5, 0.5)   # (the PyG-2 init zeroes it)
    x = torch.randn(n, IN, dtype=torch.float64, requires_grad=True)
    # the graph has what the test is about: zero-edge nodes, a node missing relations, a one-relation node
    assert not (ei[1] == 3).any() and not (ei[1] == 17).any()
    assert not ((ei[1] == 5) & ((et == 1) | (et == 3))).any() and (ei[1] == 5).any()
    assert (ei[1] == 1).any() and (et[ei[1] == 1] == 0).all()
    out = conv(x, ei, et)
    gy = torch.randn_like(out)
    grads = torch.autograd.grad((out * gy).sum(), [x] + list(conv.parameters()))
    ref = _naive(conv, x, ei, et)
    grads_ref = torch.autograd.grad((ref * gy).sum(), [x] + list(conv.parameters()))
    assert torch.allclose(out, ref, rtol=1e-12, atol=1e-12)
    for a, b in zip(grads, grads_ref):
        assert torch.allclose(a, b, rtol=1e-11, atol=1e-12)
    # a zero-edge node is x root + bias only
    assert torch.allclose(out[3], x[3] @ conv.root + conv.bias)


def test_single_relation_mean_equals_mean_all():
    torch.manual_seed(1)
    ei, et = _graph(19, 1, 80, 3, zero_nodes=(4,))
    a = pyg_restated.RGCNConvRef(5, 8, 1, 2, "mean_all").double()
    b = pyg2_oracle.RGCNConvRelMeanRef(5, 8, 1, 2, "mean_per_relation").double()
    b.load_state_dict(a.state_dict())
    x = torch.randn(19, 5, dtype=torch.float64)
    for f in ("bmm", "transform"):
        a.formulation = b.formulation = f
        assert torch.allclose(a(x, ei, et), b(x, ei, et), rtol=1e-14, atol=1e-14)


def test_oracle_models_take_either_layer():
    r1 = pyg_restated.IGMCRef(4, (32, 32), 5, 2, 0.2)
    r2 = pyg2_oracle.IGMC2Ref(4, (32, 32), 5, 2, 0.2)
    assert all(c.aggr == "mean_all" for c in r1.convs) and all(c.aggr == "mean_per_relation" for c in r2.convs)
    assert "convs.0.att" in r1.state_dict() and "convs.0.comp" in r2.state_dict()
    assert "convs.1.weight" in r2.state_dict() and "convs.1.basis" not in r2.state_dict()
    d2 = pyg2_oracle.DGCNN_RS2Ref(4, (32, 32, 1), 30, 5, 2, 0.2)
    assert d2.convs[-1].weight.shape == (2, 32, 1)
    # ARR: the same W_r under either name pair
    with torch.no_grad():
        for c1, c2 in zip(r1.convs, r2.convs):
            c2.comp.copy_(c1.att)
            c2.weight.copy_(c1.basis)
        assert float(pyg_restated.arr_regulariser(r1)) == float(pyg_restated.arr_regulariser(r2))


def _igmc(rgcn, R=5, NB=4, in0=4, L=4):
    from igmc_b200.models import IGMC
    return IGMC(in0, latent_dim=[32] * L, num_relations=R, num_bases=NB, regression=True, rgcn=rgcn)


def _dgcnn(rgcn):
    from igmc_b200.models import DGCNN_RS
    return DGCNN_RS(4, latent_dim=[32, 32, 32, 1], k=30, num_relations=5, num_bases=2, regression=True, rgcn=rgcn)


def test_pyg2_model_names_shapes_and_init():
    torch.manual_seed(0)
    m = _igmc("pyg-2")
    assert m.rgcn == "pyg-2"
    keys = list(m.state_dict())
    assert keys[:4] == ["convs.0.weight", "convs.0.comp", "convs.0.root", "convs.0.bias"]
    assert not any(k.endswith((".att", ".basis")) for k in keys)
    assert keys[-4:] == ["lin1.weight", "lin1.bias", "lin2.weight", "lin2.bias"]
    for l, c in enumerate(m.convs):
        ind = 4 if l == 0 else 32
        assert (c.in_channels, c.out_channels, c.num_relations, c.num_bases) == (ind, 32, 5, 4)
        assert c.weight.shape == (4, ind, 32) and c.comp.shape == (5, 4)
        assert c.root.shape == (ind, 32) and c.bias.shape == (32,)
        for p in (c.weight, c.comp, c.root):
            bound = math.sqrt(6.0 / (p.size(-2) + p.size(-1)))
            assert float(p.abs().max()) <= bound and float(p.abs().max()) > 0.5 * bound
        assert torch.equal(c.bias, torch.zeros(32))
    # the parameters are views of the flat bucket, in the slots of (att, basis)
    for e, (kind, l, p) in zip(m._layout, m._named_order()):
        assert p.data_ptr() == m._pview(m.flat_params, e).data_ptr()
    assert m._named_order().__next__()[2] is m.convs[0].comp
    # optimizer order = model.parameters(): weight, comp, root, bias per conv (PyG 2 registration order)
    assert list(m.parameters())[0] is m.convs[0].weight and list(m.parameters())[1] is m.convs[0].comp

    d = _dgcnn("pyg-2")
    dk = list(d.state_dict())
    assert "convs.3.weight" in dk and "convs.3.comp" in dk and "convs.3.att" not in dk
    assert d.convs[3].weight.shape == (2, 32, 1) and d.convs[3].root.shape == (32, 1)
    assert torch.equal(d.convs[3].bias, torch.zeros(1))


def test_default_model_names_unchanged():
    m = _igmc("pyg-1.4")
    assert m.rgcn == "pyg-1.4"
    assert list(m.state_dict())[:4] == ["convs.0.basis", "convs.0.att", "convs.0.root", "convs.0.bias"]
    m0 = __import__("igmc_b200.models", fromlist=["IGMC"]).IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4,
                                                                 regression=True)
    assert list(m0.state_dict()) == list(m.state_dict()) and m0.rgcn == "pyg-1.4"
    d = _dgcnn("pyg-1.4")
    assert "convs.3.basis" in d.state_dict() and "convs.3.weight" not in d.state_dict()


def test_strict_loading_across_layers_fails_and_bad_keyword_raises():
    m1, m2 = _igmc("pyg-1.4"), _igmc("pyg-2")
    for dst, src in ((m2, m1), (m1, m2)):
        for strict in (True, False):
            with pytest.raises(RuntimeError, match="other RGCNConv layer"):
                dst.load_state_dict(src.state_dict(), strict=strict)
    # a checkpoint of the same layer round-trips
    m3 = _igmc("pyg-2")
    m3.load_state_dict(m2.state_dict())
    assert torch.equal(m3.flat_params, m2.flat_params)
    d1, d2 = _dgcnn("pyg-1.4"), _dgcnn("pyg-2")
    with pytest.raises(RuntimeError):
        d2.load_state_dict(d1.state_dict())
    for bad in ("pyg-1.6", "mean", None, 2):
        with pytest.raises(ValueError):
            _igmc(bad)
        with pytest.raises(ValueError):
            _dgcnn(bad)


def test_new_mode_selects_the_same_plans():
    """the mode lives in igmc_saved_t.rel_inv_deg and needs no extra shared memory: every plan query and therefore
    ``select_plan`` answer the same for both layers over the shapes tests/test_l2_plan.py sweeps"""
    import ctypes
    from igmc_b200 import _lib
    from igmc_b200.models import select_plan
    lib = _lib.load()
    n_caps = sorted(set(list(range(2, 1201, 40)) + [256, 257, 382, 383, 422, 423, 434, 435, 446, 447, 568, 569, 1200]))
    for R in (1, 5, 10, 12, 13, 71, 256):
        for NB in (2, 4):
            for in0 in (4, 6, 8):
                a, b = _igmc("pyg-1.4", R, NB, in0), _igmc("pyg-2", R, NB, in0)
                assert bytes(a._cmodel) == bytes(b._cmodel)
                for B in (16, 50):
                    for n_cap in n_caps:
                        assert select_plan(a._cmodel, n_cap, B, 132) == select_plan(b._cmodel, n_cap, B, 132)
                for plan in (0, 1, 2, 4, _lib.plan_l2(4)):
                    for bw in (0, 1):
                        assert lib.igmc_model_plan(ctypes.byref(b._cmodel), 402, plan, bw) == \
                            lib.igmc_model_plan(ctypes.byref(a._cmodel), 402, plan, bw)


def test_saved_struct_carries_the_table():
    import ctypes
    from igmc_b200 import _lib
    P = ctypes.sizeof(ctypes.c_void_p)
    assert _lib.Saved.rel_inv_deg.offset == _lib.Saved.l2_scratch.offset + P   # trailing field
    assert _lib.Saved().rel_inv_deg is None                                       # NULL: PyG 1.4.2 semantics
