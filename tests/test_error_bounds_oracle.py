"""CPU checks of the layer-by-layer fp64 oracle and its magnitude pass (tests/error_bounds.py), and a numpy emulation of
the relation-space kernels' 3xTF32 tensor-core products that ties the committed error constants to the arithmetic."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pyg_restated
from tests import edge_weight_oracle as ewo
from tests import error_bounds as eb
from tests import pyg2_oracle
from tests.test_gpu_model import _oracle_batch


def _ref(rgcn, in0, L, R=5, NB=4, dgcnn_last=None, k=30):
    torch.manual_seed(0)
    if dgcnn_last is None:
        ref = pyg2_oracle.igmc_ref(rgcn, in0, (32,) * L, R, NB, 0.2, 2)     # multiply_by 2: scales dpred too
    else:
        ref = pyg2_oracle.dgcnn_rs_ref(rgcn, in0, (32, 32, 32, dgcnn_last), k, R, NB, 0.2)
    with torch.no_grad():
        for c in ref.convs:
            c.bias.uniform_(-0.3, 0.3)     # PyG 2 zero-inits the bias
    return pyg_restated.set_formulation(ref.double().train(), "transform")


def _oracle_saved(ref, ob, ek, hk):
    """what the kernels would save, computed by the whole restated model: states, hidden scales, SortPooling order and
    ReLU outputs, and dpred of the MSE + ARR loss; with the model's own fp64 loss gradients in ``.grad``"""
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    ref.zero_grad()
    dg = isinstance(ref, pyg_restated.DGCNN_RSRef)
    B = ob["num_graphs"]
    if dg:
        out, cs = ref(tb["x"], tb["edge_index"], tb["edge_type"], tb["batch"], ek, hk, B, return_states=True)
    else:
        out, cs = ref(tb["x"], tb["edge_index"], tb["edge_type"], ek, hk, return_states=True)
    loss = F.mse_loss(out, tb["y"].view(-1)) + 0.001 * pyg_restated.arr_regulariser(ref)
    loss.backward()
    cs = cs.detach()
    widths = [c.out_channels for c in ref.convs]
    saved = dict(states=list(torch.split(cs, widths, 1)), out=out.detach(), hidden_keep=hk)
    mult = 1.0 if dg else float(ref.multiply_by)
    saved["dpred"] = 2.0 * (out.detach() - tb["y"].view(-1)) / B * mult
    pre1 = _readout_branches(ref, ob, tb, cs, saved)
    saved["gscale"] = (pre1 > 0).double() * hk.double() * 2.0
    return saved


def _readout_branches(ref, ob, tb, cs, saved):
    """the readout branches the kernels save of the restated model's concat states ``cs`` into ``saved`` (DGCNN_RS:
    SortPooling order, conv1 and conv2 ReLU outputs); returns the lin1 pre-activation"""
    B = ob["num_graphs"]
    with torch.no_grad():
        if isinstance(ref, pyg_restated.DGCNN_RSRef):
            z = pyg_restated.global_sort_pool(cs, tb["batch"], ref.k, B).unsqueeze(1)
            act1 = F.relu(ref.conv1d_params1(z))
            flat = F.relu(ref.conv1d_params2(ref.maxpool1d(act1))).reshape(B, -1)
            feat = flat
            nptr = np.concatenate([[0], np.cumsum(np.bincount(ob["batch"], minlength=B))])
            perm = torch.full((B, ref.k), -1, dtype=torch.long)
            for gi in range(B):
                order = nptr[gi] + np.argsort(-cs[nptr[gi]:nptr[gi + 1], -1].numpy(), kind="stable")[:ref.k]
                perm[gi, :len(order)] = torch.from_numpy(order)
            saved.update(perm=perm, act1=act1, flat=flat)
        else:
            x = tb["x"]
            feat = torch.cat([cs[x[:, 0] == 1], cs[x[:, 1] == 1]], 1)
        return ref.lin1(feat)


def _case(rgcn, in0, L, dgcnn_last=None, R=5):
    ob = _oracle_batch(R=R, h=(in0 - 2) // 2)[3]
    assert ob["x"].shape[1] == in0
    ref = _ref(rgcn, in0, L, R=R, dgcnn_last=dgcnn_last)
    gen = torch.Generator().manual_seed(11)
    ek = torch.rand(ob["edge_index"].shape[1], generator=gen) > 0.2
    hk = torch.rand(ob["num_graphs"], 128, generator=gen) > 0.5
    saved = _oracle_saved(ref, ob, ek, hk)
    params = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    aggr = ref.convs[0].aggr
    return ref, ob, eb.Graph(ob, ek), saved, params, aggr, dgcnn_last is not None


def _close(a, b, rel=1e-12):
    assert float((a - b).abs().max()) <= rel * (float(b.abs().max()) + 1e-300), (float((a - b).abs().max()),
                                                                               float(b.abs().max()))


CASES = [("pyg-1.4", 4, 4, None), ("pyg-1.4", 4, 1, None), ("pyg-1.4", 4, 8, None), ("pyg-1.4", 6, 4, None),
         ("pyg-1.4", 8, 4, None), ("pyg-2", 4, 4, None), ("pyg-2", 6, 1, None), ("pyg-2", 8, 8, None),
         ("pyg-1.4", 4, 4, 1), ("pyg-1.4", 4, 4, 8), ("pyg-2", 4, 4, 1), ("pyg-2", 6, 4, 8)]


@pytest.mark.parametrize("rgcn,in0,L,last", CASES)
def test_chained_layers_equal_whole_model_autograd(rgcn, in0, L, last):
    """per-layer forward from the saved states and the chained per-layer VJPs from dpred equal the whole restated model
    and its fp64 autograd (train mode, injected edge and hidden masks, ARR term): 1e-12 relative"""
    ref, ob, g, saved, params, aggr, dg = _case(rgcn, in0, L, last)
    pres, out = eb.forward(params, g, saved, aggr, dg)
    for pre, h in zip(pres, saved["states"]):
        _close(torch.tanh(pre), h)
    mult = 1.0 if dg else float(ref.multiply_by)
    _close(out * mult, saved["out"])
    dhid, grads = eb.backward(params, g, saved, aggr, dg, 0.001)
    assert set(grads) == set(params)
    for name, p in ref.named_parameters():
        _close(grads[name], p.grad)
    # d hid is d loss / d (lin1 output after ReLU and dropout): its sum over graphs is lin1.bias's gradient
    _close((dhid).sum(0), ref.lin1.bias.grad)


@pytest.mark.parametrize("rgcn,in0,L,last", [CASES[0], CASES[5], CASES[9], CASES[11]])
def test_magnitude_bounds_every_element(rgcn, in0, L, last):
    """M >= |ref| element by element (pre-activations, readout output, d hid, every gradient, ARR included)"""
    ref, ob, g, saved, params, aggr, dg = _case(rgcn, in0, L, last)
    pres, out = eb.forward(params, g, saved, aggr, dg)
    mpres, mout = eb.forward(params, g, saved, aggr, dg, mag=True)
    for a, m in list(zip(pres, mpres)) + [(out, mout)]:
        assert bool((m >= a.abs()).all())
    dhid, grads = eb.backward(params, g, saved, aggr, dg, 0.001)
    mdhid, mgrads = eb.backward(params, g, saved, aggr, dg, 0.001, mag=True)
    assert bool((mdhid >= dhid.abs()).all())
    for k in grads:
        assert bool((mgrads[k] >= grads[k].abs() * (1 - 1e-12)).all()), k
        assert float(mgrads[k].abs().max()) > 0, k


@pytest.mark.parametrize("rgcn,in0,L,last", [CASES[0], CASES[6], CASES[10]])
def test_magnitude_equals_value_on_nonnegative_inputs(rgcn, in0, L, last):
    """with every operand non-negative (and no ARR: its differences turn into sums) M is the value itself"""
    ref, ob, g, saved, params, aggr, dg = _case(rgcn, in0, L, last)
    params = {k: v.abs() for k, v in params.items()}
    saved = dict(saved, states=[h.abs() for h in saved["states"]], dpred=saved["dpred"].abs())
    for a, m in zip(eb.forward(params, g, saved, aggr, dg)[0], eb.forward(params, g, saved, aggr, dg, mag=True)[0]):
        assert torch.equal(a, m)
    dhid, grads = eb.backward(params, g, saved, aggr, dg, 0.0)
    mdhid, mgrads = eb.backward(params, g, saved, aggr, dg, 0.0, mag=True)
    assert torch.equal(dhid, mdhid)
    for k in grads:
        assert torch.equal(grads[k], mgrads[k]), k


def test_ratio_fails_on_nan_and_nonzero_padding():
    """a NaN or infinity in got makes the ratio infinite wherever it sits, so it cannot hide the other elements; a
    nonzero value where M == 0 is counted"""
    ref = torch.tensor([1.0, 2.0, 3.0, 0.0], dtype=torch.float64)
    M = ref.clone()
    assert eb.ratio(ref + eb.U * M, ref, M)[:2] == (1.0, 0)
    for bad in (float("nan"), float("inf")):
        got = ref.clone()
        got[1] = bad
        r, pad, worst = eb.ratio(got, ref, M)
        assert r == float("inf") and pad == 0 and worst == 1
        res = dict(branches=0, pred=(r, pad, worst))
        assert eb.violations(res) == [("pred", r, pad, worst)]
    got = ref.clone()
    got[3] = float("nan")
    assert eb.ratio(got, ref, M)[1] == 1
    assert eb.violations(dict(branches=2, states0=(0.0, 0, 0))) == [("branches", 2)]


@pytest.mark.parametrize("rgcn,in0,L,last", [CASES[0], CASES[9], CASES[11]])
def test_branches_agree_and_flipped_branches_are_found(rgcn, in0, L, last):
    """on the whole model's own branches nothing mismatches; a hidden unit zeroed although its pre-activation is
    clearly positive, a conv1 ReLU flipped and two swapped sort-pool positions are each found"""
    ref, ob, g, saved, params, aggr, dg = _case(rgcn, in0, L, last)
    hk = saved["hidden_keep"]
    assert eb.branch_mismatches(params, g, saved, dg, hk) == 0
    parts = {}
    with torch.no_grad():
        eb.head(torch.cat(saved["states"], 1), params, g, saved, dg, parts)
    pos = torch.nonzero((parts["lin1"] > 1e-3) & hk)[0]
    gscale = saved["gscale"].clone()
    gscale[pos[0], pos[1]] = 0.0
    assert eb.branch_mismatches(params, g, dict(saved, gscale=gscale), dg, hk) == 1
    gscale = saved["gscale"].clone()
    gscale[pos[0], pos[1]] = 2.0
    gscale[~hk] = 2.0                                   # a dropped unit kept
    assert eb.branch_mismatches(params, g, dict(saved, gscale=gscale), dg, hk) >= 1
    if dg:
        act1 = saved["act1"].clone()
        c = torch.nonzero(parts["conv1"] > 1e-3)[0]
        act1[c[0], c[1], c[2]] = 0.0
        assert eb.branch_mismatches(params, g, dict(saved, act1=act1), dg, hk) >= 1
        perm = saved["perm"].clone()
        perm[0, [0, 1]] = perm[0, [1, 0]]
        assert eb.branch_mismatches(params, g, dict(saved, perm=perm), dg, hk) >= 2


# ---- 3xTF32 separation ----------------------------------------------------------------------------------------------
def _tf32(a):
    """the top 10 mantissa bits: a mask of the 13 low ones (what the kernels' split and the tensor core's read keep)"""
    return (np.asarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def emulate_3xtf32(A, B, K1, drop=None):
    """[A1 | A2] . B of csrc/rgcn_rs.cu ``tiles_span`` / ``tiles_span2`` in fp32: k-steps of 8, even steps of the
    first span (K1 columns) into (d, e), odd steps and the second span into (d2, e2), e / e2 taking the cross terms
    lo_a hi_b then hi_a lo_b, result (d + d2) + (e + e2).  One k-step's 8 products (exact tf32 x tf32) are summed
    exactly and added to the fp32 accumulator with one rounding.  ``drop``: "al_bh" or "ah_bl" leaves that term out."""
    A, B = np.asarray(A, np.float32), np.asarray(B, np.float32)
    ah, bh = _tf32(A), _tf32(B)
    al, bl = _tf32(A - ah), _tf32(B - bh)          # lo = x - hi is exact in fp32; the tensor core reads 10 bits of it
    acc = {n: np.zeros((A.shape[0], B.shape[1]), np.float32) for n in ("d", "e", "d2", "e2")}

    def add(name, a, b, k0):
        s = slice(k0, k0 + 8)
        acc[name] = (acc[name].astype(np.float64) + a[:, s].astype(np.float64) @ b[s].astype(np.float64)) \
            .astype(np.float32)

    for k0 in range(0, A.shape[1], 8):
        second = k0 >= K1 or (k0 // 8) % 2 == 1 and (k0 // 16 + 1) * 16 <= K1
        d, e = ("d2", "e2") if second else ("d", "e")
        if drop != "al_bh":
            add(e, al, bh, k0)
        if drop != "ah_bl":
            add(e, ah, bl, k0)
        add(d, ah, bh, k0)
    return (acc["d"] + acc["d2"]) + (acc["e"] + acc["e2"])


def _layer1_operands():
    """one real layer-1 transform of the relation-space kernels on the R = 5 oracle batch: A = [AGG' | h] (the
    1/deg-scaled per-relation sums of the layer-0 states, fp32) and B = [W_1 .. W_R ; root] (fp32)"""
    R = 5
    ob = _oracle_batch(R=R)[3]
    ref = _ref("pyg-1.4", 4, 4, R=R)
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    with torch.no_grad():
        h = torch.tanh(ref.convs[0](tb["x"], tb["edge_index"], tb["edge_type"])).float().double()
        src, dst = tb["edge_index"]
        N = h.shape[0]
        agg = torch.zeros(N * R, 32, dtype=torch.float64).index_add_(0, dst * R + tb["edge_type"], h[src])
        deg = torch.bincount(dst, minlength=N).clamp(min=1).double()
        agg = (agg.view(N, R, 32).float() * (1.0 / deg.float()).view(N, 1, 1)).reshape(N, R * 32)
        c = ref.convs[1]
        W = torch.einsum("rb,bio->rio", c.att, c.basis).float().reshape(R * 32, 32)
        B = torch.cat([W, c.root.float()], 0)
    return torch.cat([agg, h.float()], 1).numpy(), B.numpy(), R * 32


def _worst(C, A, B):
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    return float((np.abs(C.astype(np.float64) - A64 @ B64) / (eb.U * (np.abs(A64) @ np.abs(B64)))).max())


def test_3xtf32_emulation_within_kappa_and_lost_cross_term_beyond():
    """the kernels' 3xTF32 product on real operands stays within KAPPA["states"] u M; the same product without either
    cross term exceeds it (so the committed constant separates fp32-level accuracy from a TF32 slip)"""
    A, B, K1 = _layer1_operands()
    assert A.shape[1] == K1 + 32 and np.count_nonzero(A[:, :K1]) > 0
    ok = _worst(emulate_3xtf32(A, B, K1), A, B)
    print("3xTF32 emulation: largest err / (u M) = %.2f (KAPPA states %g)" % (ok, eb.KAPPA["states"]))
    assert ok <= eb.KAPPA["states"]
    for drop in ("ah_bl", "al_bh"):
        bad = _worst(emulate_3xtf32(A, B, K1, drop), A, B)
        print("  without %s: %.0f" % (drop, bad))
        assert bad > eb.KAPPA["states"], drop


# ---- edge terms: the per-rating gradient of attribute_pairs (igmc_edge_grad) ---------------------------------------
def _eval_case(rgcn, in0, L, NB, R, last):
    """the restated model in eval mode on the oracle batch and what the kernels keep of its eval forward, seeded as
    the gradient pass of attribute_pairs seeds them: dpred = d score / d lin2 output (multiply_by) for IGMC; for
    DGCNN_RS dstate, the readout's VJP seeded with 1 at the concat states (true widths)"""
    ob = _oracle_batch(R=R, h=(in0 - 2) // 2)[3]
    assert ob["x"].shape[1] == in0
    ref = _ref(rgcn, in0, L, R=R, NB=NB, dgcnn_last=last).eval()
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    B, dg = ob["num_graphs"], last is not None
    with torch.no_grad():
        if dg:
            _, cs = ref(tb["x"], tb["edge_index"], tb["edge_type"], tb["batch"], num_graphs=B, return_states=True)
        else:
            _, cs = ref(tb["x"], tb["edge_index"], tb["edge_type"], return_states=True)
    saved = dict(states=list(torch.split(cs, [c.out_channels for c in ref.convs], 1)))
    saved["gscale"] = (_readout_branches(ref, ob, tb, cs, saved) > 0).double()
    saved["dpred"] = torch.full((B,), 1.0 if dg else float(ref.multiply_by), dtype=torch.float64)
    params = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    g = eb.Graph(ob)
    if dg:
        saved["dstate"] = eb.readout_dstate(params, g, saved, True)
    return ref, ob, tb, g, saved, params, ref.convs[0].aggr, dg


# (rgcn, in0, L, NB, R, DGCNN_RS last layer width or None)
EDGE_CASES = [("pyg-1.4", 4, 4, 4, 5, None), ("pyg-1.4", 4, 1, 2, 5, None), ("pyg-1.4", 6, 8, 2, 1, None),
              ("pyg-1.4", 8, 4, 4, 13, None), ("pyg-2", 4, 4, 2, 5, None), ("pyg-1.4", 6, 1, 4, 13, None),
              ("pyg-2", 8, 8, 2, 1, None), ("pyg-1.4", 4, 4, 2, 5, 1), ("pyg-2", 4, 4, 4, 13, 1),
              ("pyg-2", 6, 4, 2, 5, 8)]


def _segments(g, aggr, R):
    """segment id of every directed edge and the segment's size"""
    dst, et = g.edge_index[1], g.edge_type
    seg = dst * R + et if aggr == "mean_per_relation" else dst
    return seg, torch.bincount(seg)[seg]


@pytest.mark.parametrize("rgcn,in0,L,NB,R,last", EDGE_CASES)
def test_edge_terms_equal_weighted_model_autograd(rgcn, in0, L, NB, R, last):
    """edge_terms from the restated model's own fp64 states and seed equal d (sum of scores) / d w_e of the weighted
    restatement by autograd (DGCNN_RS in the restatement's own pooling order): 1e-12 relative"""
    ref, ob, tb, g, saved, params, aggr, dg = _eval_case(rgcn, in0, L, NB, R, last)
    kw = dict(batch=tb["batch"], num_graphs=ob["num_graphs"], perm=saved["perm"]) if dg else {}
    want = ewo.autograd_edge_grad(ref, tb["x"], tb["edge_index"], tb["edge_type"], **kw)
    got = eb.edge_terms(params, g, saved, aggr, dg)
    assert float(want.abs().max()) > 1e-6
    _close(got, want)


@pytest.mark.parametrize("rgcn,in0,L,NB,R,last", EDGE_CASES)
def test_edge_magnitude_bounds_and_exact_zeros(rgcn, in0, L, NB, R, last):
    """M >= |ref| per edge; an edge whose segment has one entry is exactly 0 in fp64 too; with L = 1 every edge into a
    node other than the two targets has M == 0.  DGCNN_RS: the dstate magnitude bounds its value as well"""
    _, _, _, g, saved, params, aggr, dg = _eval_case(rgcn, in0, L, NB, R, last)
    ref, M = eb.edge_terms(params, g, saved, aggr, dg), eb.edge_terms(params, g, saved, aggr, dg, mag=True)
    assert bool((M >= ref.abs() * (1 - 1e-12)).all()) and float(M.max()) > 0
    _, size = _segments(g, aggr, R)
    single = size == 1
    print("edge terms %s: %d edges, %d in single-entry segments" % ((rgcn, in0, L, NB, R, last), len(M), int(single.sum())))
    assert int(single.sum()) > 0 and bool((ref[single] == 0).all())
    if L == 1:
        target = (g.users | g.items)[g.edge_index[1]]
        assert bool((M[~target] == 0).all()) and bool((M[target] > 0).any())
    if dg:
        ds, mds = eb.readout_dstate(params, g, saved, True), eb.readout_dstate(params, g, saved, True, mag=True)
        assert bool((mds >= ds.abs()).all()) and float(mds.max()) > 0


def emulate_edge_grad(params, g, saved, aggr, dpres, plant=None):
    """igmc_edge_grad's arithmetic (csrc/rgcn_l2.cu ``edge_terms``) in numpy fp32 from fp32 operands (h, att, basis,
    each layer's d pre): dZ' = d pre . basis^T rounded (1/deg(v) applied to it under mean_all), p = sum_b att dZ'
    rounded, the products h * p rounded and summed to t, the segment's sum of t divided once by its size, t - mean
    (mean_per_relation: times 1/|N_r(v)|), the layers added from the top one down.  ``plant`` is one slip: "inv_seg"
    drops the 1/|segment|, "segment" takes v's whole in-list as the segment under mean_per_relation, "layer" leaves
    layer 0's term out, "tf32_h" truncates h to TF32"""
    f = np.float32
    att_n, basis_n = eb.conv_names(params)[:2]
    R = params["convs.0." + att_n].shape[0]
    per_rel = aggr == "mean_per_relation" and plant != "segment"
    seg, size = _segments(g, "mean_per_relation" if per_rel else "mean_all", R)
    seg, size = seg.numpy(), size.numpy().astype(f)
    src, dst, et = g.edge_index[0].numpy(), g.edge_index[1].numpy(), g.edge_type.numpy()
    N = g.x.shape[0]
    one = plant == "inv_seg"
    invdeg = np.ones(N, f) if one else f(1) / np.maximum(np.bincount(dst, minlength=N), 1).astype(f)
    inv = np.ones(len(seg), f) if one else f(1) / size
    out = np.zeros(len(seg), f)
    for l in reversed(range(len(dpres))):
        if plant == "layer" and l == 0:
            continue
        h = (g.x if l == 0 else saved["states"][l - 1]).numpy().astype(f)
        if plant == "tf32_h":
            h = _tf32(h)
        att = params["convs.%d.%s" % (l, att_n)].numpy().astype(f)
        basis = params["convs.%d.%s" % (l, basis_n)].numpy().astype(f)[:, :h.shape[1]]
        dz = np.einsum("vk,bik->vbi", dpres[l].numpy().astype(f).astype(np.float64), basis.astype(np.float64)).astype(f)
        if not per_rel:
            dz = dz * invdeg[:, None, None]
        p = np.einsum("rb,vbi->vri", att.astype(np.float64), dz.astype(np.float64)).astype(f)
        t = (h[src] * p[dst, et]).sum(1, dtype=f)
        tot = np.zeros(seg.max() + 1 if len(seg) else 0, f)
        np.add.at(tot, seg, t)
        d = t - tot[seg] / size
        out = out + (d * inv if per_rel else d)
    return out


@pytest.mark.parametrize("rgcn", ["pyg-1.4", "pyg-2"])
def test_edge_emulation_within_kappa_and_planted_slips_beyond(rgcn):
    """the fp32 emulation of igmc_edge_grad on fp32 operands stays within KAPPA["edge"] u M of edge_terms on the same
    operands; a dropped 1/|segment|, the pyg-1.4 segment under pyg-2 and a layer's term left out each exceed it by far.
    TF32-truncated h is 100s of times the emulation's own ratio but only a few KAPPA["edge"]: M carries the magnitude
    pass's d pre (the bound on the kernel's own d pre error), far above |d pre|, so it cannot single out a 2^-11 error
    in h"""
    _, _, _, g, saved, params, aggr, _ = _eval_case(rgcn, 4, 4, 4, 5, None)
    params = {k: v.float().double() for k, v in params.items()}
    saved = dict(saved, states=[h.float().double() for h in saved["states"]])
    dpres = []
    eb.backward(params, g, saved, aggr, False, 0.0, dpres=dpres)
    ref, M = eb.edge_terms(params, g, saved, aggr, False), eb.edge_terms(params, g, saved, aggr, False, mag=True)
    ok, pad, _ = eb.ratio(torch.from_numpy(emulate_edge_grad(params, g, saved, aggr, dpres)), ref, M)
    print("edge emulation %s: largest err / (u M) = %.3g (KAPPA edge %g)" % (rgcn, ok, eb.KAPPA["edge"]))
    assert ok <= eb.KAPPA["edge"] and pad == 0
    for plant in ("inv_seg", "layer", "tf32_h") + (("segment",) if rgcn == "pyg-2" else ()):
        bad = eb.ratio(torch.from_numpy(emulate_edge_grad(params, g, saved, aggr, dpres, plant)), ref, M)[0]
        print("  with %s: %.3g" % (plant, bad))
        if plant == "tf32_h":
            assert bad > 100 * ok, plant
        else:
            assert bad > 100 * eb.KAPPA["edge"], plant


# ---- optimizer and prepared weights ---------------------------------------------------------------------------------
def emulate_adam(p, m, v, g, step, lr, b1, b2, eps, wd, plant=None):
    """k_adam (csrc/optim.cu) in numpy fp32, one rounding per operation; bias corrections 1 - exp(step log beta) in
    double, rounded to fp32.  ``plant``: "step" (bias corrections of the step after), "wd" (weight decay left out),
    "eps_in_sqrt" (sqrt(v / bc2 + eps) in place of sqrt(v) / sqrt(bc2) + eps)"""
    f = np.float32
    p, m, v, g = [np.asarray(t, np.float32) for t in (p, m, v, g)]
    s = step + (1 if plant == "step" else 0)
    bc1 = f(1.0 - np.exp(s * np.log(np.float64(f(b1)))))
    bc2 = f(1.0 - np.exp(s * np.log(np.float64(f(b2)))))
    gg = g
    if wd and plant != "wd":
        gg = f(np.float64(f(wd)) * p + gg)        # fmaf: the fp32 product is exact in fp64
    mi = f(b1) * m + (f(1) - f(b1)) * gg
    vi = f(b2) * v + (f(1) - f(b2)) * gg * gg
    den = np.sqrt(vi / bc2 + f(eps)) if plant == "eps_in_sqrt" else np.sqrt(vi) / np.sqrt(bc2) + f(eps)
    return mi, vi, p - (f(lr) / bc1) * (mi / den)


def _adam_state(fresh, n=4096, seed=3):
    """parameters ~ 0.1, gradients ~ 1e-3 (a few exact zeros: padding slots), moments of a resumed run or zero"""
    rng = np.random.default_rng(seed)
    p = (rng.standard_normal(n) * 0.1).astype(np.float32)
    g = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    p[:8], g[:8] = 0, 0
    if fresh:
        m = v = np.zeros(n, np.float32)
    else:
        m = (rng.standard_normal(n) * 1e-3).astype(np.float32)
        v = ((1.5 * m) ** 2 + 1e-8).astype(np.float32)
        m[:8], v[:8] = 0, 0
    return p, m, v, g


ADAM_CASES = {   # name -> (fresh state, step, weight decay, lr)
    "step1": (True, 1, 0.0, 1e-3), "step2": (False, 2, 0.0, 1e-3), "step3_wd": (False, 3, 1e-2, 1e-3),
    "step5000_wd": (False, 5000, 1e-2, 2e-4),
}


@pytest.mark.parametrize("case", sorted(ADAM_CASES))
def test_adam_emulation_within_kappa(case):
    fresh, step, wd, lr = ADAM_CASES[case]
    p, m, v, g = _adam_state(fresh)
    terms = eb.adam_terms(*[torch.from_numpy(t) for t in (p, m, v, g)], step, lr, 0.9, 0.999, 1e-8, wd)
    res = eb.adam_check([torch.from_numpy(t) for t in emulate_adam(p, m, v, g, step, lr, 0.9, 0.999, 1e-8, wd)], terms)
    print("adam emulation %s: %s" % (case, {k: round(r[0], 3) for k, r in res.items()}))
    assert not eb.violations(res), res


@pytest.mark.parametrize("plant,case", [("step", "step1"), ("step", "step2"), ("step", "step3_wd"),
                                        ("wd", "step3_wd"), ("wd", "step5000_wd"),
                                        ("eps_in_sqrt", "step2"), ("eps_in_sqrt", "step5000_wd")])
def test_adam_planted_slips_beyond_kappa(plant, case):
    """an off-by-one step in the bias corrections (steps 1 to 3: at step 5000 both are ~1 and the slip is below one
    rounding of |p|), weight decay left out, eps inside the square root: each moves the parameter by far more than
    KAPPA["adam"] u M.  The margins on these states are printed; the assertion asks for 100x"""
    fresh, step, wd, lr = ADAM_CASES[case]
    p, m, v, g = _adam_state(fresh)
    terms = eb.adam_terms(*[torch.from_numpy(t) for t in (p, m, v, g)], step, lr, 0.9, 0.999, 1e-8, wd)
    got = emulate_adam(p, m, v, g, step, lr, 0.9, 0.999, 1e-8, wd, plant)
    res = eb.adam_check([torch.from_numpy(t) for t in got], terms)
    worst = max(r[0] for r in res.values())
    print("adam %s at %s: largest err / (u M) %.3g = %.0f x KAPPA" % (plant, case, worst, worst / eb.KAPPA["adam"]))
    assert worst > 100 * eb.KAPPA["adam"]


def emulate_wprep(params, L, R, in0, plant=None):
    """igmc_prep_weights in fp32: W_r[k][j] = fma chain over the bases; ``plant`` "basis_tf32" rounds the basis
    operand to TF32 (10 mantissa bits), "drop_basis" leaves the last basis out"""
    ref, M, copied, written = eb.wprep_terms(params, L, R, in0)
    out = torch.zeros_like(ref, dtype=torch.float32)
    att_n, basis_n = eb.conv_names(params)[:2]
    slab = 32 * ((R + 1) * 32 + 4)
    for l in range(L):
        at = params["convs.%d.%s" % (l, att_n)].float()
        bs = params["convs.%d.%s" % (l, basis_n)].float()
        if plant == "basis_tf32":
            bs = (bs.view(torch.int32) & ~0x1FFF).view(torch.float32)
        NB = at.shape[1] - (1 if plant == "drop_basis" else 0)
        W = torch.zeros(R, bs.shape[1], 32, dtype=torch.float32)
        for b in range(NB):       # w = fmaf(att, basis, w): product exact in fp64, one rounding per term
            W = (at[:, b, None, None].double() * bs[b].double() + W.double()).float()
        rt = params["convs.%d.root" % l].float()
        fin = bs.shape[1]
        inp = (fin + 3) & ~3
        K1p = (R * inp + 7) & ~7
        KS = K1p + ((inp + 7) & ~7) + 4
        for d in (0, 1) if l else (0,):
            rows = torch.zeros(32, KS)
            rows[:, :R * inp].view(32, R, inp)[:, :, :fin] = W.permute(2, 0, 1) if d == 0 else W.permute(1, 0, 2)
            rows[:, K1p:K1p + fin] = rt.t() if d == 0 else rt
            o = (l * 2 + d) * slab
            out[o:o + 32 * KS] = rows.reshape(-1)
    return out, (ref, M, copied, written)


@pytest.mark.parametrize("L,R,NB,rgcn", [(1, 5, 4, "pyg-1.4"), (4, 8, 2, "pyg-1.4"), (2, 5, 4, "pyg-2")])
def test_wprep_emulation_within_kappa_and_planted_slips_beyond(L, R, NB, rgcn):
    from igmc_b200.models import IGMC
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * L, num_relations=R, num_bases=NB, regression=True, rgcn=rgcn)
    params = {k: v.detach().clone() for k, v in m.state_dict().items()}
    out, terms = emulate_wprep(params, L, R, 4)
    res = eb.wprep_check(out, terms)
    print("wprep emulation L%d R%d NB%d %s: %.3g" % (L, R, NB, rgcn, res["wprep"][0]))
    assert not eb.violations(res), res
    for plant in ("basis_tf32", "drop_basis"):
        bad = eb.wprep_check(emulate_wprep(params, L, R, 4, plant)[0], terms)["wprep"][0]
        print("  with %s: %.3g = %.0f x KAPPA" % (plant, bad, bad / eb.KAPPA["wprep"]))
        assert bad > 100 * eb.KAPPA["wprep"], plant
    # a root column off by one row, and a stray value in the padding, are each found exactly
    _, M, copied, written = terms
    for where in (copied, written & (M == 0) & ~copied):
        o = out.clone()
        i = int(torch.nonzero(where)[len(torch.nonzero(where)) // 2])
        o[i] += 1e-3
        r = eb.wprep_check(o, terms)
        assert r["wprep_root"][1] + r["wprep"][1] == 1
