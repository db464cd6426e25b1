"""A numpy fp32 emulation of k_pair_grad_raw (csrc/influence.cu) against the per-pair bound of tests/error_bounds.py,
without a GPU: the emulation stays inside KAPPA["grad"] * u * M, and each planted slip of the kernel's indexing or
summation exceeds it by at least 100x.

The kernel's inputs are built in fp64 on a small oracle batch: graph q's raw rows (per layer dW_r | d root | d bias,
csrc/common.cuh igmc_raw_off) from ``backward``'s d pre of that graph alone, split into CL partial rows by the node
ranges the CTAs of a cluster own (tests/helpers.py own_counts) and rounded to fp32.  The emulation sums them in the
kernel's order: ranks in order, then r (d basis, an fmaf chain), then k (d att, one fmaf chain over j per k)."""
import numpy as np
import pytest
import torch

from oracle import pyg_restated
from tests import error_bounds as eb
from tests import pyg2_oracle
from tests.helpers import a4, own_counts
from tests.test_gpu_model import _oracle_batch

f32 = np.float32


def raw_off(R, in0, l):
    """igmc_raw_off: layer l's offset in a raw row, layers [dW_r: R x inp x 32 | d root: inp x 32 | d bias: 32]"""
    per = lambda inp: (R + 1) * inp * 32 + 32      # noqa: E731
    return 0 if l == 0 else per(a4(in0)) + (l - 1) * per(32)


def _fma(a, b, c):
    """fmaf in numpy: the fp32 product is exact in fp64, one rounding of the sum (to fp64, then to fp32)"""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def _setup(in0, L, R, NB, rgcn="pyg-1.4", mb=2.0):
    """(params, oracle batch, saved, aggr) of a restated IGMC with fp32-valued parameters on a 6-graph oracle batch:
    the states its forward saves (rounded to fp32), the ReLU mask as gscale and a loss seed per graph"""
    ob = _oracle_batch(R=R, h=(in0 - 2) // 2, B=6)[3]
    torch.manual_seed(0)
    ref = pyg2_oracle.igmc_ref(rgcn, in0, (32,) * L, R, NB, 0.0, mb)
    with torch.no_grad():
        for c in ref.convs:
            c.bias.uniform_(-0.3, 0.3)
        for p in ref.parameters():
            p.copy_(p.float().double())
    ref = pyg_restated.set_formulation(ref.double().eval(), "transform")
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    with torch.no_grad():
        out, cs = ref(tb["x"], tb["edge_index"], tb["edge_type"], None, None, return_states=True)
        cs = cs.float().double()
        x = tb["x"]
        pre1 = ref.lin1(torch.cat([cs[x[:, 0] == 1], cs[x[:, 1] == 1]], 1))
    saved = dict(states=list(torch.split(cs, [32] * L, 1)), gscale=(pre1 > 0).double(),
                 dpred=(2.0 * (out - tb["y"].view(-1)) * mb).float().double())
    params = {k: v.detach().clone() for k, v in ref.state_dict().items()}
    return params, ob, saved, ref.convs[0].aggr


def raw_rows(params, ob, saved, q, aggr, CL):
    """graph q's CL partial raw rows [CL, raw count] in fp32: CTA c's row holds the terms of the nodes it owns"""
    sub, sv = eb.graph_view(ob, saved, q)
    g = eb.Graph(sub)
    dpres = []
    eb.backward(params, g, sv, aggr, False, 0.0, dpres=dpres)
    L = len(dpres)
    att_n, basis_n = eb.conv_names(params)[:2]
    R = params["convs.0." + att_n].shape[0]
    in0 = g.x.shape[1]
    n = g.x.shape[0]
    cnt = own_counts(n, CL)
    lo = np.concatenate([[0], np.cumsum(cnt)])
    rows = np.zeros((CL, raw_off(R, in0, L)), np.float64)
    for l in range(L):
        fin = in0 if l == 0 else 32
        inp = a4(fin)
        W = torch.einsum("rb,bio->rio", params["convs.%d.%s" % (l, att_n)],
                         params["convs.%d.%s" % (l, basis_n)]).requires_grad_(True)
        root = params["convs.%d.root" % l].clone().requires_grad_(True)
        bias = params["convs.%d.bias" % l].clone().requires_grad_(True)
        hin = g.x if l == 0 else sv["states"][l - 1]
        pre = eb.layer_pre(hin, [torch.eye(R, dtype=torch.float64), W, root, bias], g, aggr)
        for c in range(CL):
            mask = torch.zeros(n, 1, dtype=torch.float64)
            mask[lo[c]:lo[c + 1]] = 1.0
            dW, dr, db = torch.autograd.grad(pre, [W, root, bias], dpres[l] * mask, retain_graph=True)
            blk = np.zeros((R + 1, inp, 32))
            blk[:R, :fin] = dW.numpy()
            blk[R, :fin] = dr.numpy()
            o = raw_off(R, in0, l)
            rows[c, o:o + (R + 1) * inp * 32] = blk.reshape(-1)
            rows[c, o + (R + 1) * inp * 32:o + (R + 1) * inp * 32 + 32] = db.numpy()
    return rows.astype(f32)


def emulate(gp, params, R, NB, in0, L, slip=None):
    """k_pair_grad_raw of one graph on its partial rows ``gp`` [CL, raw count] fp32: {state_dict name: fp32 array}.
    ``slip`` plants one of the kernel mistakes the bound must catch"""
    CL = gp.shape[0]
    att_n, basis_n = eb.conv_names(params)[:2]
    out = {}
    for l in range(L):
        fin = in0 if l == 0 else 32
        inp = a4(fin)
        stride = fin if slip == "in_for_inp" and l == 0 else inp
        nq = CL - 1 if slip == "drop_last_cta" else CL
        row = gp[:, raw_off(R, in0, l):]
        idx = (np.arange(R + 1)[:, None, None] * stride + np.arange(fin)[None, :, None]) * 32 + np.arange(32)
        dWs = np.zeros((R + 1, fin, 32), f32)
        for q in range(nq):                            # ranks in order
            dWs = dWs + row[q][idx]
        at = params["convs.%d.%s" % (l, att_n)].numpy().astype(f32).reshape(-1)
        a = at.reshape(NB, R).T if slip == "att_bR" else at.reshape(R, NB)
        bs = params["convs.%d.%s" % (l, basis_n)].numpy().astype(f32)         # [NB, in, 32]
        dbasis = np.zeros((NB, fin, 32), f32)
        for r in range(R):                             # fmaf chain over r
            dbasis = _fma(np.broadcast_to(a[r][:, None, None], dbasis.shape), dWs[r][None], dbasis)
        datt = np.zeros((R, NB), f32)
        for k in range(fin):                           # per k: fmaf chain over j, then datt += s
            s = np.zeros((R, NB), f32)
            for j in range(32):
                s = _fma(dWs[:R, k, j][:, None], np.broadcast_to(bs[:, k, j][None, :], (R, NB)), s)
            datt = s if slip == "datt_last_k" else datt + s
        root = dWs[R - 1] if slip == "root_from_R_minus_1" else dWs[R]
        lb = l - 1 if slip == "bias_prev_layer" and l > 0 else l
        ob_ = raw_off(R, in0, lb) + (R + 1) * a4(in0 if lb == 0 else 32) * 32
        bias = np.zeros(32, f32)
        for q in range(nq):
            bias = bias + gp[q, ob_:ob_ + 32]
        out.update({"convs.%d.%s" % (l, att_n): datt, "convs.%d.%s" % (l, basis_n): dbasis, "convs.%d.root" % l: root,
                    "convs.%d.bias" % l: bias})
    return out


def _ratio(params, ob, saved, q, aggr, got):
    grads, mgrads, _, _ = eb.pair_terms(params, ob, saved, q, aggr)
    keys = sorted(got)
    cat = lambda d: torch.cat([torch.as_tensor(np.asarray(d[k], np.float64)).reshape(-1) for k in keys])  # noqa: E731
    return eb.ratio(cat(got), cat(grads), cat(mgrads))


CASES = [  # in0, L, R, NB, CL, rgcn
    (6, 4, 5, 2, 2, "pyg-1.4"), (4, 2, 12, 4, 4, "pyg-1.4"), (8, 1, 1, 2, 3, "pyg-2"), (4, 8, 2, 4, 1, "pyg-1.4")]


@pytest.mark.parametrize("in0,L,R,NB,CL,rgcn", CASES)
def test_emulation_within_the_bound(in0, L, R, NB, CL, rgcn):
    params, ob, saved, aggr = _setup(in0, L, R, NB, rgcn)
    worst = 0.0
    for q in range(3):
        gp = raw_rows(params, ob, saved, q, aggr, CL)
        r, pad, _ = _ratio(params, ob, saved, q, aggr, emulate(gp, params, R, NB, in0, L))
        assert pad == 0
        worst = max(worst, r)
    print("emulated k_pair_grad_raw in0 %d L %d R %d NB %d CL %d: largest err/(u M) %.3f" % (in0, L, R, NB, CL, worst))
    assert worst <= eb.KAPPA["grad"]


SLIPS = ["in_for_inp", "att_bR", "drop_last_cta", "datt_last_k", "root_from_R_minus_1", "bias_prev_layer"]


@pytest.fixture(scope="module")
def slip_case():
    """in0 = 6 (inp 8), L 4, R 5, NB 2, CL 2: every planted slip stays in bounds of the rows it reads"""
    params, ob, saved, aggr = _setup(6, 4, 5, 2)
    return params, ob, saved, aggr, [raw_rows(params, ob, saved, q, aggr, 2) for q in range(3)]


@pytest.mark.parametrize("slip", SLIPS)
def test_planted_slips_exceed_the_bound(slip, slip_case):
    params, ob, saved, aggr, gps = slip_case
    worst = max(_ratio(params, ob, saved, q, aggr, emulate(gp, params, 5, 2, 6, 4, slip))[0]
                for q, gp in enumerate(gps))
    print("slip %s: largest err/(u M) %.3g" % (slip, worst))
    assert worst >= 100 * eb.KAPPA["grad"], (slip, worst)
