"""Per-element fp32 error bounds (tests/error_bounds.py) of the per-pair gradients (igmc_pair_seed and igmc_pair_grad,
csrc/influence.cu), on every kernel plan and in the regimes their assembly branches on.

Each case declares what it is next to its builders: the plan, CTAs per graph, raw or row assembly, R, NB, L, in0, the
RGCN layer, the seed (loss with y, or score), multiply_by and the regimes it claims.  The test builds a fresh model
from that metadata, runs ``InferenceEngine.pair_gradients`` on P <= B pairs (one batch: when it finishes, the model's
train workspace holds that batch's forward and backward) and asserts that the model and the batch enter every claimed
regime.  Against the kernel's own inputs (the saved states, hid_gscale, the engine's dpred buffer and the oracle batch
of the same pairs, asserted equal to the engine's) it checks:

* the seed bit for bit: fp32(fp32(2 fp32(pred - y)) multiply_by) (loss), multiply_by (score), 0 for padding graphs;
* the conv block of every pair per element within KAPPA["grad"] u M of ``backward`` on that graph alone, exactly 0
  where M == 0, no NaN, no branch mismatch;
* the readout block bit for bit from the kernel's own factors (d lin1.weight = dhid (x) feat, d lin1.bias = dhid,
  d lin2.weight = dpred hid, d lin2.bias = dpred), feat bit for bit the two target state rows, dhid within
  KAPPA["dhid"], hid within KAPPA["hid"] of relu(lin1 feat + b);
* no write outside the pairs' rows (NaN guard rows around the output; a padded tail never writes).

Separately: an influence training pass leaves the padding rows of its per-batch conv / factor buffers exactly 0, and
with K = 3 checkpoints every slice is bit-identical to a run on that checkpoint alone, which is itself bounded against
that checkpoint's parameters.  tests/test_pair_grad_bounds_coverage.py checks the coverage of the cases without a
GPU."""
import os
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from oracle import extract_np
from tests import error_bounds as eb
from tests.helpers import batch_equal

pytestmark = pytest.mark.gpu

L2 = _lib.plan_l2


# ---- data: dict(A, u, v, h, mnph) ----------------------------------------------------------------------------------
def _with_cold_start(A):
    import scipy.sparse as ssp
    return ssp.csr_matrix(ssp.bmat([[A, None], [None, ssp.csr_matrix((1, 1), dtype=A.dtype)]]), dtype=A.dtype)


def _synth(R, h=1, mnph=30, n=8, cold=False, seed=3):
    """the first n rated pairs of a 120 x 90 synthetic matrix with R rating levels (mnph 30, h 1: n_cap 62); ``cold``:
    one more user and item, neither rated, and their pair last"""
    from igmc_b200.data import build_adj, synth_ratings
    u, v, lab = synth_ratings(120, 90, 2500, num_classes=R, seed=seed)
    A = build_adj(u, v, lab, 120, 90)
    u, v = u[:n], v[:n]
    if cold:
        A = _with_cold_start(A)
        u, v = np.append(u[:n - 1], 120), np.append(v[:n - 1], 90)
    return dict(A=A, u=u, v=v, h=h, mnph=mnph)


def _degenerate(n=None):
    """the mixed batch of tests/test_gpu_regimes.py: 2-node subgraphs without edges (isolated and cold-start pairs),
    targets without in-edges and 202-node subgraphs (mnph 100)"""
    from tests.test_gpu_regimes import _degenerate_matrix, _mixed_pairs
    A, pairs = _degenerate_matrix()
    sel = _mixed_pairs(pairs)[:n]
    return dict(A=A, u=np.array([p[0] for p in sel]), v=np.array([p[1] for p in sel]), h=1, mnph=100)


def _ml100k_402():
    """four pairs of the heaviest ml_100k* users and items at mnph 200: up to 402-node subgraphs"""
    from igmc_b200.data import make_synthetic_dataset
    A = make_synthetic_dataset("ml_100k", seed=0)["adj_train"]
    du, di = np.diff(A.indptr), np.diff(A.tocsc().indptr)
    coo = A.tocoo()
    k = np.argsort(-(du[coo.row] + di[coo.col]), kind="stable")[:4]
    return dict(A=A, u=coo.row[k].astype(np.int64), v=coo.col[k].astype(np.int64), h=1, mnph=200)


# ---- regimes: name -> check(m, eng, b, ob, tags) -------------------------------------------------------------------
def _sizes(ob):
    return np.bincount(ob["batch"], minlength=ob["num_graphs"])


def _edges(ob):
    return np.bincount(ob["batch"][ob["edge_index"][1]], minlength=ob["num_graphs"])


def _cold_start(m, eng, b, ob, tags):
    assert np.any((_sizes(ob) == 2) & (_edges(ob) == 0) & (tags >= 0))


def _mixed(m, eng, b, ob, tags):
    _cold_start(m, eng, b, ob, tags)
    indeg = np.bincount(ob["edge_index"][1], minlength=len(ob["x"]))
    target = (ob["x"][:, 0] == 1) | (ob["x"][:, 1] == 1)
    assert np.any(target & (indeg == 0)) and _sizes(ob).max() == 202


def _large_pre_activations(m, eng, b, ob, tags):
    """conv parameters x4: more than 2 % of the states in tanh's flat part (|h| > 0.9; none unscaled)"""
    st = m._workspace(b, True)["states"][:len(ob["x"])]
    assert float((st.abs() > 0.9).double().mean()) > 0.02


REGIME_CHECKS = {
    "cold_start": _cold_start,
    "mixed_degenerate": _mixed,
    "batch_of_one": lambda m, eng, b, ob, tags: b.num_graphs == 1,
    "padded_tail": lambda m, eng, b, ob, tags: bool(np.any(tags < 0)) and bool(np.any(tags >= 0)),
    "large_pre_activations": _large_pre_activations,
    "large_subgraphs": lambda m, eng, b, ob, tags: b._priv["n_cap"] == 402 and _sizes(ob).max() > 300,
    "multiply_by": lambda m, eng, b, ob, tags: m.multiply_by not in (0, 1),
}


# ---- cases --------------------------------------------------------------------------------------------------------
def case(data, plan, R=5, NB=4, L=4, in0=4, rgcn="pyg-1.4", seed="loss", mb=1, B=None, n_cap=62, scale=1.0,
         regimes=()):
    """``B``: the engine's batch size (default: the number of pairs); ``scale``: conv parameters multiplied by it"""
    return dict(data=data, plan=plan, ctas=_lib.ctas_per_graph(plan), assembly="raw" if _lib.is_rs(plan) else "row",
                R=R, NB=NB, L=L, in0=in0, rgcn=rgcn, seed=seed, mb=mb, B=B, n_cap=n_cap, scale=scale,
                regimes=tuple(regimes) + (("multiply_by",) if mb not in (0, 1) else ()))


CASES = {
    # raw assembly (k_pair_grad_raw): every cluster plan at R = 1 and R = 12 (dWs[13], 48 att entries)
    **{"R1_nb%d_plan%d" % (nb, p): case(lambda: _synth(1), p, R=1, NB=nb, seed=s)
       for p, nb, s in ((1, 2, "loss"), (2, 4, "score"), (3, 2, "loss"), (4, 4, "score"))},
    **{"R12_nb%d_plan%d" % (nb, p): case(lambda: _synth(12), p, R=12, NB=nb, seed=s)
       for p, nb, s in ((1, 4, "score"), (2, 2, "loss"), (3, 4, "loss"), (4, 4, "loss"))},
    "R2_nb4_plan2": case(lambda: _synth(2), 2, R=2),
    "R5_nb2_plan1": case(lambda: _synth(5), 1, NB=2, seed="score"),
    "R8_nb2_plan4": case(lambda: _synth(8), 4, R=8, NB=2),
    # layer counts (raw offsets, factor-row width) and input widths (layer 0 padded to a4(in0))
    "L1_plan2": case(lambda: _synth(5), 2, L=1),
    "L1_plan3": case(lambda: _synth(5), 3, L=1, seed="score"),
    "L8_plan1": case(lambda: _synth(5), 1, L=8, seed="score"),
    "L8_plan4_nb2": case(lambda: _synth(5), 4, L=8, NB=2),
    "in6_plan1": case(lambda: _synth(5, h=2, mnph=10), 1, in0=6, n_cap=42),
    "in6_plan4_nb2": case(lambda: _synth(5, h=2, mnph=10), 4, in0=6, NB=2, n_cap=42, seed="score"),
    "in8_plan2": case(lambda: _synth(5, h=3, mnph=10), 2, in0=8, n_cap=62, seed="score"),
    "in8_plan3_R12": case(lambda: _synth(12, h=3, mnph=10), 3, R=12, in0=8, n_cap=62),
    "pyg2_plan2": case(lambda: _synth(5), 2, rgcn="pyg-2"),
    "pyg2_plan4_score": case(lambda: _synth(5), 4, rgcn="pyg-2", seed="score"),
    "mb2_plan1_score": case(lambda: _synth(5), 1, mb=2, seed="score"),
    "mb3_plan4": case(lambda: _synth(5), 4, mb=3),
    "scaled4_plan2": case(lambda: _synth(5), 2, scale=4.0, regimes=("large_pre_activations",)),
    "scaled4_plan4_score": case(lambda: _synth(5), 4, scale=4.0, seed="score", regimes=("large_pre_activations",)),
    "ml100k_402_plan4": case(_ml100k_402, 4, n_cap=402, regimes=("large_subgraphs",)),
    # row assembly (k_pair_grad_rows): plan 0 and the L2 plan with 1, 2, 4 and 8 CTAs per subgraph
    "R13_plan0": case(lambda: _synth(13), 0, R=13),
    "R13_plan0_score_nb2": case(lambda: _synth(13), 0, R=13, NB=2, seed="score"),
    "L1_in6_plan0": case(lambda: _synth(5, h=2, mnph=10), 0, L=1, in0=6, n_cap=42),
    "L8_in8_plan0_score": case(lambda: _synth(5, h=3, mnph=10), 0, L=8, in0=8, n_cap=62, seed="score"),
    "l2x1": case(lambda: _synth(5), L2(1)),
    "l2x1_score_L8": case(lambda: _synth(5), L2(1), L=8, seed="score"),
    "l2x2_R71_nb2_score": case(lambda: _synth(71), L2(2), R=71, NB=2, seed="score"),
    "l2x2_L1_in8": case(lambda: _synth(5, h=3, mnph=10), L2(2), L=1, in0=8, n_cap=62),
    "l2x4_pyg2": case(lambda: _synth(5), L2(4), rgcn="pyg-2"),
    "l2x4_in6_nb2_score": case(lambda: _synth(5, h=2, mnph=10), L2(4), in0=6, NB=2, n_cap=42, seed="score"),
    "l2x8": case(lambda: _synth(5), L2(8)),
    "l2x8_pyg2_score_mb2": case(lambda: _synth(5), L2(8), rgcn="pyg-2", seed="score", mb=2),
    # degenerate batches
    "cold_start_plan2": case(lambda: _synth(5, cold=True), 2, regimes=("cold_start",)),
    "cold_start_plan0_score": case(lambda: _synth(5, cold=True), 0, seed="score", regimes=("cold_start",)),
    "mixed_plan4": case(_degenerate, 4, n_cap=202, regimes=("mixed_degenerate",)),
    "mixed_l2x2_score": case(_degenerate, L2(2), n_cap=202, seed="score", regimes=("mixed_degenerate",)),
    "one_pair_plan1_score": case(lambda: _synth(5, n=1), 1, seed="score", regimes=("batch_of_one",)),
    "one_pair_plan0": case(lambda: _synth(5, n=1), 0, regimes=("batch_of_one",)),
    "tail_plan2": case(lambda: _synth(5, n=5), 2, B=8, regimes=("padded_tail",)),
    "tail_plan3_score": case(lambda: _synth(5, n=3), 3, B=4, seed="score", regimes=("padded_tail",)),
    "tail_l2x4": case(lambda: _synth(5, n=5), L2(4), B=8, regimes=("padded_tail",)),
}

# K = 3 checkpoints (test_checkpoints_are_each_their_own_run)
CHECKPOINT_CASES = {
    "K3_plan2": case(lambda: _synth(5, n=6), 2, B=8, regimes=("padded_tail",)),
    "K3_plan0_score": case(lambda: _synth(13), 0, R=13, seed="score"),
}


def build_model(c, device="cuda", seed=0):
    """the IGMC a case declares (its own initialisation under ``seed``, PyG 2 biases drawn, conv parameters scaled)"""
    from igmc_b200.models import IGMC
    torch.manual_seed(seed)
    m = IGMC(c["in0"], latent_dim=[32] * c["L"], num_relations=c["R"], num_bases=c["NB"], regression=True,
             rgcn=c["rgcn"], multiply_by=c["mb"])
    with torch.no_grad():
        for conv in m.convs:
            if c["rgcn"] == "pyg-2":
                conv.bias.uniform_(-0.3, 0.3)
            for p in conv.parameters():
                p.mul_(c["scale"])
    m = m.to(device)
    m.kernel_plan = c["plan"]
    return m


def _labels(d, R, seed):
    return None if seed == "score" else \
        np.random.default_rng(len(d["u"])).integers(1, R + 1, len(d["u"])).astype(np.float32)


def _run(m, d, y, B, checkpoints=None, sample_seed=5):
    """one pair_gradients run of the engine with NaN guard rows around its output: (G [K, P, PC'], engine, batch,
    oracle batch, tags); asserts that the guard rows are untouched and the oracle batch equals the engine's"""
    u, v, A = d["u"], d["v"], d["A"]
    P = len(u)
    eng = rc.InferenceEngine(m, A, h=d["h"], max_nodes_per_hop=d["mnph"], batch_size=B, sample_seed=sample_seed,
                             checkpoints=checkpoints)
    try:
        eng.start_pair_gradients(u, v, y)
        K, _, W = eng.run["out"].shape
        guard = torch.full((K, P + 2, W), float("nan"), device="cuda")
        eng.run["out"] = guard[:, 1:P + 1]
        assert eng.run["steps"] == 1
        while eng.step():
            pass
        G = eng.finish()
        torch.cuda.synchronize()
    finally:
        eng.close()
    assert torch.isnan(guard[:, 0]).all() and torch.isnan(guard[:, P + 1]).all()     # no write outside the rows
    b = eng.batches[0]
    tags = eng.slots[0]["tag"].cpu().numpy()
    ni = A.shape[1]
    pu = np.concatenate([u, np.repeat(u[-1:], B - P)]).astype(np.int64)
    pv = np.concatenate([v, np.repeat(v[-1:], B - P)]).astype(np.int64)
    assert np.array_equal(tags, np.where(np.arange(B) < P, np.arange(B), -1))
    R = m.num_relations
    ob = extract_np.extract_batch(extract_np.RatingCSR(A), pu, pv, np.zeros(B, np.int64),
                                  np.arange(1, R + 1, dtype=np.float32), d["h"], 1.0, d["mnph"], seed=sample_seed,
                                  pair_ids=pu * ni + pv)
    res = batch_equal(b, ob)
    assert all(res.values()), res
    return G, eng, b, ob, tags


def _check_run(name, m, G, eng, b, ob, tags, y, params=None, k=0):
    """every check of the module docstring on checkpoint slice ``k`` of a finished run (the model's train workspace
    holds its forward and backward); returns {quantity: largest ratio}"""
    ws = m._workspace(b, True)
    B, PC = b.num_graphs, m._cmodel.conv_param_count
    N = len(ob["x"])
    saved = eb.device_saved(m, ws, N, True)
    dpred = eng.preds[0][:B]
    saved["dpred"] = dpred.double().cpu()
    mb = torch.tensor(float(m._cmodel.multiply_by), dtype=torch.float32, device="cuda")
    pred = ws["pred"][:B]
    # the seed, bit for bit
    real = torch.from_numpy(tags >= 0).cuda()
    if y is None:
        want = mb.expand(B)
    else:
        yy = torch.from_numpy(y).cuda()[torch.from_numpy(np.maximum(tags, 0)).cuda()]
        want = ((pred - yy) * 2.0) * mb
    want = torch.where(real, want, torch.zeros_like(want))
    assert torch.equal(dpred, want), (name, dpred, want)
    aggr = "mean_per_relation" if m.rgcn == "pyg-2" else "mean_all"
    names = {id(p): n for n, p in m.named_parameters()}
    ent = {names[id(p)]: e for e, (_, _, p) in zip(m._layout, m._named_order())}
    st = ws["states"]
    nptr = np.concatenate([[0], np.cumsum(_sizes(ob))])
    worst, bad = {}, []
    for q in range(B):
        t = int(tags[q])
        if t < 0:
            continue
        row = G[k, t]
        dhid, feat, hid = ws["dhid"][q], ws["feat"][q], ws["hid"][q]
        # the factors: feat is the two target rows of the saved states
        xq = ob["x"][nptr[q]:nptr[q + 1]]
        ui, vi = nptr[q] + int(np.nonzero(xq[:, 0] == 1)[0][0]), nptr[q] + int(np.nonzero(xq[:, 1] == 1)[0][0])
        assert torch.equal(feat, torch.cat([st[ui], st[vi]])), (name, q)
        # the readout block, bit for bit from the factors
        assert torch.equal(m._pview(row, ent["lin1.weight"]), dhid[:, None] * feat[None, :]), (name, q)
        assert torch.equal(m._pview(row, ent["lin1.bias"]), dhid), (name, q)
        assert torch.equal(m._pview(row, ent["lin2.weight"])[0], dpred[q] * hid), (name, q)
        assert torch.equal(m._pview(row, ent["lin2.bias"])[0], dpred[q]), (name, q)
        res = eb.check_pair(m, ob, saved, q, row[:PC], aggr, params, dhid=dhid, hid=hid)
        bad += [(q,) + v for v in eb.violations(res)]
        for key, val in res.items():
            if key != "branches":
                worst[key] = max(worst.get(key, 0.0), val[0])
    for key, r in sorted(worst.items()):
        print("pair grad bounds %-24s %-5s err/(uM) %9.3f  kappa %4g" % (name, key, r, eb.kappa_of(key)))
    assert not bad, (name, bad)
    return worst


def _enter(c, m, d):
    """the model as declared; returns the labels of the run"""
    assert (len(m.convs), m.num_relations, m.num_bases, m.rgcn, m.num_features) == \
        (c["L"], c["R"], c["NB"], c["rgcn"], c["in0"])
    assert 2 * d["h"] + 2 == c["in0"]
    return _labels(d, c["R"], c["seed"])


def _claims(c, m, eng, b, ob, tags):
    assert m._plan(b) == c["plan"] and b._priv["n_cap"] == c["n_cap"]
    assert _lib.ctas_per_graph(m._workspace(b, True)["cluster"]) == c["ctas"]
    assert _lib.is_rs(m._workspace(b, True)["cluster"]) == (c["assembly"] == "raw")
    for regime in c["regimes"]:
        assert REGIME_CHECKS[regime](m, eng, b, ob, tags) is not False, regime


@pytest.mark.parametrize("name", list(CASES))
def test_pair_grad_bounds(name):
    c = CASES[name]
    d = c["data"]()
    m = build_model(c)
    y = _enter(c, m, d)
    B = c["B"] or len(d["u"])
    G, eng, b, ob, tags = _run(m, d, y, B)
    assert G.shape == (1, len(d["u"]), m._cmodel.param_count)
    _claims(c, m, eng, b, ob, tags)
    _check_run(name, m, G, eng, b, ob, tags, y)


@pytest.mark.parametrize("name", list(CHECKPOINT_CASES))
def test_checkpoints_are_each_their_own_run(name):
    """K = 3: slice j of the run is bit-identical to a run on checkpoint j alone, which is bounded against checkpoint
    j's parameters (a prepared-weight or parameter swap between checkpoints fails either)"""
    c = CHECKPOINT_CASES[name]
    d = c["data"]()
    m = build_model(c)
    y = _enter(c, m, d)
    B = c["B"] or len(d["u"])
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for j in range(3):
            paths.append(os.path.join(tmp, "ck%d.pth" % j))
            torch.save(build_model(c, seed=j + 1).state_dict(), paths[-1])
        G, eng, b, ob, tags = _run(m, d, y, B, checkpoints=paths)
        _claims(c, m, eng, b, ob, tags)
        assert G.shape[0] == 3
        for j, p in enumerate(paths):
            Gj, eng, b, ob, tags = _run(m, d, y, B, checkpoints=[p])
            assert torch.equal(Gj[0], G[j]), (name, j)
            _check_run("%s[%d]" % (name, j), m, Gj, eng, b, ob, tags, y, params=torch.load(p))


@pytest.mark.parametrize("plan", [2, L2(2)])
def test_influence_training_pass_padding_rows_are_zero(plan):
    """a self-influence pass over fewer pairs than the batch: the padding rows of its per-batch conv and factor
    buffers (NaN before the pass) are exactly 0, the real rows finite"""
    c = case(None, plan)
    d = _synth(5, n=5)
    m = build_model(c)
    y = _labels(d, 5, "loss")
    eng = rc.InferenceEngine(m, d["A"], h=1, max_nodes_per_hop=30, batch_size=8, sample_seed=5)
    try:
        eng.start_self_influence((d["u"], d["v"], y))
        bufs = eng.run["bufs"]
        bufs["conv"].fill_(float("nan"))
        bufs["fac"].fill_(float("nan"))
        while eng.step():
            pass
        s = eng.finish()
        torch.cuda.synchronize()
    finally:
        eng.close()
    assert m._plan(eng.batches[0]) == plan
    assert torch.isfinite(s).all()
    for k in ("conv", "fac"):
        assert torch.isfinite(bufs[k][:5]).all(), k
        assert torch.equal(bufs[k][5:], torch.zeros_like(bufs[k][5:])), k
