"""Explaining predicted ratings by the nodes of their enclosing subgraphs on the GPU (igmc_b200/recommend.py
explain_nodes, csrc/explain.cu).

* every occluded score equals the eval forward of a foreign batch built from the subgraph with every rating of the
  node filtered out of edge_index / edge_type (its node kept), on the engine's plan and node capacity: bit for bit on
  plans 2, 4, 0 (R = 13) and L2, h = 2, rgcn="pyg-2" and DGCNN_RS; plan 1 within 8 ulps of the pair's largest score;
* the listed nodes, labels and rating counts are the subgraph's; the score is predict_pairs bit for bit; a cold-start
  pair owns no position;
* a node with exactly one rating has explain_pairs' delta of that rating, bit for bit;
* the occluded scores are within 1e-4 RMSE of the fp64 restated forward on the oracle's subgraphs;
* order, top-m and padding; results do not depend on B or graph replay;
* checkpoints, graph updates and steady-state steps without a host synchronisation."""
import os
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.util_functions import Batch, RatingGraph
from oracle import extract_np, pyg_restated
from tests import pyg2_oracle
from tests import support
from tests.test_gpu_explain import _expected_order, _pairs, _subgraph, _with_cold_start
from tests.test_gpu_graph_update import _apply_scipy

pytestmark = pytest.mark.gpu


def _run(eng, u, v, m=None):
    """(NodeExplanation, occluded scores [T] in position order) of one engine run"""
    eng.start_explain_nodes(u, v, m)
    while eng.step():
        pass
    occ = eng.run["occ"]
    return eng.finish(), occ


def _positions(x):
    """the subgraph's positions: its nodes with node_label >= 2 (x is the one-hot of node_label), in order"""
    return torch.nonzero(x.argmax(1) >= 2).flatten()


def _node_masked_forward(model, sub, plan, n_cap, B=256):
    """eval scores [N - 2] of the subgraph without the ratings of the node at position j, for every j: foreign
    batches of copies with every directed edge that has the node as an endpoint filtered out (the node itself kept),
    on the engine's kernel plan and node capacity"""
    x, ei, et, _ = sub
    n = x.shape[0]
    pos = _positions(x)
    out = []
    own = model.kernel_plan
    model.kernel_plan = plan
    model.eval()
    try:
        with torch.no_grad():
            for j0 in range(0, len(pos), B):
                ps = pos[j0:j0 + B]
                G = len(ps)
                keep = (ei[0][None, :] != ps[:, None]) & (ei[1][None, :] != ps[:, None])      # [G, E]
                g_of, e_of = keep.nonzero(as_tuple=True)
                b = Batch.from_arrays(x.repeat(G, 1), ei[:, e_of] + g_of * n, et[e_of],
                                      torch.arange(G, device="cuda").repeat_interleave(n), torch.zeros(G),
                                      num_graphs=G)
                b._priv["n_cap"] = n_cap
                out.append(model(b).clone())
    finally:
        model.kernel_plan = own
    return torch.cat(out) if out else torch.zeros(0, device="cuda")


def _records(sub):
    """per position of the subgraph: its global id, label and rating count"""
    x, ei, _, gid = sub
    pos = _positions(x)
    lab = x.argmax(1)
    deg = torch.zeros(x.shape[0], dtype=torch.int64, device="cuda").index_add_(0, ei[0], torch.ones_like(ei[0]))
    return np.stack([t[pos].cpu().numpy() for t in (gid.long(), lab, deg)])


# ---- 1. occluded scores == node-filtered foreign forward ---------------------------------------------------------------
CASES = {
    # name: (dataset, h, mnph, model kwargs, forced kernel plan, expected plan, small pairs)
    "plan 2 ml_1m": ("ml_1m", 1, 100, {}, "auto", 2, False),
    "plan 1 ml_1m": ("ml_1m", 1, 100, {}, 1, 1, False),
    "plan 4 ml_100k": ("ml_100k", 1, 200, {}, "auto", 4, False),
    "plan 0 R=13": ("r13", 1, 50, {}, "auto", 0, False),
    "L2 plan ml_100k uncapped": ("ml_100k", 1, None, {}, "auto", "l2", True),
    "h=2": ("ml_1m", 2, 20, {}, "auto", None, False),
    "pyg-2": ("ml_1m", 1, 100, dict(rgcn="pyg-2"), "auto", 2, False),
    "DGCNN_RS": ("ml_1m", 1, 100, dict(dgcnn=True), "auto", None, False),
}

INEXACT = {"plan 1 ml_1m"}      # held to 8 ulps, as test_gpu_explain holds explain_pairs on plan 1


@pytest.mark.parametrize("name", list(CASES))
def test_occluded_scores_equal_the_node_filtered_forward(name):
    dsn, h, mnph, kw, force, plan, small = CASES[name]
    A0 = support.adj(dsn)
    R = 13 if dsn == "r13" else 5
    A = _with_cold_start(A0)
    m = support.model(R, h=h, **kw, pyg2_bias=True)
    m.kernel_plan = force
    u, v = _pairs(A, small)
    B, seed = 64, 7
    eng = rc.InferenceEngine(m, A, h=h, max_nodes_per_hop=mnph, batch_size=B, sample_seed=seed)
    ex, occ = _run(eng, u, v)
    eng.close()
    cl = next(iter(m._plans.values()))
    if plan == "l2":
        assert _lib.l2_csize(cl) > 0
    elif plan is not None:
        assert cl == plan, (name, cl)
    base = rc.predict_pairs(m, A, u, v, h=h, max_nodes_per_hop=mnph, batch_size=B, sample_seed=seed)
    assert torch.equal(ex.score, base), name
    off = ex.offsets.cpu().numpy()
    nn = ex.num_nodes.cpu().numpy()
    assert np.array_equal(np.diff(off), nn) and nn[2] == 0 and nn[0] > 0 and nn[1] > 0   # cold start: no position
    score, occ = ex.score.cpu().numpy(), occ.cpu().numpy()
    delta_of_pos = np.concatenate([occ[off[q]:off[q + 1]] - score[q] for q in range(3)]).astype(np.float32)
    fields = [t.cpu().numpy() for t in (ex.node, ex.label, ex.ratings, ex.delta)]
    for q in range(2):
        sub, n_cap = _subgraph(A, R, int(u[q]), int(v[q]), h, mnph, seed)
        assert sub[0].shape[0] - 2 == nn[q]
        rec = _records(sub)
        seg = slice(off[q], off[q + 1])
        o = _expected_order(off[q], off[q + 1], delta_of_pos) - off[q]       # j of every listed entry
        for f in range(3):
            assert np.array_equal(fields[f][seg], rec[f][o]), (name, q, f)
        assert np.array_equal(fields[3][seg], delta_of_pos[seg][o], equal_nan=True), (name, q)
        want = _node_masked_forward(m, sub, cl, n_cap).cpu().numpy()
        got = occ[seg]
        if name in INEXACT:
            bound = 8 * float(np.spacing(np.abs(want).max().astype(np.float32)))
            assert float(np.abs(got - want).max()) <= bound, (name, q, float(np.abs(got - want).max()), bound)
        else:
            bad = int((got != want).sum())
            assert bad == 0, (name, q, bad, float(np.abs(got - want).max()))


# ---- 2. a node with one rating is that rating's explain_pairs entry ------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, dict(dgcnn=True)], ids=["IGMC", "DGCNN_RS"])
def test_single_rating_node_is_the_rating_delta(kw):
    A = support.adj("ml_100k")
    m = support.model(5, **kw, pyg2_bias=True)
    u, v = np.array([3, 40, 100]), np.array([7, 50, 2])
    args = dict(max_nodes_per_hop=50, batch_size=64, sample_seed=3)
    nd = rc.explain_nodes(m, A, u, v, **args)
    ed = rc.explain_pairs(m, A, u, v, **args)
    assert torch.equal(nd.score, ed.score)
    checked = 0
    for q in range(3):
        a0, a1 = int(nd.offsets[q]), int(nd.offsets[q + 1])
        b0, b1 = int(ed.offsets[q]), int(ed.offsets[q + 1])
        users, items = ed.user[b0:b1].cpu().numpy(), ed.item[b0:b1].cpu().numpy()
        deltas = ed.delta[b0:b1].cpu().numpy()
        for node, lab, r, d in zip(*(t[a0:a1].cpu().numpy() for t in (nd.node, nd.label, nd.ratings, nd.delta))):
            if r != 1:
                continue
            hit = np.flatnonzero(users == node) if lab % 2 == 0 else np.flatnonzero(items == node)
            assert len(hit) == 1, (q, node, lab)
            assert np.float32(d).view(np.int32) == deltas[hit[0]].view(np.int32), (q, node, d, deltas[hit[0]])
            checked += 1
    assert checked > 3, checked


# ---- 3. against the fp64 restated forward ----------------------------------------------------------------------------------
@pytest.mark.parametrize("rgcn", ["pyg-1.4", "pyg-2"])
def test_occluded_scores_against_oracle(rgcn):
    A = _with_cold_start(support.adj("ml_1m"))
    R, mnph, seed = 5, 100, 7
    m = support.model(R, rgcn=rgcn, pyg2_bias=True)
    ref = pyg2_oracle.igmc_ref(rgcn, 4, (32,) * 4, R, 4, 0.0)
    ref.load_state_dict({k: v.double().cpu() for k, v in m.state_dict().items()})
    ref = pyg_restated.set_formulation(ref.double(), "transform").cuda().eval()
    u, v = _pairs(A)
    ex = rc.explain_nodes(m, A, u[:2], v[:2], max_nodes_per_hop=mnph, batch_size=128, sample_seed=seed)
    ni = A.shape[1]
    errs = []
    for q in range(2):
        ob = extract_np.extract_batch(extract_np.RatingCSR(A), u[q:q + 1], v[q:q + 1], np.zeros(1, np.int64),
                                      np.arange(1, R + 1, dtype=np.float32), 1, 1.0, mnph, seed=seed,
                                      pair_ids=u[q:q + 1] * ni + v[q:q + 1])
        sub = ob["subs"][0]
        tb = pyg_restated.to_torch_batch(ob, torch.float64, device="cuda")
        x, ei, et = tb["x"], tb["edge_index"], tb["edge_type"]
        n = x.shape[0]
        nu_ = len(sub["u_nodes"])
        lab = x.argmax(1)
        gid = np.concatenate([sub["u_nodes"], sub["v_nodes"]])
        key = {(int(lab[i]) % 2, int(gid[i])): i for i in range(n) if int(lab[i]) >= 2}
        assert len(key) == n - 2 and nu_ <= n
        o0, o1 = int(ex.offsets[q]), int(ex.offsets[q + 1])
        assert o1 - o0 == n - 2
        ps = torch.as_tensor([key[(int(l) % 2, int(g))] for l, g in zip(ex.label[o0:o1].tolist(),
                                                                          ex.node[o0:o1].tolist())], device="cuda")
        got = (ex.score[q] + ex.delta[o0:o1]).double().cpu().numpy()
        want = np.zeros(len(ps))
        with torch.no_grad():
            for j0 in range(0, len(ps), 128):
                pp = ps[j0:j0 + 128]
                G = len(pp)
                keep = (ei[0][None, :] != pp[:, None]) & (ei[1][None, :] != pp[:, None])
                eig, etg = pyg_restated.dropout_adj(ei.repeat(1, G), et.repeat(G), 1.0, True, keep.reshape(-1))
                eig = eig + torch.repeat_interleave(torch.arange(G, device="cuda") * n, keep.sum(1))[None, :]
                want[j0:j0 + G] = ref(x.repeat(G, 1), eig, etg).cpu().numpy()
        errs.append(got - want)
    rmse = float(np.sqrt(np.mean(np.concatenate(errs) ** 2)))
    print("%s: node-occluded scores vs fp64 oracle RMSE %.2e" % (rgcn, rmse))
    assert rmse <= 1e-4, rmse


# ---- 4. order, top-m, padding, determinism ---------------------------------------------------------------------------------
def test_order_topm_and_determinism():
    A = _with_cold_start(support.adj("ml_1m"))
    m = support.model(5)
    m.kernel_plan = 2                  # the same plan at every batch size
    u, v = _pairs(A)
    results = {}
    for B in (1, 50, 256):
        for use_graph in (True, False):
            eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=B, sample_seed=2, use_graph=use_graph)
            results[(B, use_graph)] = _run(eng, u, v)[0]
            tops = {k: eng.explain_nodes(u, v, k) for k in (1, 10, 256)} if (B, use_graph) == (50, True) else None
            eng.close()
            if tops:
                ex = results[(B, use_graph)]
                off = ex.offsets.cpu().numpy()
                for k, t in tops.items():
                    assert t.node.shape == (3, k) and torch.equal(t.score, ex.score)
                    for q in range(3):
                        n = min(k, off[q + 1] - off[q])
                        for f, pad in (("node", -1), ("label", -1), ("ratings", 0), ("delta", 0)):
                            a, b = getattr(t, f)[q], getattr(ex, f)[off[q]:off[q] + n]
                            assert torch.equal(a[:n], b), (k, q, f)
                            assert (a[n:] == pad).all(), (k, q, f)
    first = results[(50, True)]
    d = first.delta.cpu().numpy()
    off = first.offsets.cpu().numpy()
    for q in range(3):
        a = np.abs(d[off[q]:off[q + 1]])
        assert (np.diff(a[~np.isnan(a)]) <= 0).all() and not np.isnan(a[:int((~np.isnan(a)).sum())]).any()
    assert (first.ratings >= 1).all() and (first.label >= 2).all()
    for key, r in results.items():
        for f in r._fields:
            assert torch.equal(getattr(r, f), getattr(first, f)), (key, f)


def test_validation_and_empty_input():
    A = support.adj("ml_100k")
    m = support.model(5)
    with pytest.raises(IndexError):
        rc.explain_nodes(m, A, [A.shape[0]], [0])
    with pytest.raises(NotImplementedError):
        rc.explain_nodes(m, A, [0], [0], _lib.TOPK_MAX + 1)
    ex = rc.explain_nodes(m, A, [], [])
    assert ex.score.shape == (0,) and ex.offsets.tolist() == [0] and ex.delta.shape == (0,)
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=200, batch_size=50)
    ex = eng.explain_nodes([], [], 3)
    assert ex.node.shape == (0, 3) and ex.offsets.tolist() == [0]
    eng.close()


# ---- 5. checkpoints, graph updates, steady state ---------------------------------------------------------------------------
def test_two_checkpoints_are_the_fp32_mean():
    A = _with_cold_start(support.adj("ml_100k"))
    m = support.model(5)
    u, v = _pairs(A, small=True)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for c in range(2):
            paths.append(os.path.join(tmp, "model_checkpoint%d.pth" % c))
            torch.save(support.model(5, seed=c + 1).state_dict(), paths[-1])
        runs = []
        for ck in (paths, paths[:1], paths[1:]):
            eng = rc.InferenceEngine(m, A, max_nodes_per_hop=200, batch_size=50, checkpoints=ck)
            runs.append(_run(eng, u, v))
            eng.close()
    (ens, occ), (e0, o0), (e1, o1) = runs
    assert torch.equal(ens.score, (e0.score + e1.score) / 2)
    assert torch.equal(occ, (o0 + o1) / 2)
    assert torch.equal(ens.num_nodes, e0.num_nodes)
    assert ens.delta.numel() > 0 and not torch.equal(ens.delta, e0.delta)


def test_engine_explains_nodes_across_updates():
    A = support.adj("ml_1m")
    m = support.model(5)
    g = RatingGraph(A, reserve_nnz=2000)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=64, sample_seed=4)
    rng = np.random.default_rng(5)
    u, v = _pairs(_with_cold_start(A))
    u, v = u[:2], v[:2]
    try:
        eng.explain_nodes(u, v, 10)
        coo = A.tocoo()
        k = rng.choice(A.nnz, 300, replace=False)
        du = np.concatenate([coo.row[k[:150]], rng.integers(0, A.shape[0], 150)])
        dv = np.concatenate([coo.col[k[:150]], rng.integers(0, A.shape[1], 150)])
        dx = np.concatenate([np.zeros(75, np.int64), rng.integers(1, 6, 225)])
        g.update(du, dv, dx)
        A2 = _apply_scipy(A, du, dv, dx, g.shape)
        got = eng.explain_nodes(u, v)
        fresh = rc.InferenceEngine(m, RatingGraph(A2), max_nodes_per_hop=100, batch_size=64, sample_seed=4)
        want = fresh.explain_nodes(u, v)
        fresh.close()
    finally:
        eng.close()
    for f in got._fields:
        assert torch.equal(getattr(got, f), getattr(want, f)), f


def test_steady_state_steps_do_not_sync():
    A = support.adj("ml_1m")
    m = support.model(5)
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=50, sample_seed=1)
    u, v = np.array([11, 12]), np.array([40, 41])
    outs = []
    try:
        for rep in range(2):
            eng.start_explain_nodes(u, v)
            while eng.run["phase"] == "base":
                assert eng.step()
            for _ in range(4):              # eager warm-up and capture of both slots of the occlusion pass
                assert eng.step()
            assert len(eng.graphs) == 2
            torch.cuda.set_sync_debug_mode("error")
            try:
                while eng.step():
                    pass
            finally:
                torch.cuda.set_sync_debug_mode("default")
            outs.append(eng.finish())
            assert int(eng.extractor.err.item()) == 0
    finally:
        eng.close()
    for f in outs[0]._fields:
        assert torch.equal(getattr(outs[0], f), getattr(outs[1], f)), f
