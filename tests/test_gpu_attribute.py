"""Attributing predicted ratings on the GPU (igmc_b200/recommend.py attribute_pairs, igmc_edge_grad in csrc/rgcn_l2.cu).

* every rating's gradient matches fp64 autograd of the weighted restatement (tests/edge_weight_oracle.py) on the
  kernel's own subgraphs, per pair max |got - ref| <= 2e-4 max |ref|: IGMC with both RGCN layers, DGCNN_RS in the
  kernel's SortPooling order, R = 5, 13 and 71, h = 2, ml_1m* without a node cap, B = 1 and a padded tail, a cold-start
  pair and a rated target;
* the score is predict_pairs bit for bit, the listed ratings are explain_pairs', the order is the documented one of
  the engine's own values, top-m truncates and pads, results do not depend on B or graph replay;
* checkpoints, graph updates, and steady-state steps without a host synchronisation."""
import functools
import os
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.data import build_adj, synth_ratings
from igmc_b200.util_functions import Batch, RatingGraph
from tests import edge_weight_oracle as ewo
from tests import pyg2_oracle
from tests import support
from tests.test_gpu_explain import _pairs, _subgraph, _with_cold_start
from tests.test_gpu_graph_update import _apply_scipy

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _r71():
    nu, ni = 300, 250
    u, v, lab = synth_ratings(nu, ni, 6000, 71, seed=6)
    return build_adj(u, v, lab, nu, ni)


def _ref(m, R, h, rgcn, dgcnn):
    F = 2 * h + 2
    ref = pyg2_oracle.dgcnn_rs_ref(rgcn, F, (32, 32, 32, 1), m.k, R, 4, 0.0) if dgcnn else \
        pyg2_oracle.igmc_ref(rgcn, F, (32,) * 4, R, 4, 0.0)
    ref.load_state_dict({k: v.double().cpu() for k, v in m.state_dict().items()})
    return ref.double().cuda().eval()


def _kernel_perm(m, sub):
    """the SortPooling order [1, k] of the L2-plan eval forward of the subgraph alone (node indices, -1 past its end)"""
    x, ei, et, _ = sub
    b = Batch.from_arrays(x, ei, et, torch.zeros(x.shape[0], dtype=torch.int64, device="cuda"), torch.zeros(1),
                          num_graphs=1)
    own = m.kernel_plan
    m.kernel_plan = _lib.plan_l2(1)
    try:
        with torch.no_grad():
            _, saved = m._launch_forward(b, False, m.make_dropout(False))
            return saved["ws"]["sp"]["perm"][:1].clone()
    finally:
        m.kernel_plan = own


def _by_rating(ex, q, sub):
    """pair q's listed (user, item) -> its rating index j in the subgraph's edge_index, and the grads in j order"""
    _, ei, _, gid = sub
    mm = ei.shape[1] // 2
    gid_h, ei_h = gid.cpu().numpy(), ei.cpu().numpy()
    key = {(int(gid_h[ei_h[0, j]]), int(gid_h[ei_h[1, j]])): j for j in range(mm)}
    o0, o1 = int(ex.offsets[q]), int(ex.offsets[q + 1])
    js = np.array([key[(a, b)] for a, b in zip(ex.user[o0:o1].tolist(), ex.item[o0:o1].tolist())], np.int64)
    got = np.zeros(mm)
    got[js] = ex.grad[o0:o1].double().cpu().numpy()
    return js, got


CASES = {
    # name: (dataset, R, h, mnph, model kwargs, batch size)
    "pyg-1.4": ("ml_1m", 5, 1, 100, {}, 64),
    "pyg-2": ("ml_1m", 5, 1, 100, dict(rgcn="pyg-2"), 64),
    "DGCNN_RS": ("ml_1m", 5, 1, 100, dict(dgcnn=True), 64),
    "DGCNN_RS pyg-2": ("ml_1m", 5, 1, 100, dict(dgcnn=True, rgcn="pyg-2"), 64),
    "R=13 padded tail": ("r13", 13, 1, 50, {}, 2),
    "R=71 B=1": ("r71", 71, 1, 50, {}, 1),
    "h=2": ("ml_1m", 5, 2, 20, {}, 64),
    "ml_1m uncapped": ("ml_1m", 5, 1, None, {}, 64),
}


@pytest.mark.parametrize("name", list(CASES))
def test_grad_matches_fp64_autograd(name):
    dsn, R, h, mnph, kw, B = CASES[name]
    A0 = _r71() if dsn == "r71" else support.adj(dsn)
    A = _with_cold_start(A0)
    m = support.model(R, h=h, **kw, pyg2_bias=True)
    u, v = _pairs(A)
    seed = 7
    ex = rc.attribute_pairs(m, A, u, v, h=h, max_nodes_per_hop=mnph, batch_size=B, sample_seed=seed)
    assert m.kernel_plan == "auto"                      # the gradient pass gave the model its plan back
    ne = ex.num_edges.cpu().numpy()
    assert ne[0] > 0 and ne[1] > 0 and ne[2] == 0       # a rated pair, an unrated pair, the cold-start pair
    ref = _ref(m, R, h, kw.get("rgcn", "pyg-1.4"), kw.get("dgcnn", False))
    sizes = []
    for q in range(2):
        sub, _ = _subgraph(A, R, int(u[q]), int(v[q]), h, mnph, seed)
        x, ei, et, gid = sub
        mm = ei.shape[1] // 2
        assert mm == ne[q]
        sizes.append(x.shape[0])
        gid_h, ei_h = gid.cpu().numpy(), ei.cpu().numpy()
        assert not ((gid_h[ei_h[0, :mm]] == u[q]) & (gid_h[ei_h[1, :mm]] == v[q])).any()   # own rating excluded
        extra = {}
        if kw.get("dgcnn"):
            extra = dict(batch=torch.zeros(x.shape[0], dtype=torch.int64, device="cuda"), num_graphs=1,
                         perm=_kernel_perm(m, sub))
        want = ewo.rating_grad(ewo.autograd_edge_grad(ref, x.double(), ei, et, **extra), mm).cpu().numpy()
        js, got = _by_rating(ex, q, sub)
        assert np.array_equal(np.sort(js), np.arange(mm))
        err, scale = float(np.abs(got - want).max()), float(np.abs(want).max())
        print("%s pair %d: %d nodes, %d ratings, max |grad| %.3e, max err %.3e" % (name, q, x.shape[0], mm, scale, err))
        assert scale > 0 and err <= 2e-4 * scale, (name, q, err, scale)
    if name == "ml_1m uncapped":
        assert max(sizes) > 256, sizes                  # beyond what the shared-memory plans hold


def _run(eng, u, v, m=None):
    """(Attribution, gradients [T] in position order, user / item / rating [T] in position order)"""
    eng.start_attribute(u, v, m)
    while eng.step():
        pass
    run = eng.run
    pos = tuple(run[k].clone() for k in ("occ", "user", "item", "rating"))
    return eng.finish(), pos


def test_score_ratings_order_topm_and_determinism():
    A = _with_cold_start(support.adj("ml_1m"))
    m = support.model(5)
    u, v = _pairs(A)
    base = rc.predict_pairs(m, A, u, v, max_nodes_per_hop=100, batch_size=50, sample_seed=2)
    exp = rc.explain_pairs(m, A, u, v, max_nodes_per_hop=100, batch_size=50, sample_seed=2)
    results = {}
    for B in (50, 256):
        for use_graph in (True, False):
            eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=B, sample_seed=2, use_graph=use_graph)
            at, pos = _run(eng, u, v)
            results[(B, use_graph)] = at
            if (B, use_graph) == (50, True):
                tops = {k: eng.attribute_pairs(u, v, k) for k in (1, 10, 256)}
            eng.close()
            if (B, use_graph) != (50, True):
                continue
            assert torch.equal(at.score, base)
            assert torch.equal(at.num_edges, exp.num_edges) and torch.equal(at.offsets, exp.offsets)
            off = at.offsets.cpu().numpy()
            for q in range(3):
                s = slice(off[q], off[q + 1])
                mine = sorted(zip(at.user[s].tolist(), at.item[s].tolist(), at.rating[s].tolist()))
                theirs = sorted(zip(exp.user[s].tolist(), exp.item[s].tolist(), exp.rating[s].tolist()))
                assert mine == theirs, q
            g, pu, pi, pr = (t.cpu().numpy() for t in pos)
            _, order = rc.explain_order_host(None, g, off)
            assert np.array_equal(at.grad.cpu().numpy(), g[order])
            assert np.array_equal(at.user.cpu().numpy(), pu[order]) and np.array_equal(at.item.cpu().numpy(), pi[order])
            assert np.array_equal(at.rating.cpu().numpy(), pr[order])
            for k, t in tops.items():
                assert t.grad.shape == (3, k) and torch.equal(t.score, at.score)
                for q in range(3):
                    n = min(k, off[q + 1] - off[q])
                    for f in ("user", "item", "rating", "grad"):
                        a, b = getattr(t, f)[q], getattr(at, f)[off[q]:off[q] + n]
                        assert torch.equal(a[:n], b), (k, q, f)
                        assert (a[n:] == (0 if f == "grad" else -1)).all(), (k, q, f)
    first = results[(50, True)]
    for key, r in results.items():
        for f in r._fields:
            assert torch.equal(getattr(r, f), getattr(first, f)), (key, f)


def test_validation_and_empty_input():
    A = support.adj("ml_100k")
    m = support.model(5)
    with pytest.raises(IndexError):
        rc.attribute_pairs(m, A, [A.shape[0]], [0])
    with pytest.raises(ValueError):
        rc.attribute_pairs(m, A, [0, 1], [0])
    at = rc.attribute_pairs(m, A, [], [], 4)
    assert at.grad.shape == (0, 4) and at.offsets.tolist() == [0]
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=200, batch_size=50)
    at = eng.attribute_pairs([], [])
    assert at.grad.shape == (0,) and at.offsets.tolist() == [0]
    eng.close()


def test_three_checkpoints_are_the_fp32_mean():
    A = _with_cold_start(support.adj("ml_100k"))
    m = support.model(5)
    u, v = _pairs(A, small=True)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for c in range(3):
            paths.append(os.path.join(tmp, "model_checkpoint%d.pth" % c))
            torch.save(support.model(5, seed=c + 1).state_dict(), paths[-1])
        runs = []
        for ck in (paths, paths[:1], paths[1:2], paths[2:]):
            eng = rc.InferenceEngine(m, A, max_nodes_per_hop=200, batch_size=50, checkpoints=ck)
            runs.append(_run(eng, u, v))
            eng.close()
    (ens, pe), (a0, p0), (a1, p1), (a2, p2) = runs
    mean = lambda a, b, c: ((a + b) + c) / torch.full_like(a, 3.0)     # (a CUDA tensor / a scalar multiplies by 1/3)
    assert torch.equal(ens.score, mean(a0.score, a1.score, a2.score))
    assert torch.equal(pe[0], mean(p0[0], p1[0], p2[0]))
    assert torch.equal(ens.num_edges, a0.num_edges) and not torch.equal(ens.grad, a0.grad)
    assert ens.grad.numel() > 0


def test_engine_attributes_across_updates():
    A = support.adj("ml_1m")
    m = support.model(5, rgcn="pyg-2", pyg2_bias=True)
    g = RatingGraph(A, reserve_nnz=2000)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=64, sample_seed=4)
    rng = np.random.default_rng(5)
    u, v = _pairs(_with_cold_start(A))
    u, v = u[:2], v[:2]
    try:
        eng.attribute_pairs(u, v, 10)
        coo = A.tocoo()
        k = rng.choice(A.nnz, 300, replace=False)
        du = np.concatenate([coo.row[k[:150]], rng.integers(0, A.shape[0], 150)])
        dv = np.concatenate([coo.col[k[:150]], rng.integers(0, A.shape[1], 150)])
        dx = np.concatenate([np.zeros(75, np.int64), rng.integers(1, 6, 225)])
        g.update(du, dv, dx)
        A2 = _apply_scipy(A, du, dv, dx, g.shape)
        got = eng.attribute_pairs(u, v)
        fresh = rc.InferenceEngine(m, RatingGraph(A2), max_nodes_per_hop=100, batch_size=64, sample_seed=4)
        want = fresh.attribute_pairs(u, v)
        fresh.close()
    finally:
        eng.close()
    for f in got._fields:
        assert torch.equal(getattr(got, f), getattr(want, f)), f


def test_steady_state_steps_do_not_sync():
    A = support.adj("ml_1m")
    m = support.model(5, dgcnn=True)
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=2, sample_seed=1)
    u, v = np.arange(11, 23), np.arange(40, 52)
    outs = []
    try:
        for rep in range(2):
            eng.start_attribute(u, v)
            while eng.run["phase"] == "base":
                assert eng.step()
            for _ in range(4):              # eager warm-up and capture of both slots of the gradient pass
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
