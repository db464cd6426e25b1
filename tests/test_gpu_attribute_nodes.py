"""Attributing predicted ratings to the nodes of their enclosing subgraphs on the GPU (igmc_b200/recommend.py
attribute_nodes, igmc_node_grad_scatter in csrc/explain.cu).

* grad is bit for bit the documented-order sum of the raw igmc_edge_grad of the same batch: per node, its in-list
  ratings' two directed-edge gradients summed in list order;
* grad matches fp64 autograd of the weighted restatement (tests/edge_weight_oracle.py) with m_e = g[src] g[dst] and
  d/dg at g = 1, per pair max |got - ref| <= 2e-4 max |ref|: IGMC pyg-1.4 / pyg-2, DGCNN_RS in the kernel's SortPooling
  order, R = 5 / 13, h = 2 and ml_1m* without a node cap;
* the output is NaN-prefilled and no position is left NaN; the score is predict_pairs bit for bit; the nodes listed
  are explain_nodes'; results do not depend on B or graph replay; checkpoints are the fp32 mean."""
import os
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import recommend as rc
from tests import edge_weight_oracle as ewo
from tests import support
from tests.test_gpu_attribute import _kernel_perm, _ref
from tests.test_gpu_explain import _pairs, _subgraph, _with_cold_start
from tests.test_gpu_explain_nodes import _positions

pytestmark = pytest.mark.gpu


def _run(eng, u, v, m=None, prefill=False):
    """(NodeAttribution, gradients [T] in position order, node / label / ratings [T] in position order); with
    ``prefill`` the gradient buffer is NaN-filled before the gradient pass writes it"""
    eng.start_attribute_nodes(u, v, m)
    while eng.run["phase"] == "base":
        if not eng.step():
            break
    run = eng.run
    if prefill and run.get("occ") is not None:
        run["occ"].fill_(float("nan"))
    while eng.step():
        pass
    pos = tuple(run[k].clone() for k in ("occ", "user", "item", "rating"))
    return eng.finish(), pos


def _node_autograd(ref, x, ei, et, **kw):
    """d score / d g_n at g = 1 for every node, the weight of rating e being g[src] g[dst] on both its edges"""
    g = torch.ones(x.shape[0], dtype=x.dtype, device=x.device, requires_grad=True)
    w = g[ei[0]] * g[ei[1]]
    ewo.weighted_forward(ref, x, ei, et, w, **kw).sum().backward()
    return g.grad.detach()


CASES = {
    # name: (dataset, R, h, mnph, model kwargs, batch size)
    "pyg-1.4": ("ml_1m", 5, 1, 100, {}, 64),
    "pyg-2": ("ml_1m", 5, 1, 100, dict(rgcn="pyg-2"), 64),
    "DGCNN_RS": ("ml_1m", 5, 1, 100, dict(dgcnn=True), 64),
    "R=13": ("r13", 13, 1, 50, {}, 2),
    "h=2": ("ml_1m", 5, 2, 20, {}, 64),
    "ml_1m uncapped": ("ml_1m", 5, 1, None, {}, 64),
}


@pytest.mark.parametrize("name", list(CASES))
def test_grad_matches_fp64_autograd(name):
    dsn, R, h, mnph, kw, B = CASES[name]
    A0 = support.adj(dsn)
    A = _with_cold_start(A0)
    m = support.model(R, h=h, **kw, pyg2_bias=True)
    u, v = _pairs(A)
    seed = 7
    eng = rc.InferenceEngine(m, A, h=h, max_nodes_per_hop=mnph, batch_size=B, sample_seed=seed)
    at, (occ, *_) = _run(eng, u, v, prefill=True)
    eng.close()
    assert m.kernel_plan == "auto"
    assert not torch.isnan(occ).any()                    # every position written
    nn = at.num_nodes.cpu().numpy()
    assert nn[0] > 0 and nn[1] > 0 and nn[2] == 0
    ref = _ref(m, R, h, kw.get("rgcn", "pyg-1.4"), kw.get("dgcnn", False))
    off = at.offsets.cpu().numpy()
    occ = occ.double().cpu().numpy()
    sizes = []
    for q in range(2):
        sub, _ = _subgraph(A, R, int(u[q]), int(v[q]), h, mnph, seed)
        x, ei, et, _ = sub
        sizes.append(x.shape[0])
        assert x.shape[0] - 2 == nn[q]
        extra = {}
        if kw.get("dgcnn"):
            extra = dict(batch=torch.zeros(x.shape[0], dtype=torch.int64, device="cuda"), num_graphs=1,
                         perm=_kernel_perm(m, sub))
        want = _node_autograd(ref, x.double(), ei, et, **extra)[_positions(x)].cpu().numpy()
        got = occ[off[q]:off[q + 1]]
        err, scale = float(np.abs(got - want).max()), float(np.abs(want).max())
        print("%s pair %d: %d nodes, max |grad| %.3e, max err %.3e" % (name, q, x.shape[0], scale, err))
        assert scale > 0 and err <= 2e-4 * scale, (name, q, err, scale)
    if name == "ml_1m uncapped":
        assert max(sizes) > 256, sizes


def test_grad_is_the_in_list_sum_of_the_raw_edge_grad():
    """the engine's node values against igmc_edge_grad of the same batch, summed in the documented order here"""
    A = _with_cold_start(support.adj("ml_1m"))
    m = support.model(5)
    u, v = _pairs(A)
    B = 4                                       # one gradient batch: all three pairs and a padded slot
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=B, sample_seed=2)
    eng.start_attribute_nodes(u, v)
    while eng.run["phase"] == "base":
        assert eng.step()
    run = eng.run
    assert eng.step() is False
    b = eng.batches[0]                          # the gradient batch, and igmc_edge_grad's output for it
    eg = run["gws"]["edge_grad"].cpu().numpy()
    occ, ratings = run["occ"].cpu().numpy(), run["rating"].cpu().numpy()
    at = eng.finish()
    eng.close()
    p = b._priv
    node_ptr, edge_ptr = p["node_ptr"].cpu().numpy(), p["edge_ptr"].cpu().numpy()
    lab = p["node_label"].cpu().numpy()
    lists = b._adj[1]                           # the extractor's in-lists, which igmc_edge_grad walked
    in_ptr, in_eid = lists["adj_in_ptr"].cpu().numpy(), lists["adj_eid"].cpu().numpy()
    off = at.offsets.cpu().numpy()
    for q in range(3):
        e0, mm = int(edge_ptr[q]), int(edge_ptr[q + 1] - edge_ptr[q]) // 2
        pos = [n for n in range(node_ptr[q], node_ptr[q + 1]) if lab[n] >= 2]
        assert len(pos) == off[q + 1] - off[q]
        for j, n in enumerate(pos):
            acc = np.float32(0)
            for t, e in enumerate(in_eid[in_ptr[n]:in_ptr[n + 1]]):
                a = int(e) if int(e) - e0 < mm else int(e) - mm
                r = np.float32(eg[a] + eg[a + mm])
                acc = r if t == 0 else np.float32(acc + r)
            assert np.float32(acc).view(np.int32) == occ[off[q] + j].view(np.int32), (q, j)
            assert ratings[off[q] + j] == in_ptr[n + 1] - in_ptr[n]


def test_score_nodes_order_and_determinism():
    A = _with_cold_start(support.adj("ml_1m"))
    m = support.model(5)
    m.kernel_plan = 2                  # the base pass's plan at every batch size (the gradient pass forces L2)
    u, v = _pairs(A)
    base = rc.predict_pairs(m, A, u, v, max_nodes_per_hop=100, batch_size=50, sample_seed=2)
    exp = rc.explain_nodes(m, A, u, v, max_nodes_per_hop=100, batch_size=50, sample_seed=2)
    results = {}
    for B in (1, 50, 256):
        for use_graph in (True, False):
            eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=B, sample_seed=2, use_graph=use_graph)
            results[(B, use_graph)] = at = _run(eng, u, v)[0]
            if (B, use_graph) == (50, True):
                top = eng.attribute_nodes(u, v, 10)
                off = at.offsets.cpu().numpy()
                for q in range(3):
                    n = min(10, off[q + 1] - off[q])
                    assert torch.equal(top.grad[q, :n], at.grad[off[q]:off[q] + n])
                    assert (top.node[q, n:] == -1).all() and (top.ratings[q, n:] == 0).all()
            eng.close()
    first = results[(50, True)]
    assert torch.equal(first.score, base)
    assert torch.equal(first.num_nodes, exp.num_nodes) and torch.equal(first.offsets, exp.offsets)
    off = first.offsets.cpu().numpy()
    for q in range(3):
        s = slice(off[q], off[q + 1])
        assert sorted(zip(first.node[s].tolist(), first.label[s].tolist(), first.ratings[s].tolist())) == \
            sorted(zip(exp.node[s].tolist(), exp.label[s].tolist(), exp.ratings[s].tolist()))
        a = np.abs(first.grad[s].cpu().numpy())
        assert (np.diff(a) <= 0).all()
    for key, r in results.items():
        for f in r._fields:
            assert torch.equal(getattr(r, f), getattr(first, f)), (key, f)


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
    (ens, pe), (e0, p0), (e1, p1) = runs
    assert torch.equal(ens.score, (e0.score + e1.score) / 2)
    assert torch.equal(pe[0], (p0[0] + p1[0]) / 2)
    assert ens.grad.numel() > 0
