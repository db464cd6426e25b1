"""Element-by-element fp32 error bounds of the model kernels on foreign batches the extractor never builds
(tests/foreign_batch_cases.py): targets as the last nodes of their graph, edges shuffled, self-loops, parallel edges
of one and of two types, ratings with one direction only, sender / receiver hubs that put one CTA's in-lists and
another's out-lists past the list buffers of a cluster plan, edge-less and single graphs.

The protocol is test_gpu_error_bounds.test_error_bounds' with the same KAPPA: an eval forward, then a train step
(``fused_step``, ARR 0.001, the kernels' own hash edge and hidden dropout; one case the one-launch train kernel), every
quantity checked by ``eb.check_device``.  Each check prints its largest err / (u M).

Also: a foreign batch whose edge types leave [0, R) raises IndexError before anything is launched; malformed batches
raise; a rating label past the model's relations is flagged by the extractors (IGMC_ERR_LABEL) and refused on the
host where the engine can see it."""
import functools

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from tests import error_bounds as eb
from tests import foreign_batch_cases as fb
from tests.test_gpu_error_bounds import _dgcnn, _igmc, _report, _ws
from tests.test_gpu_regimes import _images, _restaged_step_bit_identical

pytestmark = pytest.mark.gpu

R = 5
L2_1, L2_2 = _lib.plan_l2(1), _lib.plan_l2(2)


@functools.lru_cache(maxsize=None)
def _small():
    return fb.small(R)


@functools.lru_cache(maxsize=None)
def _ml_100k():
    return fb.ml_100k()


def _foreign(ob):
    from igmc_b200.util_functions import Batch
    return Batch.from_arrays(ob["x"], ob["edge_index"], ob["edge_type"], ob["batch"], ob["y"], ob["num_graphs"])


@functools.lru_cache(maxsize=None)
def _ml_100k_mnph100():
    return fb.ml_100k(B=16, mnph=100)


BATCHES = {
    "permuted": lambda: fb.permuted(_small(), 1),
    "multigraph": lambda: fb.multigraph(_small(), R, 2),
    "ml_100k_permuted": lambda: fb.permuted(_ml_100k(), 6),
    "staging_split": lambda: fb.staging_split(_ml_100k_mnph100(), _small(), R)[0],
    "edgeless": lambda: fb.with_edgeless(_small(), 8, 5),
    "multigraph_B1": lambda: fb.multigraph(_small(), R, 3, graphs=[0]),
}

# case id -> (model builder, batch, expected plan)
CASES = {
    **{"%s_plan%d" % (k, p): (lambda p=p: _igmc(4, R, plan=p), k, p)
       for k in ("permuted", "multigraph") for p in (0, 1, 2, 3, 4, L2_1, L2_2)},
    "ml_100k_permuted_plan4": (lambda: _igmc(4, R, plan=4), "ml_100k_permuted", 4),
    **{"nb2_multigraph_plan%d" % p: (lambda p=p: _igmc(4, R, NB=2, plan=p), "multigraph", p) for p in (0, 2, 4)},
    **{"pyg2_multigraph_plan%d" % p: (lambda p=p: _igmc(4, R, plan=p, rgcn="pyg-2"), "multigraph", p)
       for p in (0, 2, L2_2)},
    **{"dgcnn_k30_multigraph_plan%d" % p: (lambda p=p: _dgcnn(30, 1, p), "multigraph", p) for p in (2, L2_2)},
    "staging_split_plan2": (lambda: _igmc(4, R, plan=fb.SPLIT_PLAN), "staging_split", fb.SPLIT_PLAN),
    **{"%s_plan%d" % (k, p): (lambda p=p: _igmc(4, R, plan=p), k, p)
       for k in ("edgeless", "multigraph_B1") for p in (2, 0)},
    "multigraph_plan2_one_launch": (lambda: _igmc(4, R, plan=2), "multigraph", 2),
    "multigraph_plan4_restaged": (lambda: _igmc(4, R, plan=4), "multigraph", 4),
}
ONE_LAUNCH = {"multigraph_plan2_one_launch"}
RESTAGED = {"multigraph_plan4_restaged", "staging_split_plan2"}


def _staging_split_regimes(m, b):
    """from the list-image headers of the step (tab[:, 2]: lists staged): a CTA whose forward (in-) lists are staged
    while its backward (out-) lists are read from global memory with per-edge dropout hashing, and a CTA with the
    reverse"""
    tabs, _ = _images(m, b)
    b._stage = None
    f, w = tabs["fwd"], tabs["bwd"]
    assert np.any((f[:, 2] == 1) & (w[:, 2] == 0)), "no CTA with staged forward and global backward lists"
    assert np.any((f[:, 2] == 0) & (w[:, 2] == 1)), "no CTA with global forward and staged backward lists"


REGIME = {"staging_split_plan2": _staging_split_regimes}


@pytest.mark.parametrize("case", list(CASES))
def test_foreign_batch_bounds(case, monkeypatch):
    from igmc_b200.models import edge_keep_reference, hidden_keep_reference, splitmix64
    build_model, which, plan = CASES[case]
    ob = BATCHES[which]()
    b = _foreign(ob)
    m = build_model()
    assert m._plan(b) == plan
    REGIME.get(case, lambda m, b: None)(m, b)
    m.eval()
    with torch.no_grad():
        m(b)
    b.check()
    bad = _report(case, "eval", eb.check_device(m, ob, _ws(m, False), False))
    m.train()
    step = 30
    m._step = step
    seed = splitmix64(m.drop_seed + step + 1)      # the step's own draws (the step increments _step first)
    ek = edge_keep_reference(seed, ob["edge_index"].shape[1], m.adj_dropout)
    hk = hidden_keep_reference(seed, b.num_graphs, m.hidden_dropout_p)
    if case in ONE_LAUNCH:
        monkeypatch.setenv("IGMC_FUSED_FB", "1")
        assert m.fused_update_ok(b)
        saved = m.forward_backward(b)
        m._launch_grad_reduce(b, saved, loss_scale=1.0 / b.num_graphs, arr=0.001)
    else:
        m.fused_step(b, ARR=0.001)
    b.check()
    bad += _report(case, "train", eb.check_device(m, ob, _ws(m, True), True, ek, 0.001, hk))
    assert not bad, bad
    if case in RESTAGED:
        m._step = step
        _restaged_step_bit_identical(m, b, hk, step)


# ---- what the models refuse -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad_type", [R, -1, 255])
@pytest.mark.parametrize("entry", ["forward", "fused_step", "forward_backward", "stage_batch", "dgcnn_forward"])
def test_edge_type_outside_relations_raises_before_launch(entry, bad_type):
    ob = fb.multigraph(_small(), R, 2)
    ob["edge_type"] = ob["edge_type"].copy()
    ob["edge_type"][len(ob["edge_type"]) // 2] = bad_type
    b = _foreign(ob)
    assert b._priv["type_range"] == (min(int(ob["edge_type"].min()), bad_type), max(int(ob["edge_type"].max()),
                                                                                       bad_type))
    m = _dgcnn(30, 1, 2) if entry == "dgcnn_forward" else _igmc(4, R, plan=2)
    m.train(entry != "forward")
    call = dict(forward=lambda: m(b), dgcnn_forward=lambda: m(b), fused_step=lambda: m.fused_step(b, ARR=0.001),
                forward_backward=lambda: m.forward_backward(b), stage_batch=lambda: m.stage_batch(b))[entry]
    with torch.no_grad(), pytest.raises(IndexError, match="edge type %d" % bad_type):
        call()
    # nothing was launched on the batch: no adjacency, no workspace, no list image
    assert b._adj is None and not m._ws and not getattr(b, "_stage", None)
    b.check()


@pytest.mark.parametrize("which", ["empty_graph", "no_label0"])
def test_malformed_batch_raises(which):
    parts = fb.split(fb.permuted(_small(), 1))
    x, ei, et, y = parts[4]
    if which == "empty_graph":
        parts[4] = (x[:0], ei[:, :0], et[:0], y)
    else:
        x = x.copy()
        x[np.argmax(x, 1) == 0] = np.eye(x.shape[1], dtype=x.dtype)[2]      # the target user relabelled a plain user
        parts[4] = (x, ei, et, y)
    ob = fb.collate(parts)
    b = _foreign(ob)
    m = _igmc(4, R, plan=2)
    m.eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="malformed batch"):
        m(b)
        b.check()


# ---- rating labels past the model's relations on the extracted path -----------------------------------------------
def _graph_and_model():
    from igmc_b200.data import build_adj, synth_ratings
    from igmc_b200.models import IGMC
    nu, ni = 120, 90
    u, v, lab = synth_ratings(nu, ni, 2500, R, 3)
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True).cuda()
    m.eval()
    return build_adj(u, v, lab, nu, ni), m


def test_label_past_relations_raises_and_delete_restores():
    from igmc_b200 import recommend as rc
    from igmc_b200.util_functions import RatingGraph
    A, m = _graph_and_model()
    g = RatingGraph(A, reserve_nnz=16)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=30, batch_size=32, sample_seed=5)
    free = next((u, v) for u in range(A.shape[0]) for v in range(A.shape[1]) if not A[u, v])
    pu, pv = np.arange(40) % A.shape[0], (np.arange(40) * 7) % A.shape[1]
    pu[0], pv[3] = free[0], free[1]
    try:
        g.update([free[0]], [free[1]], [R + 1])          # stored label R: one past the model's relations
        with pytest.raises(RuntimeError, match="rating label"):
            eng.predict_pairs(pu, pv)
        with pytest.raises(RuntimeError, match="rating label"):
            eng.recommend(np.array([free[0], 3]), 5)
        g.update([free[0]], [free[1]], [0])              # value 0 deletes the rating
        got_s, got_t = eng.predict_pairs(pu, pv), eng.recommend(np.array([free[0], 3]), 5)
        fresh = rc.InferenceEngine(m, RatingGraph(A), max_nodes_per_hop=30, batch_size=32, sample_seed=5)
        want_s, want_t = fresh.predict_pairs(pu, pv), fresh.recommend(np.array([free[0], 3]), 5)
        fresh.close()
        assert torch.equal(got_s, want_s)
        assert torch.equal(got_t[0], want_t[0]) and torch.equal(got_t[1], want_t[1])
    finally:
        eng.close()


def test_session_value_past_relations_raises():
    from igmc_b200 import recommend as rc
    from igmc_b200.util_functions import RatingGraph
    A, m = _graph_and_model()
    g = RatingGraph(A)
    u = 3
    v = next(v for v in range(A.shape[1]) if not A[u, v])
    sess = rc.RatingSessions(g, np.array([u]), np.array([0]), np.array([v]), np.array([R + 1]))
    with pytest.raises(RuntimeError, match="rating label"):
        rc.recommend_sessions(m, sess, 5, max_nodes_per_hop=30)


def test_class_values_longer_than_relations_raise():
    from igmc_b200.train_eval import OnlineTrainer
    from igmc_b200.models import FusedAdam
    from igmc_b200.util_functions import RatingGraph
    A, m = _graph_and_model()
    with pytest.raises(ValueError, match="6 class values for a model of 5 relations"):
        OnlineTrainer(m, RatingGraph(A), FusedAdam(m), batch_size=8, max_nodes_per_hop=30,
                      class_values=np.arange(1, 7, dtype=np.float32))
