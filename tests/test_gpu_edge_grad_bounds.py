"""Element-by-element fp32 error bounds of attribute_pairs' per-edge gradient (igmc_edge_grad, the EG mode of
k_l2_backward in csrc/rgcn_l2.cu) and of the DGCNN_RS SortPooling backward's ``dstate`` that seeds it
(tests/error_bounds.py ``edge_terms`` / ``readout_dstate``).

Each case drives the kernels as the gradient pass of InferenceEngine does, on one batch: the L2-plan eval forward with
c CTAs per subgraph, for DGCNN_RS igmc_sortpool_backward seeded with 1 into a NaN-filled ``dstate``, then
igmc_edge_grad into a NaN-filled buffer.  Per directed edge:

    |got - ref| <= KAPPA["edge"] * 2^-24 * M,   got == 0 exactly where M == 0,

every edge of a single-entry segment (pyg-2: a type run of one entry) is exactly 0, no element is left NaN (every
edge has one writer and the top layer stores), and a second run over a zero-filled buffer is bit-identical.  DGCNN_RS:
``dstate`` within KAPPA["dstate"], exactly 0 in the padding columns of its width-1 last layer.  One end-to-end test ties
attribute_pairs' per-rating values bit for bit to the raw gradient of a batch of the same pairs.  Each case prints its
largest err / (u M) and the counts it asserted on."""
import ctypes as C

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.models import l2_cluster
from igmc_b200.util_functions import RatingGraph, SubgraphExtractor, _stream_ptr
from tests import error_bounds as eb
from tests import support
from tests.test_gpu_error_bounds import _many_relations, _ml_100k_batch, _scaled, _small
from tests.test_gpu_explain import _pairs, _with_cold_start
from tests.test_gpu_regimes import _extracted

pytestmark = pytest.mark.gpu


def _igmc(in0, R, NB, L=4, rgcn="pyg-1.4"):
    from tests.test_gpu_relation_mean import _models
    return _models(in0, R, NB=NB, L=L, rgcn=rgcn)[1]


def _dgcnn(NB, rgcn="pyg-1.4"):
    """DGCNN_RS with k 30 and a width-1 last layer; NB 2 and pyg-1.4 are the reference's defaults"""
    if rgcn == "pyg-1.4":
        from tests.test_gpu_dgcnn import _models
        return _models(5, NB, 30)[1]
    from tests.test_gpu_relation_mean import _models
    return _models(4, 5, NB=NB, dgcnn_k=30, rgcn=rgcn)[1]


def _ml_1m(B=16, mnph=100):
    ds = support.dataset("ml_1m")
    tu, tv, tl = ds["train"]
    idx = np.arange(B)
    return _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, 1, mnph)


def _ml_1m_uncapped():
    b, ob = _ml_1m(2, None)
    assert b._priv["n_cap"] > 256
    return b, ob


def _cold_start():
    """a rated pair, an unrated pair and the cold-start pair (a subgraph without edges) of ml_1m*"""
    A = _with_cold_start(support.adj("ml_1m"))
    u, v = _pairs(A)
    return _extracted(A, (u, v, np.zeros(3, np.int64)), 5, 1, 100)


# case id -> (model builder, batch builder, CTAs per subgraph)
CASES = {
    **{"ml_1m_nb%d_c%d" % (nb, c): (lambda nb=nb: _igmc(4, 5, nb), _ml_1m, c) for nb, c in ((2, 1), (4, 1), (2, 2),
                                                                                            (2, 8))},
    **{"pyg2_ml_1m_nb%d_c%d" % (nb, c): (lambda nb=nb: _igmc(4, 5, nb, rgcn="pyg-2"), _ml_1m, c)
       for nb, c in ((2, 1), (4, 2), (2, 8))},
    "dgcnn_nb2_k30": (lambda: _dgcnn(2), _ml_1m, 1),
    "dgcnn_pyg2_nb4_k30": (lambda: _dgcnn(4, "pyg-2"), _ml_1m, 2),
    "ml_1m_uncapped_nb2_c1": (lambda: _igmc(4, 5, 2), _ml_1m_uncapped, 1),
    "L1_nb2": (lambda: _igmc(4, 5, 2, L=1), _ml_1m, 1),
    "L8_nb2": (lambda: _igmc(4, 5, 2, L=8), _ml_1m, 1),
    "L8_pyg2_nb4": (lambda: _igmc(4, 5, 4, L=8, rgcn="pyg-2"), _ml_1m, 2),
    "h2_nb2": (lambda: _igmc(6, 5, 2), lambda: _ml_100k_batch(2, 40, 4), 1),
    "h3_pyg2_nb4": (lambda: _igmc(8, 5, 4, rgcn="pyg-2"), lambda: _ml_100k_batch(3, 25, 4), 1),
    "R1_foreign_nb2": (lambda: _igmc(4, 1, 2), lambda: _small(R=1), 1),
    "R13_foreign_pyg2_nb2": (lambda: _igmc(4, 13, 2, rgcn="pyg-2"), lambda: _small(R=13), 1),
    "R71_pyg2_nb2_c8": (lambda: _igmc(4, 71, 2, rgcn="pyg-2"), _many_relations, 8),
    "R71_pyg2_nb4_c1": (lambda: _igmc(4, 71, 4, rgcn="pyg-2"), _many_relations, 1),
    "scaled4_nb2": (lambda: _scaled(_igmc(4, 5, 2)), _ml_1m, 1),
    "scaled4_pyg2_nb2": (lambda: _scaled(_igmc(4, 5, 2, rgcn="pyg-2")), _ml_1m, 1),
    "foreign_nb4_c2": (lambda: _igmc(4, 5, 4), _small, 2),
    "foreign_pyg2_nb2_c1": (lambda: _igmc(4, 5, 2, rgcn="pyg-2"), _small, 1),
    "cold_start_nb2": (lambda: _igmc(4, 5, 2), _cold_start, 1),
}


def _edge_grad(m, b, csize, fill):
    """the gradient pass of attribute_pairs on batch ``b`` with ``csize`` CTAs per subgraph: (edge_grad [edge cap]
    over a buffer filled with ``fill``, dstate [node cap, 32 L] over NaN (DGCNN_RS, else None), the eval workspace)"""
    lib, p, B = _lib.load(), b._priv, b.num_graphs
    f32 = dict(dtype=torch.float32, device="cuda")
    own = (m.kernel_plan, m._plans)
    m.kernel_plan, m._plans = _lib.plan_l2(csize), {}
    try:
        m.eval()
        with torch.no_grad():
            _, saved = m._launch_forward(b, False, m.make_dropout(False))
        ws = saved["ws"]
        assert ws["cluster"] == _lib.plan_l2(csize)
        S = _lib.Saved.from_buffer_copy(saved["S"])
        scratch = torch.empty(2, p["node_cap"], _lib.HIDDEN, **f32)
        S.l2_scratch = scratch.data_ptr()
        ext = m._cmodel.readout != 0
        seed = torch.full((B,), 1.0 if ext else float(m._cmodel.multiply_by), **f32)
        dstate = None
        if ext:
            dstate = torch.full((p["node_cap"], _lib.HIDDEN * len(m.convs)), float("nan"), **f32)
            pgrad = torch.zeros(m._cmodel.param_count, **f32)
            S.dstate = dstate.data_ptr()
            _lib.check(lib.igmc_sortpool_backward(C.byref(m._csort), m.flat_params.data_ptr(), ws["states"].data_ptr(),
                                                  p["node_ptr"].data_ptr(), B, p["n_cap"], C.byref(ws["sp"]["S"]),
                                                  seed.data_ptr(), dstate.data_ptr(), 1.0, pgrad.data_ptr(),
                                                  b._err.data_ptr(), _stream_ptr()), "igmc_sortpool_backward")
        eg = torch.full((p["edge_cap"],), fill, **f32)
        adj_c, _ = b.adjacency()
        d, _ = m.make_dropout(False)
        _lib.check(lib.igmc_edge_grad(C.byref(m._cmodel), m.flat_params.data_ptr(), p["node_label"].data_ptr(),
                                      p["node_ptr"].data_ptr(), p["edge_ptr"].data_ptr(), C.byref(adj_c), B,
                                      p["n_cap"], C.byref(d), C.byref(S), seed.data_ptr(), eg.data_ptr(),
                                      ws["cluster"], b._err.data_ptr(), _stream_ptr()), "igmc_edge_grad")
        torch.cuda.synchronize()
        b.check()
        return eg, dstate, ws
    finally:
        m.kernel_plan, m._plans = own


def _graph(b):
    """the oracle-batch view of a device batch (what eb.Graph reads)"""
    return dict(x=b.x.cpu().numpy(), edge_index=b.edge_index.cpu().numpy(), edge_type=b.edge_type.cpu().numpy(),
                batch=b.batch.cpu().numpy(), num_graphs=b.num_graphs)


def _segment_size(g, aggr, R):
    dst, et = g.edge_index[1], g.edge_type
    seg = dst * R + et if aggr == "mean_per_relation" else dst
    return torch.bincount(seg)[seg]


def _check(m, ob, ws, eg, dstate, label):
    """{quantity: eb.ratio result} of the raw edge gradient (and dstate) against the fp64 recomputation, plus the
    reference values; asserts the exact-zero and no-NaN claims"""
    params = {k: v.detach().double().cpu().contiguous() for k, v in m.state_dict().items()}
    aggr = "mean_per_relation" if m.rgcn == "pyg-2" else "mean_all"
    dg = m._cmodel.readout != 0
    g = eb.Graph(ob)
    N, E = g.x.shape[0], g.edge_index.shape[1]
    saved = eb.device_saved(m, ws, N, False)
    saved["dpred"] = torch.full((g.num_graphs,), 1.0 if dg else float(m.multiply_by), dtype=torch.float64)
    res = {}
    if dg:
        widths = [c.out_channels for c in m.convs]
        got = dstate[:N].double().cpu()
        pad = lambda t: torch.cat([eb._pad32(x, 32) for x in torch.split(t, widths, 1)], 1)
        ref, M = eb.readout_dstate(params, g, saved, True), eb.readout_dstate(params, g, saved, True, mag=True)
        res["dstate"] = eb.ratio(got, pad(ref), pad(M))
        assert widths[-1] == 1 and bool((got[:, 32 * (len(widths) - 1) + 1:] == 0).all())
        saved["dstate"] = torch.cat([got[:, 32 * l:32 * l + w] for l, w in enumerate(widths)], 1)
    got = eg[:E].double().cpu()
    ref, M = eb.edge_terms(params, g, saved, aggr, dg), eb.edge_terms(params, g, saved, aggr, dg, mag=True)
    res["edge"] = eb.ratio(got, ref, M)
    assert not bool(torch.isnan(got).any()), "edges left unwritten"
    single = _segment_size(g, aggr, m.num_relations) == 1
    zero = M == 0
    assert bool((got[single] == 0).all()), "a single-entry segment with a nonzero gradient"
    print("edge grad %-24s %d edges, %d in single-entry segments, %d with M == 0" % (label, E, int(single.sum()),
                                                                                     int(zero.sum())))
    for key, (r, npad, worst) in res.items():
        print("edge grad %-24s %-6s err/(uM) %9.4f  kappa %4g  nonzero-at-M=0 %d  worst %d"
              % (label, key, r, eb.KAPPA[key], npad, worst))
    return res, single, zero, ref, M


@pytest.mark.parametrize("case", list(CASES))
def test_edge_grad_bounds(case):
    build_model, build_batch, csize = CASES[case]
    b, ob = build_batch()
    m = build_model()
    eg, dstate, ws = _edge_grad(m, b, csize, float("nan"))
    res, single, zero, _, _ = _check(m, ob, ws, eg, dstate, case)
    assert int(single.sum()) > 0, "no single-entry segment: the regime is not exercised"
    if len(m.convs) == 1:
        assert int(zero.sum()) > len(zero) // 2      # only edges into the two targets have a term at L = 1
    eg0, dstate0, _ = _edge_grad(m, b, csize, 0.0)
    assert torch.equal(eg0[:len(zero)], eg[:len(zero)])
    if dstate is not None:
        n = ob["x"].shape[0]
        assert torch.equal(dstate0[:n], dstate[:n])
    bad = [(k, v) for k, v in res.items() if not v[0] <= eb.KAPPA[k] or v[1]]
    assert not bad, bad


@pytest.mark.parametrize("dgcnn", [False, True])
def test_attribute_pairs_is_the_bounded_raw_gradient(dgcnn):
    """attribute_pairs on NB = 2 models (the reference's default): every per-rating value is bit for bit the sum of
    the two directed-edge values of igmc_edge_grad on a batch of the same pairs, sampling seed and B, on the plan the
    engine chose, and that sum is within KAPPA["edge"] of ref_j + ref_{j+m} with M_j + M_{j+m}"""
    A = _with_cold_start(support.adj("ml_1m"))
    m = _dgcnn(2) if dgcnn else _igmc(4, 5, 2)
    m.eval()
    u, v = _pairs(A)
    B, seed, mnph = len(u), 7, 100
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=mnph, batch_size=B, sample_seed=seed)
    try:
        eng.start_attribute(u, v)
        while eng.step():
            pass
        pos = eng.run["occ"].cpu().numpy().copy()
        at = eng.finish()
    finally:
        eng.close()
    ni = A.shape[1]
    ex = SubgraphExtractor(RatingGraph(A), [0], [0], [0], np.arange(1, 6, dtype=np.float32), 1, 1.0, mnph,
                           max_batch=B, seed=seed)
    b = ex.extract(pairs=(u, v, np.zeros(B, np.int64)), pair_ids=u * ni + v)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    csize = l2_cluster(b._priv["n_cap"], B, sms)
    eg, dstate, ws = _edge_grad(m, b, csize, float("nan"))
    edge_ptr = b._priv["edge_ptr"][:B + 1].cpu().numpy()
    offsets = at.offsets.cpu().numpy()
    assert np.array_equal(np.diff(edge_ptr) // 2, at.num_edges.cpu().numpy())
    out = np.zeros(int(offsets[-1]), np.float32)
    rc.edge_grad_scatter_host(edge_ptr, np.arange(B), eg.cpu().numpy(), offsets, out)
    assert np.array_equal(out, pos), float(np.abs(out - pos).max())
    res, _, _, ref, M = _check(m, _graph(b), ws, eg, dstate, "attribute_pairs dgcnn=%s" % dgcnn)
    rref, rM = [], []
    for q in range(B):
        e0, mm = int(edge_ptr[q]), int(edge_ptr[q + 1] - edge_ptr[q]) // 2
        rref.append(ref[e0:e0 + mm] + ref[e0 + mm:e0 + 2 * mm])
        rM.append(M[e0:e0 + mm] + M[e0 + mm:e0 + 2 * mm])
    r = eb.ratio(torch.from_numpy(out), torch.cat(rref), torch.cat(rM))
    print("attribute_pairs dgcnn=%s: %d ratings, per-rating err/(uM) %.4f" % (dgcnn, len(out), r[0]))
    assert r[0] <= eb.KAPPA["edge"] and r[1] == 0
    bad = [(k, v) for k, v in res.items() if not v[0] <= eb.KAPPA[k] or v[1]]
    assert not bad, bad
