"""Per-element fp32 error bounds (tests/error_bounds.py) in the regimes the train kernels branch on: relation counts
that give each mix of weight-gradient tile counts, layer counts 1..8 on every plan family, degenerate batches, the
staging limits of tests/helpers.py REGIMES and the readout variants.

Each case declares what it is next to its builders: R, NB, L, in0, rgcn, readout, the kernel plan, n_cap and the
regimes it claims.  The test builds the model from that metadata, asserts that the model and batch enter every
claimed regime (``REGIME_CHECKS``: plan, list-image tables, batch shapes), then runs an eval forward and (unless
the case is eval-only) one ``fused_step`` with ARR 0.001 and the kernels' own dropout draws, and bounds every layer's
states, the predictions, ``d hid`` and ``flat_grad`` per element as tests/test_gpu_error_bounds.py does.
tests/test_regime_bounds_coverage.py checks from the metadata alone, without a GPU, that the cases still cover every
tile-count class, plan family x layer count, REGIMES entry, RGCN layer and readout."""
import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from tests import error_bounds as eb
from tests.helpers import REGIMES, SEG, XCH, image_tables, layer0_tile_rows
from tests.test_gpu_error_bounds import _report
from tests.test_gpu_regimes import (_degenerate_matrix, _dense, _dense_block_matrix, _extracted, _images, _matrix,
                                    _mixed_pairs, _small_batch)

pytestmark = pytest.mark.gpu

L2 = _lib.plan_l2(2)


# ---- batches: dict(b, ob) and optionally edge_keep (injected edge dropout), prelude (batches evaluated first) -------
def _small(R=5, B=8):
    """B pairs of a 120 x 90 synthetic matrix, mnph 30 (n_cap 62)"""
    b, ob = _small_batch(B, R)
    return dict(b=b, ob=ob)


def _degenerate(which):
    """the mixed batch of tests/test_gpu_regimes.py (2-node subgraphs without edges, cold-start targets, 202-node
    subgraphs), one isolated pair (B = 1) or one normal pair"""
    A, pairs = _degenerate_matrix()
    sel = {"mixed": _mixed_pairs(pairs), "one_isolated": [pairs["iso"][2]], "one_normal": [pairs["bg"][2]]}[which]
    b, ob = _extracted(A, tuple(np.array(c) for c in zip(*sel)), 5, 1, 100)
    return dict(b=b, ob=ob)


def _emptied_in_lists():
    """the mixed batch as a foreign batch with an injected edge_keep that drops every in-edge of four nodes (a target
    item among them): their mean aggregate is empty and the layer is the root term alone"""
    from igmc_b200.util_functions import Batch
    A, pairs = _degenerate_matrix()
    _, ob = _extracted(A, tuple(np.array(c) for c in zip(*_mixed_pairs(pairs))), 5, 1, 100)
    b = Batch.from_arrays(ob["x"], ob["edge_index"], ob["edge_type"], ob["batch"], ob["y"], ob["num_graphs"])
    nptr = np.concatenate([[0], np.cumsum(np.bincount(ob["batch"], minlength=ob["num_graphs"]))])
    n_u1 = int((ob["x"][nptr[1]:nptr[2], 0::2].sum(1) > 0).sum())
    chosen = np.array([nptr[1] + n_u1, nptr[1] + 3, nptr[3] + 7, nptr[3] + n_u1 + 5])
    dst = ob["edge_index"][1]
    ek = torch.from_numpy((np.random.default_rng(6).random(len(dst)) > 0.2) & ~np.isin(dst, chosen))
    return dict(b=b, ob=ob, edge_keep=ek, emptied=chosen)


def _block_pairs(n, extra=()):
    """pairs inside the fully rated 101 x 101 block and of the sparse background (tests/test_gpu_regimes.py)"""
    A, (u, v, lab) = _dense_block_matrix(5)
    blk = np.nonzero((u < 101) & (v < 101))[0]
    bg = np.nonzero(u >= 101)[0]
    pick = np.array([blk[17], bg[0], blk[5000], bg[1]] + [blk[i] for i in extra])[:n]
    b, ob = _extracted(A, (u[pick], v[pick], lab[pick]), 5, 1, 100)
    return dict(b=b, ob=ob)


def _hinted_block():
    """mnph 200: a sparse batch first (it sizes list_hint), then pairs inside a fully rated 201 x 201 block"""
    from igmc_b200.data import synth_ratings
    bu, bv, bl = synth_ratings(700, 1400, 50000, num_classes=5, seed=6)
    A, (u, v, lab) = _matrix([_dense(201, 201, 1.1, 5, 7), (bu + 201, bv + 201, bl)], 901, 1601)
    sparse = np.nonzero(u >= 201)[0][:8]
    pick = np.concatenate([np.nonzero(u < 201)[0][[5, 999, 20000, 40000]], sparse[:4]])
    pre, _ = _extracted(A, (u[sparse], v[sparse], lab[sparse]), 5, 1, 200)
    b, ob = _extracted(A, (u[pick], v[pick], lab[pick]), 5, 1, 200)
    return dict(b=b, ob=ob, prelude=[pre])


def _dense_r12(dim, density, seed, h, n, pick_seed):
    """~200-node subgraphs of a dense dim x dim matrix with 12 rating levels (mnph 100)"""
    A, (u, v, lab) = _matrix([_dense(dim, dim, density, 12, seed)], dim, dim)
    pick = np.random.default_rng(pick_seed).choice(len(u), n, replace=False)
    b, ob = _extracted(A, (u[pick], v[pick], lab[pick]), 12, h, 100)
    return dict(b=b, ob=ob)


# ---- regimes: name -> check(m, b, ob, case, data) run before the steps --------------------------------------------
def _tabs(m, b):
    tabs, imgs = _images(m, b)
    b._stage = None
    return tabs, imgs


def _eval_headers(m, b):
    st = m.stage_batch(b, training=False)
    img, t = st["fwd"]
    b._stage = None
    return t["tab"][:, :4].cpu().numpy(), img.lcap


def _bwd_chunks_past_xch(m, b, ob, c, d):
    r = REGIMES["bwd_chunks_past_xch"]
    tabs, imgs = _tabs(m, b)
    entered = False
    for row in tabs["bwd"]:
        lens, nex = image_tables(row, c["n_cap"], c["plan"])
        entered |= bool(np.any((np.arange(len(lens)) >= XCH * imgs["bwd"].chunk) & (lens > SEG) & (nex == 0)))
    assert entered and int(tabs["bwd"][:, 3].max()) >= r["own"]


def _layer0_tile_passes(name):
    def check(m, b, ob, c, d):
        r = REGIMES[name]
        tabs, imgs = _tabs(m, b)
        own = int(tabs["bwd"][:, 3].max())
        assert c["in0"] == r["in0"] and own >= r["own"]
        assert own > layer0_tile_rows(c["R"], c["in0"], imgs["bwd"].chunk)
    return check


def _fwd_staged_bwd_global(m, b, ob, c, d):
    lo, hi = REGIMES["fwd_staged_bwd_global"]["entries"]
    tabs, _ = _tabs(m, b)
    f, w = tabs["fwd"], tabs["bwd"]
    assert np.any((f[:, 2] == 1) & (w[:, 2] == 0))
    assert np.all(w[w[:, 2] == 0, 0] >= lo) and np.all(f[:, 0] <= hi)


def _fwd_global_eval(name):
    def check(m, b, ob, c, d):
        hdr, lcap = _eval_headers(m, b)
        entries = REGIMES[name]["entries"]
        glob = (hdr[:, 2] == 0) & (hdr[:, 0] >= entries)
        assert np.any(glob) and lcap < entries, (hdr, lcap)
        if name == "fwd_global_eval_hinted":
            assert int(m._cmodel.list_hint) > 0
    return check


def _ctas_without_nodes(m, b, ob, c, d):
    tabs, _ = _tabs(m, b)
    assert np.any(tabs["fwd"][:, 3] == 0) and np.any(tabs["bwd"][:, 3] == 0)


def _edges_per_graph(ob):
    return np.bincount(ob["batch"][ob["edge_index"][1]], minlength=ob["num_graphs"])


def _empty_subgraphs(m, b, ob, c, d):
    sizes = np.bincount(ob["batch"], minlength=ob["num_graphs"])
    assert sizes.min() == 2 and np.any((sizes == 2) & (_edges_per_graph(ob) == 0))


def _cold_targets(m, b, ob, c, d):
    indeg = np.bincount(ob["edge_index"][1], minlength=len(ob["x"]))
    target = (ob["x"][:, 0] == 1) | (ob["x"][:, 1] == 1)
    assert np.any(target & (indeg == 0))


def _batch_of_one(m, b, ob, c, d):
    assert ob["num_graphs"] == 1 and b.num_graphs == 1


def _emptied(m, b, ob, c, d):
    dst = ob["edge_index"][1]
    for v in d["emptied"]:
        assert np.any(dst == v) and not bool(d["edge_keep"][torch.from_numpy(dst == v)].any())


def _sortpool_pads(m, b, ob, c, d):
    assert np.bincount(ob["batch"], minlength=ob["num_graphs"]).min() < m.k


REGIME_CHECKS = {
    "bwd_chunks_past_xch": _bwd_chunks_past_xch,
    "layer0_tile_passes_in4": _layer0_tile_passes("layer0_tile_passes_in4"),
    "layer0_tile_passes_in8": _layer0_tile_passes("layer0_tile_passes_in8"),
    "fwd_staged_bwd_global": _fwd_staged_bwd_global,
    "fwd_global_eval": _fwd_global_eval("fwd_global_eval"),
    "fwd_global_eval_hinted": _fwd_global_eval("fwd_global_eval_hinted"),
    "ctas_without_nodes": _ctas_without_nodes,
    "empty_subgraphs": _empty_subgraphs,
    "cold_targets": _cold_targets,
    "batch_of_one": _batch_of_one,
    "emptied_in_lists": _emptied,
    "sortpool_pads": _sortpool_pads,
    "multiply_by": lambda m, b, ob, c, d: m.multiply_by not in (0, 1),
    "dgcnn_odd_k": lambda m, b, ob, c, d: m.k % 2 == 1,
}


# ---- cases ------------------------------------------------------------------------------------------------------
def case(batch, R=5, NB=4, L=4, in0=4, rgcn="pyg-1.4", readout="igmc", plan=2, n_cap=62, regimes=(), train=True,
         **model_kw):
    """``model_kw``: multiply_by (IGMC); latent_dim, k (DGCNN_RS; L must equal len(latent_dim))"""
    return dict(batch=batch, R=R, NB=NB, L=L, in0=in0, rgcn=rgcn, readout=readout, plan=plan, n_cap=n_cap,
                regimes=tuple(regimes), train=train, model_kw=model_kw)


def _dg(L=4, last=1, k=30, **kw):
    return dict(readout="dgcnn", L=L, latent_dim=[32] * (L - 1) + [last], k=k, **kw)


CASES = {
    # relation counts on the cluster plans: every mix of weight-gradient tile counts per warp (tests/
    # test_regime_bounds_coverage.py wgrad_classes); R = 5 is the layer-count cases', R = 12 the staging case's
    **{"R%d_nb%d_plan%d" % (R, NB, p): case(lambda R=R: _small(R), R=R, NB=NB, plan=p)
       for R, NB, p in ((1, 2, 1), (2, 4, 4), (3, 2, 2), (4, 4, 1), (6, 2, 4), (7, 4, 1), (8, 2, 4), (10, 4, 2),
                        (11, 4, 2))},
    # layer counts on every plan family (readout width 64 L, raw-row layout, reduce grid, shared-memory carve-up)
    **{"L%d_plan%d" % (L, p): case(_small, L=L, plan=p)
       for L in (1, 2, 3, 5, 8) for p in (0, 1, 2, 4, L2)},
    **{"L%d_plan3" % L: case(_small, L=L, plan=3) for L in (1, 8)},
    **{"pyg2_L%d_plan2" % L: case(_small, L=L, plan=2, rgcn="pyg-2") for L in (1, 8)},
    # degenerate batches
    **{"mixed_plan%d" % p: case(lambda: _degenerate("mixed"), plan=p, n_cap=202,
                                regimes=("empty_subgraphs", "cold_targets") + (("ctas_without_nodes",) if p > 1 else ()))
       for p in (1, 2, 4)},
    "one_isolated_plan2": case(lambda: _degenerate("one_isolated"), plan=2, n_cap=202,
                               regimes=("batch_of_one", "empty_subgraphs", "ctas_without_nodes")),
    "one_normal_plan4": case(lambda: _degenerate("one_normal"), plan=4, n_cap=202, regimes=("batch_of_one",)),
    "emptied_in_lists_plan2": case(_emptied_in_lists, plan=2, n_cap=202, regimes=("emptied_in_lists",)),
    "dgcnn_mixed_plan2": case(lambda: _degenerate("mixed"), plan=2, n_cap=202,
                              regimes=("empty_subgraphs", "sortpool_pads"), **_dg()),
    # staging regimes (tests/helpers.py REGIMES)
    "R12_plan1_bwd_chunks_past_xch": case(lambda: _dense_r12(150, 0.75, 1, 1, 4, 0), R=12, plan=1, n_cap=202,
                                          regimes=("bwd_chunks_past_xch", "layer0_tile_passes_in4")),
    "R12_plan1_in8_layer0_tile_passes": case(lambda: _dense_r12(100, 0.5, 2, 3, 3, 1), R=12, in0=8, plan=1,
                                             n_cap=202, regimes=("layer0_tile_passes_in8",)),
    "fwd_staged_bwd_global_plan2": case(lambda: _block_pairs(4), plan=2, n_cap=202,
                                        regimes=("fwd_staged_bwd_global",)),
    "fwd_global_eval_plan1": case(lambda: _block_pairs(5, (9999,)), plan=1, n_cap=202, train=False,
                                  regimes=("fwd_global_eval",)),
    "fwd_global_eval_hinted_plan4": case(_hinted_block, plan=4, n_cap=402, train=False,
                                         regimes=("fwd_global_eval_hinted",)),
    # readout variants
    **{"multiply_by%d_plan2" % k: case(_small, plan=2, multiply_by=k, regimes=("multiply_by",)) for k in (2, 3)},
    **{"dgcnn_last%d_plan2" % w: case(_small, plan=2, **_dg(last=w)) for w in (32, 17)},
    "dgcnn_one_layer_plan2": case(_small, plan=2, **_dg(L=1, last=8)),
    "dgcnn_k31_plan2": case(_small, plan=2, regimes=("dgcnn_odd_k",), **_dg(k=31, last=8)),
}


def build_model(c, device="cuda"):
    """the model a case declares (parameters from the model's own initialisation under seed 0)"""
    from igmc_b200.models import DGCNN_RS, IGMC
    torch.manual_seed(0)
    kw = dict(num_relations=c["R"], num_bases=c["NB"], regression=True, adj_dropout=0.2, rgcn=c["rgcn"])
    mk = dict(c["model_kw"])
    if c["readout"] == "dgcnn":
        m = DGCNN_RS(c["in0"], latent_dim=mk["latent_dim"], k=mk["k"], **kw)
    else:
        m = IGMC(c["in0"], latent_dim=[32] * c["L"], multiply_by=mk.get("multiply_by", 1), **kw)
    m = m.to(device)
    m.kernel_plan = c["plan"]
    return m


def _ws(m, b, train):
    return next(v for k, v in m._ws.items() if k[0] == b._priv["node_cap"] and k[1] == b.num_graphs and k[2] == train)


@pytest.mark.parametrize("name", list(CASES))
def test_regime_bounds(name):
    from igmc_b200.models import DGCNN_RS, edge_keep_reference, hidden_keep_reference, splitmix64
    c = CASES[name]
    d = c["batch"]()
    b, ob = d["b"], d["ob"]
    m = build_model(c)
    assert (len(m.convs), m.num_relations, m.num_bases, m.rgcn) == (c["L"], c["R"], c["NB"], c["rgcn"])
    assert isinstance(m, DGCNN_RS) == (c["readout"] == "dgcnn") and ob["x"].shape[1] == c["in0"]
    assert b._priv["n_cap"] == c["n_cap"] and b.num_graphs <= 16
    m.eval()
    with torch.no_grad():
        for pre in d.get("prelude", ()):
            m(pre)
    assert m._plan(b) == c["plan"]
    for regime in c["regimes"]:
        assert REGIME_CHECKS[regime](m, b, ob, c, d) is not False, regime
    with torch.no_grad():
        m(b)
    b.check()
    bad = _report(name, "eval", eb.check_device(m, ob, _ws(m, b, False), False))
    if c["train"]:
        m.train()
        step = 30
        m._step = step
        seed = splitmix64(m.drop_seed + step + 1)      # the step's own draws (the step increments _step first)
        ek = d.get("edge_keep")
        ek_ref = ek if ek is not None else edge_keep_reference(seed, ob["edge_index"].shape[1], m.adj_dropout)
        hk = hidden_keep_reference(seed, b.num_graphs, m.hidden_dropout_p)
        m.fused_step(b, ARR=0.001, edge_keep=ek)
        b.check()
        ws = _ws(m, b, True)
        bad += _report(name, "train", eb.check_device(m, ob, ws, True, ek_ref, 0.001, hk))
        if "emptied" in d:    # no kept in-edge: 1 / max(deg, 1) = 1, the aggregate is empty
            got = ws["inv_deg"][torch.from_numpy(d["emptied"]).cuda()].cpu()
            assert torch.equal(got, torch.ones(len(d["emptied"])))
    assert not bad, bad
