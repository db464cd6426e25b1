"""Per-element fp32 error bounds for the forward's fold branches in the relation-space kernels (csrc/rgcn_rs.cu,
forward_body).

With staged lists the gather stores the rows of one-segment nodes already scaled by their degree factor. The fold
pass then only visits rows with extra segments, and a chunk without extra segments skips it with its barrier. Each
case asserts from the batch's forward list images that it reaches its branch, then bounds an eval forward and one
``fused_step`` per element as tests/test_gpu_regime_bounds.py does. Both degree scalings are covered: 1/deg and the
mean per relation (PyG >= 1.6 RGCNConv)."""
import numpy as np
import pytest
import torch

from tests import error_bounds as eb
from tests.helpers import image_tables
from tests.test_gpu_error_bounds import _report
from tests.test_gpu_regime_bounds import _tabs, _ws, build_model, case
from tests.test_gpu_regimes import _dense, _extracted, _matrix, _small_batch

pytestmark = pytest.mark.gpu


def _small():
    """8 pairs of a 120 x 90 synthetic matrix, mnph 30: no list is longer than one segment"""
    b, ob = _small_batch(8, 5)
    return dict(b=b, ob=ob)


def _block50():
    """3 pairs of a fully rated 50 x 50 matrix, mnph 100: 100-node subgraphs whose every node has about 40 kept
    in-edges. At plan 4 the last CTA owns 16 of them, and each one has an extra segment."""
    A, (u, v, lab) = _matrix([_dense(50, 50, 1.1, 5, 11)], 50, 50)
    pick = np.random.default_rng(2).choice(len(u), 3, replace=False)
    b, ob = _extracted(A, (u[pick], v[pick], lab[pick]), 5, 1, 100)
    return dict(b=b, ob=ob)


def _chunks(m, b, c):
    """extra-segment counts of every staged forward chunk that has rows"""
    tabs, imgs = _tabs(m, b)
    chunk = imgs["fwd"].chunk
    out = []
    for row in tabs["fwd"]:
        if row[2] != 1:
            continue
        _, nex = image_tables(row, c["n_cap"], c["plan"])
        out += [nex[c0:c0 + chunk] for c0 in range(0, len(nex), chunk)]
    return out


def _no_extras(m, b, c):
    """a staged chunk without extra segments: the fold and its barrier are skipped"""
    assert any(len(x) and not x.any() for x in _chunks(m, b, c))


def _only_extras(m, b, c):
    """a staged chunk whose every row has extra segments: every row goes through the fold, none is scaled in the
    gather"""
    assert any(len(x) and x.all() for x in _chunks(m, b, c))


CASES = {
    "no_extras_plan2": (case(_small, plan=2), _no_extras),
    "no_extras_pyg2_plan2": (case(_small, plan=2, rgcn="pyg-2"), _no_extras),
    "only_extras_plan4": (case(_block50, plan=4, n_cap=102), _only_extras),
    "only_extras_pyg2_plan4": (case(_block50, plan=4, n_cap=102, rgcn="pyg-2"), _only_extras),
}


@pytest.mark.parametrize("name", list(CASES))
def test_fold_regime_bounds(name):
    from igmc_b200.models import edge_keep_reference, hidden_keep_reference, splitmix64
    c, check = CASES[name]
    d = c["batch"]()
    b, ob = d["b"], d["ob"]
    m = build_model(c)
    assert b._priv["n_cap"] == c["n_cap"]
    m.eval()
    assert m._plan(b) == c["plan"]
    check(m, b, c)
    with torch.no_grad():
        m(b)
    b.check()
    bad = _report(name, "eval", eb.check_device(m, ob, _ws(m, b, False), False))
    m.train()
    step = 30
    m._step = step
    seed = splitmix64(m.drop_seed + step + 1)      # the step's own draws (the step increments _step first)
    ek_ref = edge_keep_reference(seed, ob["edge_index"].shape[1], m.adj_dropout)
    hk = hidden_keep_reference(seed, b.num_graphs, m.hidden_dropout_p)
    m.fused_step(b, ARR=0.001)
    b.check()
    bad += _report(name, "train", eb.check_device(m, ob, _ws(m, b, True), True, ek_ref, 0.001, hk))
    assert not bad, bad
