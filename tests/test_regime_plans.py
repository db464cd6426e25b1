"""The shapes of tests/test_gpu_regimes.py still land in the kernel regimes they are meant to pin (host-only plan
queries, no GPU needed).  If shared-memory budgets, chunking or staging capacities are retuned so that one of these
fails, the named GPU test has silently stopped covering its branch: re-pick its shape (tests/helpers.py REGIMES)."""
import ctypes
import functools

import pytest

from igmc_b200 import _lib
from tests import support
from tests.helpers import REGIMES, XCH, layer0_tile_rows, own_counts

_cpu_model = functools.partial(support.model, seed=None, cuda=False)   # plan queries: unseeded, on the host


def _stage(m, n_cap, plan, backward):
    img = _lib.Stage()
    rc = _lib.load().igmc_stage_plan(ctypes.byref(m._cmodel), n_cap, plan, backward, ctypes.byref(img))
    assert rc == 0, rc
    return img


def _fits(m, n_cap, plan):
    lib, c = _lib.load(), ctypes.byref(m._cmodel)
    return lib.igmc_model_plan(c, n_cap, plan, 0) > 0 and lib.igmc_model_plan(c, n_cap, plan, 1) > 0


@pytest.mark.parametrize("name", sorted(REGIMES))
def test_regime_shapes_fit(name):
    r = REGIMES[name]
    assert _fits(_cpu_model(r["R"], in0=r["in0"]), r["n_cap"], r["plan"]), name


def test_bwd_chunks_past_xch():
    r = REGIMES["bwd_chunks_past_xch"]
    bwd = _stage(_cpu_model(r["R"], in0=r["in0"]), r["n_cap"], r["plan"], 1)
    assert bwd.chunk * XCH < r["own"], ("bwd_chunks_past_xch", bwd.chunk)


@pytest.mark.parametrize("name", ["layer0_tile_passes_in4", "layer0_tile_passes_in8"])
def test_layer0_tile_passes(name):
    r = REGIMES[name]
    bwd = _stage(_cpu_model(r["R"], in0=r["in0"]), r["n_cap"], r["plan"], 1)
    assert layer0_tile_rows(r["R"], r["in0"], bwd.chunk) < r["own"], (name, bwd.chunk)


def test_fwd_staged_bwd_global():
    r = REGIMES["fwd_staged_bwd_global"]
    m = _cpu_model(r["R"], in0=r["in0"])
    fwd, bwd = _stage(m, r["n_cap"], r["plan"], 0), _stage(m, r["n_cap"], r["plan"], 1)
    lo, hi = r["entries"]
    assert bwd.lcap < lo and fwd.lcap >= hi, ("fwd_staged_bwd_global", fwd.lcap, bwd.lcap)


def test_fwd_global_eval():
    r = REGIMES["fwd_global_eval"]
    fwd = _stage(_cpu_model(r["R"], in0=r["in0"]), r["n_cap"], r["plan"], 0)
    assert fwd.lcap < r["entries"], ("fwd_global_eval", fwd.lcap)


def test_fwd_global_eval_hinted():
    r = REGIMES["fwd_global_eval_hinted"]
    m = _cpu_model(r["R"], in0=r["in0"])
    m._cmodel.list_hint = 1 << 20            # any hint: the capacity it buys is capped
    fwd = _stage(m, r["n_cap"], r["plan"], 0)
    assert fwd.lcap < r["entries"], ("fwd_global_eval_hinted", fwd.lcap)


def test_ctas_without_nodes():
    r = REGIMES["ctas_without_nodes"]
    assert 0 in own_counts(r["n"], r["plan"])
    assert sum(own_counts(r["n"], r["plan"])) == r["n"]


@pytest.mark.parametrize("R", [8, 12])
def test_weight_gradient_second_tile_pass(R):
    """8 (R+1) weight-gradient column tiles over the 16 warps of a 512-thread CTA: more than 4 per warp from R = 8 on,
    so the tiles run in a second pass over the nodes (rs_plan)."""
    assert -(-8 * (R + 1) // 16) > 4
    assert -(-8 * (7 + 1) // 16) <= 4


def test_relation_count_and_width_shapes_fit():
    """every (R, in0, n_cap, plan, layers) the GPU regime tests run is accepted by the plan; R = 13 only by plan 0"""
    for R in (1, 2, 7, 8, 11, 12):
        for NB in (2, 4):
            for plan in (1, 2, 4):
                assert _fits(_cpu_model(R, in0=4, nb=NB), 62, plan), (R, NB, plan)
    m13 = _cpu_model(13, in0=4)
    assert not _fits(m13, 62, 1) and not _fits(m13, 62, 2) and _fits(m13, 62, 0)
    for in0, n_cap in ((6, 162), (8, 152)):     # h = 2 at mnph 40, h = 3 at mnph 25 on ml_100k*
        for plan in (0, 1, 2, 4):
            assert _fits(_cpu_model(5, in0=in0), n_cap, plan), (in0, n_cap, plan)
    for L in (1, 2, 3, 8):
        for plan in (0, 2):
            assert _fits(_cpu_model(5, in0=4, layers=L), 62, plan), (L, plan)
    for plan in (1, 2, 4):                      # degenerate-subgraph batches (dense 200 x 200 background)
        assert _fits(_cpu_model(5, in0=4), 202, plan), plan
