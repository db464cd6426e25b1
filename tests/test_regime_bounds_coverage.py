"""The cases of tests/test_gpu_regime_bounds.py still cover what they are there for, from their metadata and host plan
queries alone (no GPU): every mix of weight-gradient tile counts the relation-space backward runs for R <= 12, every
plan family at 1 and 8 layers, every staging regime of tests/helpers.py REGIMES, both RGCN layers and both readouts;
and every declared plan fits its model.  If the kernels are retuned (warps per CTA, tiles per warp, shared-memory
budgets), this file fails before the GPU cases silently stop covering a branch."""
import ctypes

import pytest

from igmc_b200 import _lib
from tests.helpers import REGIMES
from tests.test_gpu_regime_bounds import CASES, build_model

# restated from csrc/rgcn_rs.cu (backward_body, weight gradients): 8-column tiles of [dW_0 .. dW_{R-1} | d root], a
# warp pair per column-tile stride, at most MAXI tiles per warp and pass
THREADS, MAXI = 512, 4


def wgrad_classes(R, threads=THREADS):
    """the (pass, tile count) pairs the warps of one CTA run: warp w starts at column tile w / 2, takes every
    (warps / 2)-th tile, up to MAXI per pass (wgrad_pass<cnt>); further tiles take further passes over the nodes"""
    nwarps = threads // 32
    ntn, jstep = 4 * (R + 1), nwarps // 2
    out = set()
    for w in range(nwarps):
        for p, jp in enumerate(range(w >> 1, ntn, MAXI * jstep)):
            out.add((p, max(i + 1 for i in range(MAXI) if jp + i * jstep < ntn)))
    return frozenset(out)


def test_wgrad_classes_restate_the_kernel_table():
    want = {1: {(0, 1)}, 2: {(0, 1), (0, 2)}, 3: {(0, 2)}, 5: {(0, 3)}, 7: {(0, 4)}, 8: {(0, 4), (1, 1)},
            11: {(0, 4), (1, 2)}, 12: {(0, 4), (1, 2), (1, 3)}}
    for R, classes in want.items():
        assert wgrad_classes(R) == classes, R


def _trains_wgrad(c):
    """a case whose train step runs the weight-gradient tiles of a relation-space layer >= 1"""
    return c["train"] and _lib.is_rs(c["plan"]) and c["L"] >= 2


def test_every_tile_count_mix_is_bounded():
    """each launch's mix of tile counts (the set of (pass, count) pairs its warps run), for every R <= 12 the
    relation-space plans take: a case that drops one R loses its mix"""
    covered = {wgrad_classes(c["R"]) for c in CASES.values() if _trains_wgrad(c)}
    need = {wgrad_classes(R) for R in range(1, 13)}
    assert need <= covered, sorted(sorted(s) for s in need - covered)
    every = set().union(*need)
    assert every <= set().union(*covered)


def _family(plan):
    return "l2" if _lib.l2_csize(plan) else int(plan)


def test_every_plan_family_trains_at_1_and_8_layers():
    have = {(_family(c["plan"]), c["L"]) for c in CASES.values() if c["train"] and c["readout"] == "igmc"}
    for fam in (0, 1, 2, 3, 4, "l2"):
        for L in (1, 8):
            assert (fam, L) in have, (fam, L)


def test_every_regime_and_variant_is_claimed():
    claimed = set().union(*(c["regimes"] for c in CASES.values()))
    assert set(REGIMES) <= claimed, sorted(set(REGIMES) - claimed)
    assert {c["rgcn"] for c in CASES.values()} == {"pyg-1.4", "pyg-2"}
    assert {c["readout"] for c in CASES.values()} == {"igmc", "dgcnn"}
    for c in CASES.values():
        if c["readout"] == "dgcnn":
            assert len(c["model_kw"]["latent_dim"]) == c["L"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_declared_plan_fits(name):
    c = CASES[name]
    m = build_model(c, device="cpu")
    lib, cm = _lib.load(), ctypes.byref(m._cmodel)
    for backward in (0, 1) if c["train"] else (0,):
        assert lib.igmc_model_plan(cm, c["n_cap"], c["plan"], backward) > 0, (name, backward)
