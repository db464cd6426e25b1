"""The cases of tests/test_gpu_pair_grad_bounds.py still cover the regimes the per-pair gradient assembly branches on,
from their metadata and host plan queries alone (no GPU): every raw-assembly plan at R = 1 and R = 12, every CTA count
of the L2 plan, input widths 4, 6 and 8, 1 and 8 layers, num_bases 2 and 4 on both assembly paths, both seeds on every
plan family, PyG 2's layer, a cold-start pair, a padded tail, one pair and K > 1 checkpoints; and every declared plan
fits its model.  Removing one required case makes a test here fail."""
import ctypes

import pytest

from igmc_b200 import _lib
from tests.test_gpu_pair_grad_bounds import CASES, CHECKPOINT_CASES, build_model

ALL = {**CASES, **CHECKPOINT_CASES}


def _family(plan):
    return "l2" if _lib.l2_csize(plan) else int(plan)


def test_every_raw_plan_at_one_and_twelve_relations():
    have = {(c["plan"], c["R"]) for c in CASES.values() if c["assembly"] == "raw"}
    for plan in (1, 2, 3, 4):
        assert _lib.is_rs(plan)
        for R in (1, 12):
            assert (plan, R) in have, (plan, R)
    assert any(c["R"] == 12 and c["NB"] == 4 and c["assembly"] == "raw" for c in CASES.values())


def test_every_l2_cta_count_and_plan_0():
    have = {c["ctas"] for c in CASES.values() if _lib.l2_csize(c["plan"])}
    assert have >= {1, 2, 4, 8}, have
    assert any(c["plan"] == 0 and c["R"] > 12 for c in CASES.values())
    assert any(_lib.l2_csize(c["plan"]) and c["R"] > 12 and c["NB"] == 2 for c in CASES.values())


def test_widths_layers_and_bases_on_both_assembly_paths():
    for path in ("raw", "row"):
        sub = {n: c for n, c in CASES.items() if c["assembly"] == path}
        assert {4, 6, 8} <= {c["in0"] for c in sub.values()}, path
        assert {1, 4, 8} <= {c["L"] for c in sub.values()}, path
        assert {2, 4} <= {c["NB"] for c in sub.values()}, path
        assert "pyg-2" in {c["rgcn"] for c in sub.values()}, path


def test_both_seeds_on_every_plan_family():
    have = {(_family(c["plan"]), c["seed"]) for c in CASES.values()}
    for fam in (0, 1, 2, 3, 4, "l2"):
        for seed in ("loss", "score"):
            assert (fam, seed) in have, (fam, seed)
    l2 = {(c["ctas"], c["seed"]) for c in CASES.values() if _lib.l2_csize(c["plan"])}
    assert l2 >= {(n, s) for n in (1, 2, 4, 8) for s in ("loss", "score")}, sorted(l2)
    assert {2, 3} <= {c["mb"] for c in CASES.values()}
    assert any(c["scale"] > 1 and c["assembly"] == "raw" for c in CASES.values())


def test_degenerate_batches_and_checkpoints():
    claimed = set().union(*(c["regimes"] for c in CASES.values()))
    assert {"cold_start", "mixed_degenerate", "batch_of_one", "padded_tail", "large_subgraphs",
            "large_pre_activations"} <= claimed
    for path in ("raw", "row"):
        claimed = set().union(*(c["regimes"] for c in CASES.values() if c["assembly"] == path))
        need = {"cold_start", "mixed_degenerate", "padded_tail", "batch_of_one"}
        assert need <= claimed, (path, sorted(need - claimed))
    assert {c["assembly"] for c in CHECKPOINT_CASES.values()} == {"raw", "row"}


@pytest.mark.parametrize("name", sorted(ALL))
def test_declared_plan_fits(name):
    c = ALL[name]
    m = build_model(c, device="cpu")
    lib, cm = _lib.load(), ctypes.byref(m._cmodel)
    assert _lib.ctas_per_graph(c["plan"]) == c["ctas"]
    for backward in (0, 1):
        assert lib.igmc_model_plan(cm, c["n_cap"], c["plan"], backward) > 0, (name, backward)
