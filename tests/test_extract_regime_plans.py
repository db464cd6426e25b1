"""The extraction plan (igmc_extract_plan, csrc/extract.cu) against a restatement of its two formulas, and the cases of
tests/test_gpu_extract_regimes.py on the side of each boundary they claim, from host quantities alone (no GPU).  If the
extraction kernels are retuned (shared-memory budget, tile table, canonical buffer, class limit), this file fails
before the GPU cases silently stop covering a branch."""
import itertools

import numpy as np
import pytest

from igmc_b200 import _lib
from tests import test_gpu_extract_regimes as R_

# restated from csrc/extract.cu: one-launch tiles, tile table, canonical edges in shared memory, 12-bit local ids,
# rating classes (ballot lanes), and the shared-memory budgets of the one-launch and the generic kernels
FX_TILE, FX_TCAP, FX_CANO, FX_MAXCAP, FX_MAXR = 128, 2048, 12288, 4095, 32
FAST_SMEM, GENERIC_SMEM = 110 * 1024, 220 * 1024


def _r16(x):
    return (x + 15) & ~15


def fast_smem(num_items, B, h, cap, R, max_row_deg, edge_cap):
    """fast_smem: the one-launch kernel's tables (FastSmem) plus the item table, 0 when a limit is exceeded"""
    words = (cap + 31) // 32
    ints = 4 * cap + 4 * (cap + 1) + cap * max(R, 1) + cap * max(R, 1) * words + (FX_TCAP + 1) + FX_TCAP + FX_CANO
    smem = 4 * ints + _r16(2 * num_items)
    rows = cap * (max_row_deg if max_row_deg > 0 else num_items)
    ok = (h == 1 and 1 <= R <= FX_MAXR and cap <= FX_MAXCAP and rows <= FX_TILE * FX_TCAP and smem <= FAST_SMEM
          and edge_cap // B >= 2)
    return smem if ok else 0


def generic_fits(num_users, num_items, h, cap):
    """generic_smem: the item table (h = 1) plus the visited / candidate bitmaps and fringe list (h > 1)"""
    a = 4 * cap + 2 * num_items
    if h > 1:
        wu, wv = (num_users + 31) // 32, (num_items + 31) // 32
        a = _r16(a) + 4 * (wu + wv + max(wu, wv)) + 4 * max(num_users, num_items)
        if a > GENERIC_SMEM:
            return False
    return 8 * cap + 2 * num_items <= GENERIC_SMEM


def plan_restated(num_users, num_items, B, h, cap, R, max_row_deg, edge_cap):
    f = fast_smem(num_items, B, h, cap, R, max_row_deg, edge_cap)
    return f if f else 0 if generic_fits(num_users, num_items, h, cap) else -3


def plan_lib(*args, fast=1, adjacency=1):
    return _lib.load().igmc_extract_plan(*args, fast, adjacency)


def largest_fast_cap(R, items, max_row_deg=1):
    return max([c for c in range(1, FX_MAXCAP + 1) if plan_lib(10, items, 1, 1, c, R, max_row_deg, 1 << 20) > 0],
               default=0)


def test_plan_agrees_with_the_restatement():
    for cap, R, items, deg, h, users in itertools.product(
            (1, 31, 32, 33, 82, 83, 140, 141, 201, 206, 207, 224, 225, 469, 470, 4095, 4096),
            (0, 1, 5, 12, 32, 33), (1, 1000, 3706, 23520, 23521, 111836, 111837), (0, 1, 1180, 1181, 5000), (1, 2, 3),
            (1, 35324, 35325)):
        args = (users, items, 8, h, cap, R, deg, 8 * 2 * cap * cap)
        assert plan_lib(*args) == plan_restated(*args), args


def test_plan_switches():
    args = (100, 1000, 8, 1, 224, 5, 200, 8 * 100000)
    assert plan_lib(*args) > 0
    assert plan_lib(*args, fast=0) == 0                 # no one-launch flags: the generic kernels
    assert plan_lib(*args, adjacency=0) == 0            # no message-passing lists: the generic kernels
    assert plan_lib(100, 1000, 8, 1, 224, 5, 200, 8) == 0    # scratch slot below two edges per graph
    assert plan_lib(*args[:4], 0, *args[5:]) == -2 and plan_lib(*args[:4], 65535, *args[5:]) == -2
    assert plan_lib(*args[:3], 0, *args[4:]) == -4 and plan_lib(*args[:3], 4, *args[4:]) == -4
    assert plan_lib(*args[:2], 0, *args[3:]) == 0       # an empty batch launches nothing


def test_boundaries_of_the_issue_numbers():
    """the largest cap the one-launch path takes, and the catalogue limits of the generic path"""
    assert largest_fast_cap(5, 1000) == 224 and largest_fast_cap(5, 3706) == 206
    assert largest_fast_cap(12, 1000) == 140 and largest_fast_cap(32, 1000) == 82
    assert largest_fast_cap(1, 23520) > 0 and largest_fast_cap(1, 23521) == 0
    assert plan_lib(30, 111836, 8, 1, 201, 5, 200, 1 << 20) == 0 and plan_lib(30, 111837, 8, 1, 201, 5, 200, 1 << 20) < 0
    assert plan_lib(35324, 35324, 8, 2, 21, 5, 15, 1 << 20) == 0
    assert plan_lib(35325, 35325, 8, 2, 21, 5, 15, 1 << 20) < 0
    # the tile table at cap 222: rows of 1 180 pass, 1 181 do not
    assert plan_lib(222, 1200, 8, 1, 222, 5, 1180, 1 << 24) > 0 and plan_lib(222, 1200, 8, 1, 222, 5, 1181, 1 << 24) == 0


def test_local_id_limit_is_never_reached_on_the_one_launch_path():
    """local ids travel in 12 bits (FX_MAXCAP = 4 095): shared memory binds long before, at every R >= 1, even with an
    empty catalogue and rows of one rating"""
    for R in range(1, FX_MAXR + 1):
        c = largest_fast_cap(R, 0)
        assert 0 < c < FX_MAXCAP, (R, c)
        assert fast_smem(0, 1, 1, c + 1, R, 1, 1 << 20) == 0
    # the smallest table (R = 1, no items) at cap FX_MAXCAP is far past the budget
    words = (FX_MAXCAP + 31) // 32
    assert 4 * (9 * FX_MAXCAP + FX_MAXCAP * words) > FAST_SMEM


def _plan_of(A, cv, B, h, mnph, sess_deg=0):
    """what SubgraphExtractor.plan passes to igmc_extract_plan, from the host graph"""
    from igmc_b200.util_functions import RatingGraph
    G = RatingGraph(A)
    deg = max(G.max_row_deg, sess_deg)
    cap = G.node_cap(mnph, h, deg)
    edges = 2 * min(cap * min(cap, max(deg, 1)), max(G.nnz + sess_deg, 1))
    args = (G.num_users, G.num_items, B, h, cap, len(cv), deg, B * edges)
    got = plan_lib(*args)
    assert got == plan_restated(*args), args
    return cap, got


@pytest.mark.parametrize("name", sorted(R_.CASES))
def test_gpu_case_sits_on_its_side(name):
    c = R_.CASES[name]
    A, (pu, _, _), cv = c["build"]()
    h, _, mnph = R_.case_args(c)
    cap, plan = _plan_of(A, cv, len(pu), h, mnph)
    if c["cap"] is not None:
        assert cap == c["cap"], (name, cap)
    assert R_._side(plan) == c["path"], (name, plan)


@pytest.mark.parametrize("name", sorted(R_.SESSION_CASES))
def test_gpu_session_case_sits_on_its_side(name):
    c = R_.SESSION_CASES[name]
    A, cv, users, edits, pairs = c["build"]()
    rows = R_.session_rows(A, users, edits)
    deg = max(len(r) for r in rows)
    assert deg == c["row_deg"] and min(len(r) for r in rows) == 0
    cap, plan = _plan_of(A, cv, len(pairs), 1, c["mnph"], deg)
    assert cap == c["cap"] and R_._side(plan) == c["path"], (name, cap, plan)


def test_every_regime_is_covered_on_both_sides():
    paths = {}
    for name, c in R_.CASES.items():
        paths.setdefault(name.rsplit("_", 1)[0], set()).add(c["path"])
    assert paths["smem_r5_items1000"] == paths["smem_r12"] == paths["smem_r5_ml1m_items"] == {"fast", "generic"}
    assert paths["tile_table"] == {"fast", "generic"}
    assert paths["items_h1"] == paths["h2"] == {"generic", "none"}
    assert {R_.CASES["classes_r%d" % r]["path"] for r in (1, 32, 33)} == {"fast", "generic"}
    assert {n for n in (31, 32, 33, 64, 65) if "words_%d" % n in R_.CASES} == {31, 32, 33, 64, 65}
    assert {c["path"] for c in R_.SESSION_CASES.values()} == {"fast", "generic"}
