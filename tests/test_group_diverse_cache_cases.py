"""The group, diversity and cached-list cases of tests/group_diverse_cache_cases.py, checked without a GPU.

* every case reaches the regimes it claims, re-derived from its data alone, and between them the cases of each kernel
  reach every regime that kernel branches on;
* the launch constants the regimes depend on equal the constexprs of csrc/groups.cu, csrc/diverse.cu and
  csrc/recommend_cache.cu, so a changed block size flags the cases before they silently stop reaching a chunk boundary;
* the host twins of igmc_b200/recommend.py agree with the brute-force enumerations on every valid case the host can
  enumerate, so the twins the GPU tests compare with are held to the header's contracts at these regimes too."""
import os

import numpy as np
import pytest

from igmc_b200 import recommend as rc
from tests import group_diverse_cache_cases as gc
from tests import support
from tests.ranking_cases import same_f32

CASES = gc.all_cases()


def _of(kernel, host=True):
    return [c for c in CASES if c["kernel"] == kernel and not (host and c.get("graph") == "big")]


@pytest.mark.parametrize("case", CASES, ids=support.pid)
def test_case_reaches_its_regimes(case):
    got = gc.REGIMES[case["kernel"]](case)
    assert case["claims"] <= got, (case["claims"] - got)


def test_every_regime_is_reached():
    reached = {k: set() for k in gc.REQUIRED}
    for c in CASES:
        reached[c["kernel"]] |= c["claims"]
    for kernel, need in gc.REQUIRED.items():
        assert need <= reached[kernel], (kernel, need - reached[kernel])


def test_claims_are_declared_not_derived():
    support.claims_are_declared(gc, CASES)


def test_launch_constants_match_the_sources():
    support.launch_constants_match(gc.CONSTANTS)


def test_the_count_grid_is_what_the_cases_pass():
    with open(os.path.join(support.CSRC, "diverse.cu")) as f:
        assert "min(G->num_users, %d)" % gc.COUNT_GRID in f.read()
    assert gc.COUNT_NU > gc.COUNT_GRID and max(gc.LONG_ROWS) >= gc.COUNT_GRID


def test_the_degree_sum_case_wraps_an_int32():
    """64 copies of the long row sum past 2^31 - 1: in int32 the sum would wrap to a negative total below cap"""
    c = next(c for c in CASES if c["name"] == "one group past 2^31")
    total = 64 * gc.BIG_DEG
    assert total > 2 ** 31 - 1 and np.int64(total).astype(np.int32) < 0
    assert gc.group_rows_reference(c, *(c["rp"], np.arange(gc.BIG_DEG)))[2] == gc.ERR


# ---- the host twins against the brute force -----------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in _of("group_rows") if "bad_member" not in c["claims"]], ids=support.pid)
def test_group_rows_twin(case):
    rp, ci = gc.graph_of(case)
    want_rp, want_ci, err = gc.group_rows_reference(case)
    got_rp, got_ci = rc.group_rows_host(rp, ci, case["members"])
    if err:                                    # the twin has no capacity: the groups that fit are the same
        for g in np.flatnonzero(np.diff(want_rp) > 0):
            assert np.array_equal(got_ci[got_rp[g]:got_rp[g + 1]], want_ci[want_rp[g]:want_rp[g + 1]])
        return
    assert np.array_equal(got_rp, want_rp) and np.array_equal(got_ci, want_ci)


@pytest.mark.parametrize("case", [c for c in _of("group_pairs") if not c["invalid"]], ids=support.pid)
def test_group_pairs_twin(case):
    want, err = gc.group_pairs_reference(case)
    assert err == 0
    got = rc.group_pairs_host(case["members"], case["num_items"], case["unit_g"], case["unit_v"], case["unit_tag"],
                              case["B"])
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


@pytest.mark.parametrize("agg", ["mean", "min", "max"])
@pytest.mark.parametrize("case", _of("group_stats"), ids=support.pid)
def test_group_stats_twin(case, agg):
    want = gc.group_stats_reference(case, agg)
    with np.errstate(all="ignore"):
        key, xs, utag = rc.group_stats_host(case["preds"], case["K"], case["B"], case["M"], agg, case["tag"])
    assert same_f32(key, [k for k, _, _ in want])
    assert same_f32(xs, [[np.nan if v is None else v for v in x] for _, x, _ in want])
    assert np.array_equal(utag, [t for _, _, t in want])


def test_group_mean_differs_from_an_fp32_sum():
    """the cancellation unit: 1e8 + 1 - 1e8 is 1 in fp64 (mean 1/3) and 0 in fp32 (mean 0)"""
    c = next(c for c in CASES if c["name"] == "Gu=300 M=64 K=1 specials")
    want = gc.group_stats_reference(c, "mean")
    assert want[1][0] == gc.f32(1 / 3) and want[0][0] == gc.FLT_MAX and want[11][0] == 0.0


@pytest.mark.parametrize("case", [c for c in _of("item_union") if "bad_id" not in c["claims"]], ids=support.pid)
def test_item_union_twin(case):
    mp, lst, err = gc.item_union_reference(case)
    got_mp, got_lst, bad = rc.item_union_host(case["items"], case["num_items"])
    assert err == 0 and not bad
    assert np.array_equal(got_mp, mp) and np.array_equal(got_lst, lst)


@pytest.mark.parametrize("case", _of("cocount"), ids=support.pid)
def test_cocount_twin(case):
    want, code = gc.cocount_reference(case)
    if code:
        return
    rp, ci = gc.count_graph()
    got = rc.cocount_host(rp, ci, gc.COUNT_NU, gc.COUNT_NI, case["union"])
    assert np.array_equal(got, np.asarray(want, np.uint32))


def test_huge_reference_footing():
    """the union indices of HUGE_ITEMS put t(i, j) past 2^31 - 1, where an int32 product would wrap"""
    nz, cos = gc.huge_reference()
    assert max(nz) >= 2 ** 31 and (np.diag(cos)[[0, 1, 2, 3, 4]] == 1).all()
    i = 65534
    assert i * (2 * gc.HUGE_NU - i - 1) > 2 ** 32


@pytest.mark.parametrize("case", [c for c in _of("select") if "bad_id" not in c["claims"]], ids=support.pid)
def test_diverse_select_twin(case):
    rp, ci = gc.select_graph()
    cp, _ = gc.columns(rp, ci, gc.SEL_NI)
    union = gc.select_union(case)
    mp, lst, _ = rc.item_union_host(union, gc.SEL_NI)
    table = rc.cocount_host(rp, ci, gc.SEL_NU, gc.SEL_NI, lst)
    want = gc.select_reference(case)
    got = rc.diverse_select_host(cp, case["pool_item"], case["pool_score"], case["k"], case["penalty"], mp, table,
                                 len(lst))
    assert want[3] == 0 and not got[3].any()
    assert np.array_equal(got[0], want[0]) and same_f32(got[1], want[1]) and same_f32(got[2], want[2])


@pytest.mark.parametrize("case", _of("cosine"), ids=support.pid)
def test_item_cosine_twin(case):
    rp, ci = gc.select_graph()
    cp, _ = gc.columns(rp, ci, gc.SEL_NI)
    got = rc.item_similarity_host(rp, ci, cp, gc.SEL_NU, gc.SEL_NI, case["items"])
    assert same_f32(got, gc.cosine_reference(case))


@pytest.mark.parametrize("case", [c for c in _of("rescore") if "edit:bad" not in c["claims"]], ids=support.pid)
def test_rescore_plan_twin(case):
    rp, ci = gc.cache_graph(case["num_items"])
    off, items, full, totals, err = gc.rescore_reference(case)
    assert err == 0
    g_off, g_items, g_full, g_total = rc.rescore_plan_host(rp, ci, case["num_items"], case["users"], case["edit_u"],
                                                           case["edit_v"], case["cand"], case["exclude"])
    assert np.array_equal(g_off, off) and np.array_equal(g_items, items) and np.array_equal(g_full, full)
    assert (int(g_off[-1]), g_total) == totals


@pytest.mark.parametrize("case", _of("invalidate"), ids=support.pid)
def test_cache_invalidate_twin(case):
    want = gc.invalidate_reference(case)
    got = rc.cache_invalidate_host(case["user_off"], case["resc"], case["full"], case["complete"], case["top_s"],
                                   case["top_i"])
    for g, w in zip(got, want):
        assert same_f32(g, w) if g.dtype == np.float32 else np.array_equal(g, w)


@pytest.mark.parametrize("case", _of("settle"), ids=support.pid)
def test_cache_settle_twin(case):
    want = gc.settle_reference(case)
    got = rc.cache_settle_host(case["thr_s"], case["thr_i"], case["top_s"], case["top_i"], case["k"])
    for g, w in zip(got, want):
        assert same_f32(g, w) if g.dtype == np.float32 else np.array_equal(g, w)


@pytest.mark.parametrize("case", _of("ws_bytes"), ids=support.pid)
def test_ws_bytes_reference_is_the_largest_fitting_chunk(case):
    q, pool, ni, bound = case["args"]
    nbytes, c = gc.ws_reference(case)
    cap = bound if bound > 0 else gc.DIVERSE_WS_DEFAULT
    assert 1 <= c <= q and nbytes == gc._bytes_of(c, pool, ni)
    assert c == q or gc._bytes_of(c + 1, pool, ni) > cap
    assert c == 1 or nbytes <= cap
