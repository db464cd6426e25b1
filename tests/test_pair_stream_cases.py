"""The pair-stream cases of tests/pair_stream_cases.py, checked without a GPU.

* every case reaches the regimes it claims, re-derived from its data alone, and between them the cases of each kernel
  reach every regime that kernel branches on;
* the launch constants the regimes depend on equal the constexprs of csrc/recommend.cu, csrc/explain.cu and
  csrc/session.cu, so a changed block size flags the cases before they silently stop reaching a chunk boundary;
* the host twins of igmc_b200/recommend.py agree with the brute-force enumerations on the cases they run at a sensible
  size, so the twins other tests rely on are held to the contract at these regimes too."""
import numpy as np
import pytest

from igmc_b200 import recommend as rc
from tests import pair_stream_cases as ps
from tests import support

CASES = ps.all_cases()


def _of(kernel):
    return [c for c in CASES if c["kernel"] == kernel]


@pytest.mark.parametrize("case", CASES, ids=support.pid)
def test_case_reaches_its_regimes(case):
    got = ps.REGIMES[case["kernel"]](case)
    assert case["claims"] <= got, (case["claims"] - got)


def test_every_regime_is_reached():
    reached = {k: set() for k in ps.REQUIRED}
    for c in CASES:
        reached[c["kernel"]] |= c["claims"]
    for kernel, need in ps.REQUIRED.items():
        assert need <= reached[kernel], (kernel, need - reached[kernel])


def test_every_pair_mode_reaches_every_batch_regime():
    """B = 1, 511, 512, 513 and above P, the second stride and the tail in each mode of igmc_candidate_pairs: B = 513
    is only in the small-user cases, so dropping it from them fails here"""
    for mode in ("no_list", "shared", "per_user", "explicit"):
        reached = set().union(*(c["claims"] for c in _of("pairs") if c["mode"] == mode))
        assert ps.PAIR_PER_MODE <= reached, (mode, ps.PAIR_PER_MODE - reached)


def test_claims_are_declared_not_derived():
    support.claims_are_declared(ps, [c for c in CASES if c["name"] != "B=1 P=3"])


def test_launch_constants_match_the_sources():
    support.launch_constants_match(ps.CONSTANTS)


def test_the_big_graph_passes_int64():
    """the full-catalogue plan passes 2^32, the half-catalogue list 2^31; the enumeration at a cursor is exact"""
    full, half = _of("int64")
    assert int(ps.big_user_off(full)[-1]) > 2 ** 32 and 2 ** 31 < int(ps.big_user_off(half)[-1]) < 2 ** 32
    off = ps.big_user_off(full)
    u, v, pid, tag = ps.big_batch(full, 2 ** 32 - 300, off)
    j = int(tag[0])
    assert int(off[j]) <= 2 ** 32 - 300 < int(off[j + 1]) and (tag >= j).all()
    assert (pid == u * ps.BIG_NI + v).all() and (v < ps.BIG_NI).all()


# ---- the host twins against the brute force -----------------------------------------------------------------------------
@pytest.mark.parametrize("case", _of("plan"), ids=support.pid)
def test_plan_twin(case):
    A = ps.plan_graph()
    uo, ro, rp, _ = ps.plan_reference(case)
    hu, hro, hrp = rc.candidate_plan_host(A.indptr, A.indices, A.shape[1], case["users"], case["cand"],
                                          case["exclude"])
    assert np.array_equal(hu, uo)
    assert (hro is None) == (ro is None)
    if ro is not None:
        assert np.array_equal(hro, ro) and np.array_equal(hrp, rp)


@pytest.mark.parametrize("case", _of("lists"), ids=support.pid)
def test_lists_twin(case):
    A = ps.plan_graph()
    uo, lists, _, _ = ps.lists_reference(case)
    hu, hl = rc.candidate_lists_host(A.indptr, A.indices, A.shape[1], case["users"], case["rows"], case["exclude"])
    assert np.array_equal(hu, uo) and np.array_equal(hl, lists)


@pytest.mark.parametrize("case", [c for c in _of("pairs") if c["mode"] in ("no_list", "shared")], ids=support.pid)
def test_pairs_twin(case):
    """the first batch, one across a user boundary and the last two"""
    A = ps.plan_graph()
    P, stream, sets = ps.pairs_stream(case)
    plan = rc.candidate_plan_host(A.indptr, A.indices, A.shape[1], case["users"], case["cand"], case["exclude"])
    B = min(case["B"], 600)
    mid = int(ps.prefix(len(s) for s in sets)[len(sets) // 2]) - B // 2
    for pos in sorted({0, max(mid, 0), max(P - B, 0), P - 1}):
        got = rc.candidate_pairs_host(A.indptr, A.indices, A.shape[1], case["users"], case["cand"], case["exclude"],
                                      plan, pos, B)
        want = ps.batch_of(stream, pos, B, P)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), pos


@pytest.mark.parametrize("case", _of("offsets"), ids=support.pid)
def test_offsets_twin(case):
    assert np.array_equal(rc.explain_offsets_host(case["num_edges"]), ps.offsets_reference(case))


@pytest.mark.parametrize("case", [c for c in _of("occl") if "invalid" not in c["name"]], ids=support.pid)
def test_occlusion_pairs_twin(case):
    off = ps.offsets_reference(case)
    for pos in ps.occl_cursors(case)[:40] + ps.occl_cursors(case)[-3:]:
        got = rc.occlusion_pairs_host(off, case["pair_u"], case["pair_v"], ps.PLAN_NI, pos, case["B"])
        want = ps.occl_batch(case, pos)
        for g, w in zip(got, want[:5]):
            assert np.array_equal(g, w), pos


@pytest.mark.parametrize("case", _of("mask"), ids=support.pid)
def test_mask_twin(case):
    keep, _, _ = ps.mask_reference(case, -1)
    ms = np.asarray(case["ms"])
    j = np.where((case["j"] >= 0) & (case["j"] < ms), case["j"], -1)      # the twin takes j in range as the kernel does
    assert np.array_equal(rc.occlusion_mask_host(case["batch"]["edge_ptr"], case["tag"], j), keep)


@pytest.mark.parametrize("case", [c for c in _of("scatter") if "disagree" not in c["name"]], ids=support.pid)
def test_scatter_twin(case):
    grads = ps.scatter_grads(case)
    outs, _, err = ps.scatter_reference(case, grads, np.float32(0), -1)
    assert err == 0
    out = np.zeros(int(case["offsets"][-1]), np.float32)
    for k in range(case["K"]):
        with np.errstate(all="ignore"):
            rc.edge_grad_scatter_host(case["batch"]["edge_ptr"], case["tag"], grads[k], case["offsets"], out, k,
                                      case["K"])
        g, w = out.view(np.int32), outs[k].view(np.int32)
        assert ((g == w) | (np.isnan(out) & np.isnan(outs[k]))).all(), k


def test_corated_twin_matches_the_enumerated_rows():
    """the rows the engine test expects from retrieve=10, against the retriever's host twin"""
    from igmc_b200.data import make_synthetic_dataset
    A = make_synthetic_dataset("tiny", seed=0)["adj_train"]
    users = np.concatenate([np.arange(A.shape[0]), [3, 3, 17]])
    want = ps.corated_rows(A, users, 10)
    items, _ = rc.corated_host(A.indptr, A.indices, A.shape[0], A.shape[1], users, 10, True)
    assert np.array_equal(items, want)
