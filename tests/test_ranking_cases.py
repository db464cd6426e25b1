"""The ranking-kernel cases of tests/ranking_cases.py, checked without a GPU.

* every case reaches the regimes it claims, re-derived from its data alone, and between them the cases of each kernel
  reach every regime that kernel branches on;
* the host twins of igmc_b200/recommend.py agree with the brute-force orders written from the header's contracts on
  the same cases, so the twins are held to the contract too."""
import numpy as np
import pytest

from igmc_b200 import recommend as rc
from tests import ranking_cases as rcs
from tests import support

CASES = rcs.all_cases()


@pytest.mark.parametrize("case", CASES, ids=support.pid)
def test_case_reaches_its_regimes(case):
    got = rcs.REGIMES[case["kernel"]](case)
    assert case["claims"] <= got, (case["claims"] - got)


def test_every_regime_is_reached():
    reached = {k: set() for k in rcs.REQUIRED}
    for c in CASES:
        reached[c["kernel"]] |= c["claims"]
    for kernel, need in rcs.REQUIRED.items():
        assert need <= reached[kernel], (kernel, need - reached[kernel])


def test_palettes_hold_what_they_name():
    rng = np.random.default_rng(0)
    z = rcs.palette("signed_zero", 200, rng)
    assert (np.signbit(z) & (z == 0)).any() and (~np.signbit(z) & (z == 0)).any()
    f = rcs.palette("inf", 200, rng)
    assert (f == np.inf).any() and (f == -np.inf).any()
    n = rcs.palette("all_nan", 200, rng)
    assert np.isnan(n).all() and len(np.unique(n.view(np.uint32))) > 3 and np.signbit(n).any()
    s = rcs.palette("subnormal", 200, rng)
    assert ((s != 0) & (np.abs(s) < np.finfo(np.float32).tiny)).any()
    r = rcs.palette("random", 500, rng)
    assert len(np.unique(r)) == 500
    ids = rcs.shuffled_ids(300, rng)
    assert len(np.unique(ids)) == 300 and rcs.ID_MAX in ids and not (np.diff(ids) > 0).all()
    # the K >= 3 entries whose mean depends on the summation order
    p = np.float32([[1], [2 ** 25], [-2 ** 25]])
    assert rcs.ckpt_mean(p)[0] == 0 and rcs.ckpt_mean_reversed(p)[0] == np.float32(1) / 3


def test_topk_fits_boundary_restated():
    """16 + (k + B) * 12 bytes within 227 KB: the boundaries the GPU tests probe"""
    fits = lambda k, B: rcs.MERGE_HEAD + (k + B) * 12 <= rcs.SMEM_MAX
    assert fits(256, 19113) and not fits(256, 19114)
    assert fits(1, 19368) and not fits(1, 19369)
    smem = lambda B: rcs.MERGE_HEAD + (256 + B) * 12
    assert smem(3838) <= rcs.SMEM_DEFAULT < smem(3839)


# ---- the host twins against the brute-force orders ---------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "merge"], ids=support.pid)
def test_merge_twins_match_brute_force(case):
    slot, item, preds = rcs.merge_stream(case)
    s = rcs.ckpt_mean(preds)
    ts, ti = rcs.merge_reference(case, len(slot))
    for j in range(len(case["segs"])):
        sel = slot == j
        ws, wi = rc.rank_host(s[sel], item[sel], case["k"])
        assert np.array_equal(wi, ti[j]) and rcs.same_f32(ws, ts[j], keep_nan_bits=case["K"] == 1), j
    if sum(case["segs"]) * case["k"] <= 60000:     # the rank-counting twin is quadratic: the small streams
        for cuts in case["cuts"]:
            top_s = np.full((len(case["segs"]), case["k"]), -np.inf, np.float32)
            top_i = np.full((len(case["segs"]), case["k"]), -1, np.int64)
            for pr, tag, it, (a, b) in rcs.merge_calls(case, cuts):
                seg_s = rcs.ckpt_mean(pr)
                for j in np.unique(tag[tag >= 0]):
                    sel = tag == j
                    top_s[j], top_i[j] = rc.topk_merge_host(top_s[j], top_i[j], seg_s[sel], it[sel])
                ws, wi = rcs.merge_reference(case, b)
                assert np.array_equal(top_i, wi) and rcs.same_f32(top_s, ws), (cuts, b)


@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "influence"], ids=support.pid)
def test_influence_twin_matches_brute_force(case):
    idx, vals = rcs.influence_stream(case)
    want = rcs.influence_reference(case, len(idx))
    o = np.argsort(idx)                  # the twin's index is the position: hand it the values in id order
    idx, vals = idx[o], vals[o]
    for t in range(min(case["T"], 8)):
        pi, pv, ci, cv = rc.influence_order_host(vals[:, t], case["k"])
        assert np.array_equal(idx[pi[pi >= 0]], want[1][t][pi >= 0]) and (want[1][t][pi < 0] == -1).all()
        assert np.array_equal(idx[ci[ci >= 0]], want[3][t][ci >= 0]) and (want[3][t][ci < 0] == -1).all()
        assert rcs.same_f32(pv, want[0][t], True) and rcs.same_f32(cv, want[2][t], True)


@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "occlusion" and
                                  (sum(c["lengths"]) < 10 ** 5 or c["name"] in ("big m=0 score=True", "big m=1 score=False"))],
                         ids=support.pid)
def test_occlusion_twin_matches_brute_force(case):
    score, occluded, offsets, _, _, _ = rcs.occlusion_data(case)
    order, delta = rcs.occlusion_reference(case)
    d, o = rc.explain_order_host(score, occluded, offsets, case["m"] or None)
    assert rcs.same_f32(d, delta, keep_nan_bits=score is None)
    assert np.array_equal(o, order)


@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "corated" and c["graph"] != "bytes"],
                         ids=support.pid)
def test_corated_twin_matches_brute_force(case):
    A = rcs.GRAPHS[case["graph"]]()
    nu, ni = A.shape
    users = [u for u in case["users"] if 0 <= u < nu]
    items, paths, _ = rcs.corated_reference(dict(case, users=tuple(users)), A)
    wi, wp = rc.corated_host(A.indptr, A.indices, nu, ni, users, case["m"], case["exclude"])
    assert np.array_equal(wi, items) and np.array_equal(wp, paths)
