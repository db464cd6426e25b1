"""The draw, counterfactual and online-draw kernels against brute-force enumeration (tests/draw_cases.py,
tests/counterfactual_cases.py, tests/online_cases.py).

igmc_draws_expand, igmc_draws_mask, igmc_draws_stats, igmc_counterfactual_pairs, igmc_counterfactual_select,
igmc_online_draw and igmc_online_recent_append are called directly on buffers built here, on every case: every output
buffer pre-filled with a sentinel and sized past what the kernel may write, the guard checked; integers compared
exactly and floats bit for bit through their int32 view (NaN as NaN); the error word read after every case.  Each
entry point's argument checks are asserted once."""
import ctypes as C

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200.util_functions import _stream_ptr
from tests import counterfactual_cases as cc
from tests import draw_cases as dc
from tests import online_cases as oc
from tests import support
from tests.ranking_cases import same_f32

pytestmark = pytest.mark.gpu

GUARD = 64
S32, S64, S8, SF = -777, -(2 ** 40) - 7, 0xAB, -7.5     # sentinels: no kernel writes any of them


def _with_guard(a, value):
    a = np.asarray(a)
    return np.concatenate([a.reshape(-1), np.full(GUARD, value, a.dtype)])


def _exact(t, want, value):
    """t holds want, then its guard entries untouched"""
    got = t.cpu().numpy()
    w = _with_guard(np.asarray(want).astype(got.dtype), value)
    assert got.shape == w.shape and np.array_equal(got, w), np.flatnonzero(got != w)[:5]


@pytest.fixture
def err():
    yield torch.zeros(1, dtype=torch.int32, device="cuda")


def _take_err(e):
    """the error word, then zeroed"""
    torch.cuda.synchronize()
    v = int(e.item())
    e.zero_()
    return v


# ---- igmc_draws_expand ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in dc.all_cases() if c["kernel"] == "expand"], ids=support.name_id)
def test_draws_expand(case):
    support.assert_claims(dc.REGIMES, case)
    lib = _lib.load()
    S, B = case["S"], case["B"]
    ins = [support.dev_np(support.nonempty(case[k]), dt) for k, dt in
           (("pair_u", np.int32), ("pair_v", np.int32), ("pair_pid", np.int64), ("pair_tag", np.int64))]
    sent = (S32, S32, S64, S64, S32)
    outs = [support.filled(B, s, d, GUARD)
            for s, d in zip(sent, (torch.int32, torch.int32, torch.int64, torch.int64, torch.int32))]
    assert lib.igmc_draws_expand(S, B, *(t.data_ptr() for t in ins + outs), _stream_ptr()) == 0
    for o, w, s in zip(outs, dc.expand_reference(case), sent):
        _exact(o, w, s)


# ---- igmc_draws_mask --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in dc.all_cases() if c["kernel"] == "mask"], ids=support.name_id)
def test_draws_mask(case):
    """p = 1 keeps no edge, the one whose hash has all 32 high bits set included; a hash at the threshold is kept,
    one below it dropped"""
    support.assert_claims(dc.REGIMES, case)
    lib = _lib.load()
    ep = case["edge_ptr"]
    B, E = len(ep) - 1, int(ep[-1])
    dep = support.dev_np(support.nonempty(ep), np.int32)
    O = _lib.BatchOut()
    O.edge_ptr = dep.data_ptr()
    pid, tag, draw = (support.dev_np(support.nonempty(case[k]), dt)
                      for k, dt in (("pair_id", np.int64), ("tag", np.int64), ("draw", np.int32)))
    ek, hk = support.filled(E, S8, torch.uint8, GUARD), support.filled(B * dc.LIN1_OUT, S8, torch.uint8, GUARD)
    assert lib.igmc_draws_mask(C.byref(O), B, pid.data_ptr(), tag.data_ptr(), draw.data_ptr(), case["p"], case["seed"],
                               ek.data_ptr(), hk.data_ptr(), _stream_ptr()) == 0
    wek, whk = dc.mask_reference(case)
    _exact(ek, wek, S8)
    _exact(hk, whk, S8)


# ---- igmc_draws_stats -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in dc.all_cases() if c["kernel"] == "stats"], ids=support.name_id)
def test_draws_stats(case):
    support.assert_claims(dc.REGIMES, case)
    lib = _lib.load()
    K, B, S = case["K"], case["B"], case["S"]
    dp = support.dev_np(support.nonempty(case["preds"].reshape(-1)), np.float32)
    dt = support.dev_np(support.nonempty(case["tag"]), np.int64)
    want = dc.stats_outputs(case, SF)
    if case["mode"] == "key":
        key = support.filled(B // S, SF, torch.float32, GUARD)
        assert lib.igmc_draws_stats(dp.data_ptr(), K, B, S, dt.data_ptr(), case["beta"], None, None, None,
                                    key.data_ptr(), _stream_ptr()) == 0
        assert same_f32(key.cpu().numpy(), _with_guard(want, SF))
        return
    outs = [support.filled(len(w), SF, torch.float32, GUARD) for w in want]
    assert lib.igmc_draws_stats(dp.data_ptr(), K, B, S, dt.data_ptr(), case["beta"], *(o.data_ptr() for o in outs),
                                None, _stream_ptr()) == 0
    for o, w, name in zip(outs, want, ("value", "mean", "std")):
        assert same_f32(o.cpu().numpy(), _with_guard(w, SF)), name


# ---- igmc_counterfactual_pairs / _select -----------------------------------------------------------------------------
def _cf_query(case, size=None, removed=None):
    """igmc_counterfactual_t of a case (size / removed: device tensors to use); (struct, keep-alive)"""
    keep = [*(support.dev_np(support.nonempty(case[k]), np.int32) for k in ("users", "items", "rivals")),
            size if size is not None else support.dev_np(support.nonempty(case["size"]), np.int32),
            removed if removed is not None else support.dev_np(support.nonempty(case["removed"].reshape(-1)),
                                                               np.int32)]
    return _lib.Counterfactual(*(t.data_ptr() for t in keep), len(case["users"]), case["M"]), keep


@pytest.mark.parametrize("case", [c for c in cc.all_cases() if c["kernel"] == "cf_pairs"], ids=support.name_id)
def test_counterfactual_pairs(case, err):
    support.assert_claims(cc.REGIMES, case)
    lib = _lib.load()
    G, keep_g = support.csr_struct(*cc.graph(), cc.NU, cc.NI)
    Q, keep_q = _cf_query(case)
    off = support.dev_np(support.nonempty(case["offsets"]), np.int64)
    B = case["B"]
    for pos in case["cursors"]:
        row_cap = cc.row_cap_of(case, pos)
        u, v, pid, tag, ru, rptr, rcol, rrat, werr, rows = cc.pairs_reference(case, pos, row_cap)
        cursor = torch.tensor([pos], dtype=torch.int64, device="cuda")
        lu, lv, dru, sess = (support.filled(B, S32, torch.int32, GUARD) for _ in range(4))
        dpid, dtag = support.filled(B, S64, torch.int64, GUARD), support.filled(B, S64, torch.int64, GUARD)
        drp = support.filled(B + 1, S32, torch.int32, GUARD)
        dcol, drat = support.filled(row_cap, S32, torch.int32, GUARD), support.filled(row_cap, S8, torch.uint8, GUARD)
        assert lib.igmc_counterfactual_pairs(C.byref(G), C.byref(Q), off.data_ptr(), case["step"], cursor.data_ptr(), B,
                                             lu.data_ptr(), lv.data_ptr(), dpid.data_ptr(), dtag.data_ptr(),
                                             dru.data_ptr(), drp.data_ptr(), dcol.data_ptr(), drat.data_ptr(), row_cap,
                                             sess.data_ptr(), err.data_ptr(), _stream_ptr()) == 0
        assert _take_err(err) == werr, pos
        assert int(cursor.item()) == pos + B
        for t, w, s in ((lu, u, S32), (lv, v, S32), (dpid, pid, S64), (dtag, tag, S64), (dru, ru, S32),
                        (sess, np.arange(B), S32)):
            _exact(t, w, s)
        got_col, got_rat = dcol.cpu().numpy(), drat.cpu().numpy()
        assert (got_col[row_cap:] == S32).all() and (got_rat[row_cap:] == S8).all()   # nothing past row_cap
        if not rows:
            continue                    # ids outside G or a candidate past the row: the rows are left open
        _exact(drp, rptr, S32)
        n = int(rptr[-1])
        if n <= row_cap:
            assert np.array_equal(got_col[:n], rcol) and np.array_equal(got_rat[:n], rrat), pos


@pytest.mark.parametrize("case", [c for c in cc.all_cases() if c["kernel"] == "cf_select"], ids=support.name_id)
def test_counterfactual_select(case, err):
    support.assert_claims(cc.REGIMES, case)
    lib = _lib.load()
    G, keep_g = support.csr_struct(*cc.graph(), cc.NU, cc.NI)
    want, werr, _ = cc.select_reference(case)
    Qn, M = len(case["users"]), case["M"]
    start = dict(removed=(case["removed"], S32, np.int32), size=(case["size"], S32, np.int32),
                 count=(np.full(Qn, cc.S32), S32, np.int32), found=(np.full(Qn, 0xAB), S8, np.uint8),
                 items=(np.full(Qn * M, cc.S32), S32, np.int32), ratings=(np.full(Qn * M, cc.S32), S32, np.int32),
                 score=(np.full(Qn * (M + 1), cc.SF), SF, np.float32),
                 rival_score=(np.full(Qn * (M + 1), cc.SF), SF, np.float32))
    dev = {k: support.dev_np(_with_guard(np.asarray(a).astype(d), s), d) for k, (a, s, d) in start.items()}
    Q, keep_q = _cf_query(case, dev["size"], dev["removed"])
    off = support.dev_np(support.nonempty(case["offsets"]), np.int64)
    sc = support.dev_np(support.nonempty(case["scores"]), np.float32)
    assert lib.igmc_counterfactual_select(C.byref(G), C.byref(Q), off.data_ptr(), sc.data_ptr(), case["step"],
                                          *(dev[k].data_ptr() for k in ("count", "found", "items", "ratings", "score",
                                                                        "rival_score")),
                                          err.data_ptr(), _stream_ptr()) == 0
    assert _take_err(err) == werr
    for k, w in want.items():
        if k in ("score", "rival_score"):
            assert same_f32(dev[k].cpu().numpy(), _with_guard(w, np.float32(SF))), k
        else:
            _exact(dev[k], w, start[k][1])


# ---- igmc_online_draw / igmc_online_recent_append ---------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in oc.all_cases() if c["kernel"] == "online_draw"], ids=support.name_id)
def test_online_draw(case, err):
    support.assert_claims(oc.REGIMES, case)
    lib = _lib.load()
    G, keep_g = support.csr_struct(*oc.graph(case["empty"]))
    ring_u, ring_v = (support.dev_np(support.nonempty(r), np.int32) for r in case["ring"][:2])
    total = torch.tensor([case["total"]], dtype=torch.int64, device="cuda")
    step = torch.tensor([case["step_count"]], dtype=torch.int64, device="cuda")
    B = case["B"]
    lu, lv, lab = (support.filled(B, S32, torch.int32, GUARD) for _ in range(3))
    pid, seeds = support.filled(B, S64, torch.int64, GUARD), support.filled(3, S64, torch.int64, GUARD)
    assert lib.igmc_online_draw(C.byref(G), ring_u.data_ptr(), ring_v.data_ptr(), case["capacity"], total.data_ptr(),
                                case["thresh"], step.data_ptr(), case["step_ahead"], case["sample_seed"],
                                case["drop_seed"], B, lu.data_ptr(), lv.data_ptr(), lab.data_ptr(), pid.data_ptr(),
                                seeds.data_ptr(), err.data_ptr(), _stream_ptr()) == 0
    u, v, wlab, wpid, wseeds, werr, _ = oc.draw_reference(case)
    assert _take_err(err) == werr
    for t, w, s in ((lu, u, S32), (lv, v, S32), (lab, wlab, S32), (pid, wpid, S64), (seeds, wseeds.view(np.int64), S64)):
        _exact(t, w, s)
    assert int(total.item()) == case["total"] and int(step.item()) == case["step_count"]


@pytest.mark.parametrize("case", [c for c in oc.all_cases() if c["kernel"] == "append"], ids=support.name_id)
def test_recent_append(case, err):
    """call after call: the ring, its count and the error word"""
    support.assert_claims(oc.REGIMES, case)
    lib = _lib.load()
    cap = case["capacity"]
    ring_u, ring_v = (support.filled(cap, oc.RING_SENT, torch.int32, GUARD) for _ in range(2))
    total = torch.tensor([case["total"]], dtype=torch.int64, device="cuda")
    for (u, v, x), (wu, wv, wt, werr) in zip(case["calls"], oc.append_reference(case)):
        D = len(u)
        ins = [support.dev_np(support.nonempty(a), np.int32) for a in (u, v, x)]
        ptrs = [t.data_ptr() for t in ins] if D else [None] * 3     # D = 0: no launch, no inputs needed
        assert lib.igmc_online_recent_append(*ptrs, D, ring_u.data_ptr(), ring_v.data_ptr(), cap, total.data_ptr(),
                                             err.data_ptr(), _stream_ptr()) == 0
        assert _take_err(err) == werr
        _exact(ring_u, wu, oc.RING_SENT)
        _exact(ring_v, wv, oc.RING_SENT)
        assert int(total.item()) == wt


# ---- argument checks --------------------------------------------------------------------------------------------------
def test_argument_checks(err):
    """each entry point's -1 / -2 (igmc_online_draw: -1 .. -5) returns, decided on the host before any launch"""
    lib = _lib.load()
    st = _stream_ptr()
    buf = torch.zeros(4096, dtype=torch.int64, device="cuda")
    p = buf.data_ptr()
    # igmc_draws_expand: 1 <= S <= IGMC_DRAWS_MAX, S <= B, no NULL buffer
    for S, B in ((0, 4), (dc.DRAWS_MAX + 1, 300), (4, 3)):
        assert lib.igmc_draws_expand(S, B, *([p] * 9), st) == -1, (S, B)
    assert lib.igmc_draws_expand(1, 4, *([p] * 8), None, st) == -1
    # igmc_draws_mask: B > 0 and edge_ptr given (-1); 0 <= adj_dropout <= 1 (-2)
    O = _lib.BatchOut()
    O.edge_ptr = p
    assert lib.igmc_draws_mask(C.byref(O), 0, p, p, p, 0.5, 0, p, p, st) == -1
    assert lib.igmc_draws_mask(C.byref(_lib.BatchOut()), 1, p, p, p, 0.5, 0, p, p, st) == -1
    for bad in (1.5, -0.1, float("nan"), float("inf")):
        assert lib.igmc_draws_mask(C.byref(O), 1, p, p, p, bad, 0, p, p, st) == -2, bad
    # igmc_draws_stats: K >= 1, S in range, key or all of value / mean / std (-1); beta finite (-2)
    assert lib.igmc_draws_stats(p, 0, 4, 2, p, 0.0, None, None, None, p, st) == -1
    assert lib.igmc_draws_stats(p, 1, 300, dc.DRAWS_MAX + 1, p, 0.0, None, None, None, p, st) == -1
    assert lib.igmc_draws_stats(p, 1, 4, 2, p, 0.0, p, p, None, None, st) == -1
    for bad in (float("nan"), float("inf"), -float("inf")):
        assert lib.igmc_draws_stats(p, 1, 4, 2, p, bad, None, None, None, p, st) == -2, bad
    # igmc_counterfactual_pairs / _select: a query set with 1 <= max_removals <= 256, B > 0, step >= 0, buffers (-1)
    G, keep_g = support.csr_struct(*cc.graph(), cc.NU, cc.NI)
    for nq, M in ((0, 4), (1, 0), (1, cc.CF_MAX + 1)):
        Q = _lib.Counterfactual(p, p, p, p, p, nq, M)
        assert lib.igmc_counterfactual_pairs(C.byref(G), C.byref(Q), p, 1, p, 4, *([p] * 8), 16, p, p, st) == -1
        assert lib.igmc_counterfactual_select(C.byref(G), C.byref(Q), p, p, 1, *([p] * 6), p, st) == -1
    Q = _lib.Counterfactual(p, p, p, p, p, 1, 4)
    for B, step, cap, col in ((0, 1, 16, p), (4, -1, 16, p), (4, 1, 16, None), (4, 1, -1, p)):
        assert lib.igmc_counterfactual_pairs(C.byref(G), C.byref(Q), p, step, p, B, p, p, p, p, p, p, col, p, cap, p,
                                             p, st) == -1, (B, step, cap)
    assert lib.igmc_counterfactual_select(C.byref(G), C.byref(Q), p, p, -1, *([p] * 6), p, st) == -1
    assert lib.igmc_counterfactual_select(C.byref(G), C.byref(Q), p, p, 1, None, *([p] * 5), p, st) == -1
    # igmc_online_draw: the graph (-1), the ring (-2), recent_thresh in [0, 2^32] (-3), the step (-4), the outputs (-5)
    Go, keep_o = support.csr_struct(*oc.graph())
    args = dict(G=C.byref(Go), ru=p, rv=p, cap=8, total=p, thresh=2 ** 31, step=p, ahead=0, B=4, err=err.data_ptr())

    def draw(**kw):
        a = dict(args, **kw)
        return lib.igmc_online_draw(a["G"], a["ru"], a["rv"], a["cap"], a["total"], a["thresh"], a["step"],
                                    a["ahead"], 1, 2, a["B"], p, p, p, p, p, a["err"], st)
    assert draw(G=C.byref(_lib.CSR(None, p, p, None, None, 1, 1))) == -1
    assert draw(cap=0) == -2 and draw(ru=None) == -2
    assert draw(thresh=-1) == -3 and draw(thresh=2 ** 32 + 1) == -3
    assert draw(step=None) == -4 and draw(ahead=-1) == -4
    assert draw(B=0) == -5 and draw(err=None) == -5
    # igmc_online_recent_append: D >= 0 with inputs (-1), the ring and the error word (-2)
    assert lib.igmc_online_recent_append(p, p, p, -1, p, p, 8, p, p, st) == -1
    assert lib.igmc_online_recent_append(None, p, p, 3, p, p, 8, p, p, st) == -1
    assert lib.igmc_online_recent_append(p, p, p, 3, p, p, 0, p, p, st) == -2
    assert lib.igmc_online_recent_append(p, p, p, 3, p, p, 8, p, None, st) == -2
    torch.cuda.synchronize()
    assert _take_err(err) == 0 and not buf.any()          # nothing was launched
