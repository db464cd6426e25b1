"""igmc_elicit_pairs and igmc_elicit_stats called directly on every case of tests/elicit_cases.py: outputs pre-filled
with sentinels and guard entries past them, compared byte for byte with the numpy twins (which tests/test_elicit_host.py
holds to the brute forces), and the error word read after each case, the invalid ones included."""
import ctypes as C

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from tests import elicit_cases as ec
from tests import support

pytestmark = pytest.mark.gpu

SENT32, SENT8, SENTF = -77, 0xAB, -7.5
GUARD = 16


def _pairs(c, row_cap=None):
    """run igmc_elicit_pairs on case c: (return code, error word, outputs as host arrays incl. guards, row_cap)"""
    rp, ci, rt = ec.csr(c["rows"])
    S = len(c["rows"])
    t2 = rc._target_rows(c["targets"])
    W, A, B = t2.shape[1], c["A"], c["B"]
    L = max(len(r) for r in c["rows"]) + 1
    cap = (B // W) * L if row_cap is None else row_cap
    keep = [support.dev(c["users"], torch.int32), support.dev(rp, torch.int32), support.dev(np.r_[ci, 0], torch.int32),
            support.dev(np.r_[rt, 0], torch.uint8)]
    Sd = _lib.Sessions(*(t.data_ptr() for t in keep), S, L - 1)
    targets = support.dev(t2, torch.int32)
    us, uq = support.dev(c["unit_s"], torch.int32), support.dev(c["unit_q"], torch.int32)
    ut = support.dev(c["unit_tag"], torch.int64)
    out = dict(u=support.filled(B, SENT32, torch.int32), v=support.filled(B, SENT32, torch.int32),
               pid=support.filled(B, SENT32, torch.int64), tag=support.filled(B, SENT32, torch.int64),
               ru=support.filled(B, SENT32, torch.int32), rptr=support.filled(B + 1, SENT32, torch.int32),
               rcol=support.filled(cap, SENT32, torch.int32), rrat=support.filled(cap, SENT8, torch.uint8),
               sess=support.filled(B, SENT32, torch.int32))
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    rc_ = _lib.load().igmc_elicit_pairs(C.byref(Sd), c["num_items"], A, targets.data_ptr(), W, int(len(t2) > 1),
                                        us.data_ptr(), uq.data_ptr(), ut.data_ptr(), B, out["u"].data_ptr(),
                                        out["v"].data_ptr(), out["pid"].data_ptr(), out["tag"].data_ptr(),
                                        out["ru"].data_ptr(), out["rptr"].data_ptr(), out["rcol"].data_ptr(),
                                        out["rrat"].data_ptr(), cap, out["sess"].data_ptr(), err.data_ptr(), None)
    torch.cuda.synchronize()
    return rc_, int(err.item()), {k: v.cpu().numpy() for k, v in out.items()}, cap


@pytest.mark.parametrize("case", ec.pair_cases(), ids=lambda c: c["name"])
def test_pairs_kernel_matches_twin(case):
    c = case
    code, err, o, cap = _pairs(c)
    assert code == 0 and err == 0
    rp, ci, rt = ec.csr(c["rows"])
    B, A = c["B"], c["A"]
    out, sess, (ru, wptr, wcol, wrat) = rc.elicit_pairs_host(rp, ci, rt, c["users"], c["num_items"], A, c["targets"],
                                                             c["unit_s"], c["unit_q"], c["unit_tag"], B)
    R = len(ru)                                                         # G * A trial rows
    for k, want in (("u", out[0]), ("v", out[1]), ("pid", out[2]), ("tag", out[3]), ("sess", sess)):
        assert np.array_equal(o[k][:B], want), k
    assert np.array_equal(o["ru"][:R], ru) and np.array_equal(o["rptr"][:R + 1], wptr)
    n = int(wptr[-1])
    assert np.array_equal(o["rcol"][:n], wcol) and np.array_equal(o["rrat"][:n], wrat)
    for k, end, sent in (("u", B, SENT32), ("v", B, SENT32), ("pid", B, SENT32), ("tag", B, SENT32),
                         ("sess", B, SENT32), ("ru", R, SENT32), ("rptr", R + 1, SENT32), ("rcol", n, SENT32),
                         ("rrat", n, SENT8)):
        assert (o[k][end:] == sent).all(), k                           # nothing written past the outputs


def _bad(**change):
    c = dict(ec.pair_cases()[0])
    c.update(change)
    return c


@pytest.mark.parametrize("name,case,row_cap", [
    ("rated question", _bad(unit_q=[0, 7, 5, 4, 1]), None),
    ("session out of range", _bad(unit_s=[0, 0, 3, 1, 2]), None),
    ("negative session", _bad(unit_s=[0, -1, 0, 1, 2]), None),
    ("question out of range", _bad(unit_q=[0, 7, 12, 4, 1]), None),
    ("target out of range", _bad(targets=[1, 12, 11]), None),
    ("target below -1", _bad(targets=[[1, 2, 3], [1, -2, 3], [4, 5, 6]]), None),
    ("rows past row_cap", _bad(), 40),
    ("no room at all", _bad(), 0),
])
def test_pairs_kernel_flags_invalid_input(name, case, row_cap):
    code, err, o, cap = _pairs(case, row_cap)
    assert code == 0 and err == 7, name                                  # IGMC_ERR_CANDIDATES
    B = case["B"]
    assert (o["u"][B:] == SENT32).all() and (o["rcol"][cap:] == SENT32).all() and (o["rrat"][cap:] == SENT8).all()
    R = B // (case["A"] * len(rc._target_rows(case["targets"])[0])) * case["A"]
    assert (o["rptr"][:R + 1] <= cap).all() and (o["rptr"][R + 1:] == SENT32).all()   # rows cut short at row_cap
    assert (o["v"][:B] >= 0).all() and (o["v"][:B] < case["num_items"]).all()          # valid pairs regardless


def test_pairs_kernel_refuses_bad_layouts():
    lib = _lib.load()
    x = torch.zeros(64, dtype=torch.int64, device="cuda")
    Sd = _lib.Sessions(x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), 1, 0)
    p = x.data_ptr()
    for A, W, B in ((0, 1, 8), (257, 1, 300), (2, 0, 8), (3, 3, 8)):
        assert lib.igmc_elicit_pairs(C.byref(Sd), 12, A, p, W, 0, p, p, p, B, p, p, p, p, p, p, p, p, 8, p, p,
                                     None) == -1
        assert lib.igmc_elicit_stats(p, 1, B, A, W, p, p, None, None, None) == -1
    assert lib.igmc_elicit_stats(p, 0, 8, 2, 2, p, p, None, None, None) == -1
    assert lib.igmc_elicit_stats(p, 1, 8, 2, 2, p, None, p, None, None) == -1          # no key and no answer_mean


@pytest.mark.parametrize("case", ec.stats_cases(), ids=lambda c: c["name"])
@pytest.mark.parametrize("form", ["key", "scatter"])
def test_stats_kernel_matches_twin(case, form):
    c = case
    K, B, A, W = c["K"], c["B"], c["A"], c["W"]
    G = B // (A * W)
    preds = support.dev(np.asarray(c["preds"], np.float32).reshape(K, B), torch.float32)
    tag = support.dev(c["tag"], torch.int64)
    impact, mean, utag = rc.elicit_stats_host(np.asarray(c["preds"], np.float32), K, B, A, W, c["tag"])
    T = int(max(c["tag"])) + 1
    key = support.filled(G, SENTF, torch.float32)
    imp = support.filled(T, SENTF, torch.float32)
    am = support.filled(T * A, SENTF, torch.float32)
    args = (key.data_ptr(), None, None) if form == "key" else (None, imp.data_ptr(), am.data_ptr())
    assert _lib.load().igmc_elicit_stats(preds.data_ptr(), K, B, A, W, tag.data_ptr(), *args, None) == 0
    torch.cuda.synchronize()
    key, imp, am = key.cpu().numpy(), imp.cpu().numpy(), am.cpu().numpy()
    if form == "key":
        real = utag >= 0
        assert support.same(key[:G][real], impact[real]) and (key[:G][~real] == 0).all()
        assert (key[G:] == SENTF).all()
    else:
        want_i, want_m = np.full(T, SENTF, np.float32), np.full((T, A), SENTF, np.float32)
        for g in np.flatnonzero(utag >= 0):
            want_i[utag[g]], want_m[utag[g]] = impact[g], mean[g]
        assert support.same(imp[:T], want_i) and support.same(am[:T * A], want_m.reshape(-1))
        assert (imp[T:] == SENTF).all() and (am[T * A:] == SENTF).all()
