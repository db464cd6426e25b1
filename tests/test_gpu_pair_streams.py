"""The inference path's pair-stream kernels against brute-force enumeration (tests/pair_stream_cases.py).

* igmc_candidate_plan, igmc_candidate_lists, igmc_candidate_pairs, igmc_session_pairs, igmc_explain_count,
  igmc_explain_offsets, igmc_occlusion_pairs, igmc_occlusion_mask and igmc_edge_grad_scatter called directly on
  buffers built here: every output array compared with the enumeration, integers exactly and floats bit for bit (NaN
  as NaN); every buffer pre-filled with a sentinel and sized past what the kernel may write, the guard checked; the
  error word read after every case.  The cursor is walked from 0 in steps of B through one batch past the end, or set
  directly to positions straddling 2^31 - 1, 2^31 and 2^32 on a catalogue of 2^22 + 3 items;
* the streams of InferenceEngine runs: after start_* and after each step() the batch slot the last candidate launch
  wrote, concatenated over the run, is the enumeration in position order with its tail, for recommend (no list, a
  shared list, per-user rows, retrieve= with the retrieved rows enumerated from the 3-path counts), explicit pairs,
  sessions and both passes of explain and attribute, with graphs on and off; each occlusion slot's edge_keep is the
  mask of that slot's own extracted edge_ptr."""
import ctypes as C

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.data import make_synthetic_dataset
from igmc_b200.util_functions import _stream_ptr
from oracle import extract_np
from tests import pair_stream_cases as ps
from tests import support
from tests.ranking_cases import same_f32

pytestmark = pytest.mark.gpu

CASES = ps.all_cases()
GUARD = 64
S32, S64 = -777, -(2 ** 40) - 7      # integer sentinels: no kernel writes either


def _of(kernel):
    return [c for c in CASES if c["kernel"] == kernel]


@pytest.fixture
def err():
    e = torch.zeros(1, dtype=torch.int32, device="cuda")
    yield e


def _take_err(e):
    """the error word, then zeroed"""
    torch.cuda.synchronize()
    v = int(e.item())
    e.zero_()
    return v


def _guard_ok(t, n, value):
    return bool((t[n:].cpu() == value).all())


# ---- igmc_candidate_plan ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", _of("plan"), ids=support.name_id)
def test_candidate_plan(case, err):
    support.assert_claims(ps.REGIMES, case)
    lib, A = _lib.load(), ps.plan_graph()
    G, keep = support.csr_struct(A.indptr, A.indices, A.data - 1, *A.shape)
    uo, ro, rp, _ = ps.plan_reference(case)
    users, U = case["users"], len(case["users"])
    du = support.dev_np(users, np.int32)
    dc = None if case["cand"] is None else support.dev_np(case["cand"], np.int32)
    nrated = int(sum(len(ps.row(A, int(u))) for u in users))
    user_off, rated_off = (support.filled(U + 1, S64, torch.int64, GUARD) for _ in range(2))
    rated_pos = support.filled(nrated, S32, torch.int32, GUARD)
    Cd = _lib.Candidates()
    Cd.users, Cd.cand, Cd.user_off = du.data_ptr(), _lib.ptr(dc), user_off.data_ptr()
    Cd.rated_off, Cd.rated_pos = rated_off.data_ptr(), rated_pos.data_ptr()
    Cd.num_query, Cd.num_cand, Cd.exclude_rated = U, 0 if dc is None else len(case["cand"]), int(case["exclude"])
    _lib.check(lib.igmc_candidate_plan(C.byref(G), C.byref(Cd), err.data_ptr(), _stream_ptr()), "igmc_candidate_plan")
    assert _take_err(err) == 0
    assert np.array_equal(user_off[:U + 1].cpu().numpy(), uo) and _guard_ok(user_off, U + 1, S64)
    if ro is None:
        assert (rated_off.cpu() == S64).all() and (rated_pos.cpu() == S32).all()    # no list: nothing written
    else:
        assert np.array_equal(rated_off[:U + 1].cpu().numpy(), ro) and _guard_ok(rated_off, U + 1, S64)
        n = len(rp)
        assert np.array_equal(rated_pos[:n].cpu().numpy(), rp) and _guard_ok(rated_pos, n, S32)


# ---- igmc_candidate_lists -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", _of("lists"), ids=support.name_id)
def test_candidate_lists(case, err):
    support.assert_claims(ps.REGIMES, case)
    lib, A = _lib.load(), ps.plan_graph()
    G, keep = support.csr_struct(A.indptr, A.indices, A.data - 1, *A.shape)
    uo, lists, want_err, _ = ps.lists_reference(case)
    rows = case["rows"]
    U, width = rows.shape
    du, dr = support.dev_np(case["users"], np.int32), support.dev_np(rows, np.int32)
    user_off, out = support.filled(U + 1, S64, torch.int64, GUARD), support.filled(U * width, S32, torch.int32, GUARD)
    nbytes = C.c_int64(0)
    _lib.check(lib.igmc_candidate_lists_ws_bytes(U, width, C.byref(nbytes)), "igmc_candidate_lists_ws_bytes")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device="cuda")
    Cd = _lib.Candidates()
    Cd.users, Cd.user_off, Cd.num_query, Cd.exclude_rated = du.data_ptr(), user_off.data_ptr(), U, int(case["exclude"])
    _lib.check(lib.igmc_candidate_lists(C.byref(G), C.byref(Cd), dr.data_ptr(), width, out.data_ptr(), ws.data_ptr(),
                                        ws.numel(), err.data_ptr(), _stream_ptr()), "igmc_candidate_lists")
    assert _take_err(err) == want_err
    assert np.array_equal(user_off[:U + 1].cpu().numpy(), uo) and _guard_ok(user_off, U + 1, S64)
    n = len(lists)
    assert np.array_equal(out[:n].cpu().numpy(), lists) and _guard_ok(out, n, S32)


# ---- igmc_candidate_pairs -----------------------------------------------------------------------------------------------
def _pairs_candidates(case, A):
    """the Candidates of a pairs case, its inputs from the enumeration (so only igmc_candidate_pairs is under test)"""
    P, stream, sets = ps.pairs_stream(case, A)
    Cd, keep = _lib.Candidates(), []

    def put(a, dtype):
        t = support.dev_np(a if len(a) else [0], dtype)
        keep.append(t)
        return t.data_ptr()
    if case["mode"] == "explicit":
        Cd.pair_u, Cd.pair_v = put(case["pair_u"], np.int32), put(case["pair_v"], np.int32)
    else:
        users = case["users"]
        Cd.users, Cd.num_query = put(users, np.int32), len(users)
        Cd.user_off = put(ps.prefix(len(s) for s in sets), np.int64)
        Cd.exclude_rated = int(case["exclude"])
        if case["mode"] == "per_user":
            Cd.cand, Cd.num_cand, Cd.per_user = put(ps.flat(sets), np.int32), P, 1
        elif case["mode"] == "shared":
            Cd.cand, Cd.num_cand = put(case["cand"], np.int32), len(case["cand"])
            if case["exclude"]:
                rp = ps.rated_positions(A, users, case["cand"])
                Cd.rated_off = put(ps.prefix(len(r) for r in rp), np.int64)
                Cd.rated_pos = put(ps.flat(rp), np.int32)
    Cd.num_pairs = P
    return Cd, keep, P, stream


def _pair_outs(n):
    return tuple(support.filled(n, s, d, GUARD) for s, d in ((S32, torch.int32), (S32, torch.int32), (S64, torch.int64),
                                                             (S64, torch.int64)))


def _launch_pairs(lib, G, Cd, cursor, B, outs, at, err):
    lu, lv, pid, tag = outs
    _lib.check(lib.igmc_candidate_pairs(C.byref(G), C.byref(Cd), cursor.data_ptr(), B, lu.data_ptr() + 4 * at,
                                        lv.data_ptr() + 4 * at, pid.data_ptr() + 8 * at, tag.data_ptr() + 8 * at,
                                        err.data_ptr(), _stream_ptr()), "igmc_candidate_pairs")


def _check_outs(outs, want, n):
    for o, w, s in zip(outs, want, (S32, S32, S64, S64)):
        got = o[:n].cpu().numpy()
        assert np.array_equal(got, w), np.argwhere(got != w)[:5].ravel()
        assert _guard_ok(o, n, s)


@pytest.mark.parametrize("case", _of("pairs"), ids=support.name_id)
def test_candidate_pairs(case, err):
    """the cursor walked from 0 in steps of B through one all-padding batch past the end"""
    support.assert_claims(ps.REGIMES, case)
    lib, A = _lib.load(), ps.plan_graph()
    G, keep_g = support.csr_struct(A.indptr, A.indices, A.data - 1, *A.shape)
    Cd, keep, P, stream = _pairs_candidates(case, A)
    B = case["B"]
    nb = (P + B - 1) // B + 1
    outs = _pair_outs(nb * B)
    cursor = torch.zeros(1, dtype=torch.int64, device="cuda")
    for i in range(nb):
        _launch_pairs(lib, G, Cd, cursor, B, outs, i * B, err)
    assert _take_err(err) == 0
    assert int(cursor.item()) == nb * B
    want = ps.batch_of(stream, 0, nb * B, P)
    assert (want[3][-B:] == -1).all()
    _check_outs(outs, want, nb * B)


# ---- the int64 regime ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", _of("int64"), ids=support.name_id)
def test_int64_positions(case, err):
    """the plan of 1 120 query slots over 2^22 + 3 items passes 2^32 (a half-catalogue list 2^31): user_off exact;
    igmc_candidate_pairs with the cursor set to positions straddling 2^31 - 1, 2^31, 2^32 and P - B"""
    support.assert_claims(ps.REGIMES, case)
    lib, A = _lib.load(), ps.big_graph()
    G, keep_g = support.csr_struct(A.indptr, A.indices, A.data - 1, *A.shape)
    users, U = case["users"], len(case["users"])
    counts, rp = ps.big_counts(case)
    uo = ps.prefix(counts)
    du = support.dev_np(users, np.int32)
    dc = None if case["cand"] is None else support.dev_np(case["cand"], np.int32)
    nrated = int(sum(len(ps.row(A, int(u))) for u in users))
    user_off, rated_off = (support.filled(U + 1, S64, torch.int64, GUARD) for _ in range(2))
    rated_pos = support.filled(nrated, S32, torch.int32, GUARD)
    Cd = _lib.Candidates()
    Cd.users, Cd.cand, Cd.user_off = du.data_ptr(), _lib.ptr(dc), user_off.data_ptr()
    Cd.rated_off, Cd.rated_pos = rated_off.data_ptr(), rated_pos.data_ptr()
    Cd.num_query, Cd.num_cand, Cd.exclude_rated = U, 0 if dc is None else len(case["cand"]), 1
    _lib.check(lib.igmc_candidate_plan(C.byref(G), C.byref(Cd), err.data_ptr(), _stream_ptr()), "igmc_candidate_plan")
    assert _take_err(err) == 0
    assert np.array_equal(user_off[:U + 1].cpu().numpy(), uo) and _guard_ok(user_off, U + 1, S64)
    if dc is not None:
        assert np.array_equal(rated_off[:U + 1].cpu().numpy(), ps.prefix(len(r) for r in rp))
        n = sum(len(r) for r in rp)
        assert np.array_equal(rated_pos[:n].cpu().numpy(), ps.flat(rp))
    Cd.num_pairs = P = int(uo[-1])
    B, curs = case["B"], case["cursors"]
    outs = _pair_outs(len(curs) * B)
    cursor = torch.zeros(1, dtype=torch.int64, device="cuda")
    for i, pos in enumerate(curs):
        cursor.fill_(pos)
        _launch_pairs(lib, G, Cd, cursor, B, outs, i * B, err)
        torch.cuda.synchronize()
        assert int(cursor.item()) == pos + B
    assert _take_err(err) == 0
    want = [np.concatenate(x) for x in zip(*(ps.big_batch(case, pos, uo) for pos in curs))]
    _check_outs(outs, want, len(curs) * B)


# ---- igmc_session_pairs -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", _of("session"), ids=support.name_id)
def test_session_pairs(case, err):
    support.assert_claims(ps.REGIMES, case)
    lib = _lib.load()
    users = support.dev_np(case["users"], np.int32)
    Sv = _lib.Sessions()
    Sv.users, Sv.num_sessions = users.data_ptr(), len(case["users"])
    B = len(case["links_u"])
    lu = support.filled(B, S32, torch.int32, GUARD)
    lu[:B] = support.dev_np(case["links_u"], np.int32)
    lv = support.dev_np(case["links_v"], np.int32)
    pid, sess = support.filled(B, S64, torch.int64, GUARD), support.filled(B, S32, torch.int32, GUARD)
    _lib.check(lib.igmc_session_pairs(C.byref(Sv), case["num_items"], B, lu.data_ptr(), lv.data_ptr(), pid.data_ptr(),
                                      sess.data_ptr(), err.data_ptr(), _stream_ptr()), "igmc_session_pairs")
    u, p, s, want_err = ps.session_reference(case)
    assert _take_err(err) == want_err
    for o, w, sn in ((lu, u, S32), (pid, p, S64), (sess, s, S32)):
        assert np.array_equal(o[:B].cpu().numpy(), w) and _guard_ok(o, B, sn)
    assert np.array_equal(lv.cpu().numpy(), case["links_v"])


# ---- igmc_explain_count / igmc_explain_offsets --------------------------------------------------------------------------
@pytest.mark.parametrize("case", _of("count"), ids=support.name_id)
def test_explain_count(case, err):
    support.assert_claims(ps.REGIMES, case)
    lib = _lib.load()
    ep, tag = support.dev_np(case["edge_ptr"], np.int32), support.dev_np(case["tag"], np.int64)
    ne = support.filled(case["P"], S32, torch.int32, GUARD)
    _lib.check(lib.igmc_explain_count(ep.data_ptr(), tag.data_ptr(), len(case["tag"]), ne.data_ptr(), _stream_ptr()),
               "igmc_explain_count")
    assert np.array_equal(ne[:case["P"]].cpu().numpy(), ps.count_reference(case, S32))
    assert _guard_ok(ne, case["P"], S32)


@pytest.mark.parametrize("case", _of("offsets"), ids=support.name_id)
def test_explain_offsets(case, err):
    support.assert_claims(ps.REGIMES, case)
    lib = _lib.load()
    P = len(case["num_edges"])
    ne = support.dev_np(case["num_edges"], np.int32)
    off = support.filled(P + 1, S64, torch.int64, GUARD)
    _lib.check(lib.igmc_explain_offsets(ne.data_ptr(), P, off.data_ptr(), _stream_ptr()), "igmc_explain_offsets")
    assert np.array_equal(off[:P + 1].cpu().numpy(), ps.offsets_reference(case)) and _guard_ok(off, P + 1, S64)


# ---- igmc_occlusion_pairs -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", _of("occl"), ids=support.name_id)
def test_occlusion_pairs(case, err):
    support.assert_claims(ps.REGIMES, case)
    lib, A = _lib.load(), ps.plan_graph()
    G, keep_g = support.csr_struct(A.indptr, A.indices, A.data - 1, *A.shape)
    off = ps.offsets_reference(case)
    P, B = len(case["num_edges"]), case["B"]
    pu, pv = support.dev_np(case["pair_u"], np.int32), support.dev_np(case["pair_v"], np.int32)
    doff = support.dev_np(off, np.int64)
    curs = ps.occl_cursors(case)
    n = len(curs) * B
    lu, lv, pid, tag = _pair_outs(n)
    j = support.filled(n, S32, torch.int32, GUARD)
    cursor = torch.zeros(1, dtype=torch.int64, device="cuda")
    walk = case["cursors"] is None
    for i, pos in enumerate(curs):
        if not walk:
            cursor.fill_(pos)
        a = i * B
        _lib.check(lib.igmc_occlusion_pairs(C.byref(G), pu.data_ptr(), pv.data_ptr(), doff.data_ptr(), P,
                                            cursor.data_ptr(), B, lu.data_ptr() + 4 * a, lv.data_ptr() + 4 * a,
                                            pid.data_ptr() + 8 * a, tag.data_ptr() + 8 * a, j.data_ptr() + 4 * a,
                                            err.data_ptr(), _stream_ptr()), "igmc_occlusion_pairs")
        if not walk:                             # each launch set directly: its own advance
            torch.cuda.synchronize()
            assert int(cursor.item()) == pos + B, (i, pos)
    torch.cuda.synchronize()
    assert int(cursor.item()) == curs[-1] + B
    want = [ps.occl_batch(case, pos) for pos in curs]
    assert _take_err(err) == (ps.ERR_CANDIDATES if any(w[5] for w in want) else 0)
    want = [np.concatenate(x) for x in list(zip(*want))[:5]]
    _check_outs((lu, lv, pid, tag), want[:4], n)
    assert np.array_equal(j[:n].cpu().numpy(), want[4]) and _guard_ok(j, n, S32)


# ---- igmc_occlusion_mask / igmc_edge_grad_scatter -----------------------------------------------------------------------
def _batch_out(bt):
    t = dict(edge_ptr=support.dev_np(bt["edge_ptr"], np.int32),
             edge_index=support.dev_np(bt["edge_index"].reshape(-1), np.int64),
             edge_type=support.dev_np(bt["edge_type"], np.int64), node_gid=support.dev_np(bt["node_gid"], np.int32))
    O = _lib.BatchOut()
    O.edge_cap = bt["edge_cap"]
    for k, v in t.items():
        setattr(O, k, v.data_ptr())
    return O, t


def _records(T):
    return [support.filled(T, S32, torch.int32, GUARD) for _ in range(3)]


@pytest.mark.parametrize("case", _of("mask"), ids=support.name_id)
def test_occlusion_mask(case, err):
    support.assert_claims(ps.REGIMES, case)
    lib = _lib.load()
    O, keep_t = _batch_out(case["batch"])
    B, T, E = len(case["ms"]), case["T"], int(case["batch"]["edge_ptr"][-1])
    tag, j = support.dev_np(case["tag"], np.int64), support.dev_np(case["j"], np.int32)
    keep = support.filled(case["batch"]["edge_cap"], 7, torch.uint8, GUARD)
    rec = _records(T)
    _lib.check(lib.igmc_occlusion_mask(C.byref(O), B, tag.data_ptr(), j.data_ptr(), keep.data_ptr(), rec[0].data_ptr(),
                                       rec[1].data_ptr(), rec[2].data_ptr(), err.data_ptr(), _stream_ptr()),
               "igmc_occlusion_mask")
    wk, wr, want_err = ps.mask_reference(case, S32)
    assert _take_err(err) == want_err
    assert np.array_equal(keep[:E].cpu().numpy(), wk) and _guard_ok(keep, E, 7)
    for r, w in zip(rec, wr):
        assert np.array_equal(r[:T].cpu().numpy(), w) and _guard_ok(r, T, S32)


@pytest.mark.parametrize("case", _of("scatter"), ids=support.name_id)
def test_edge_grad_scatter(case, err):
    """K checkpoints in order; user / item / rating written at k = 0 only (reset to the sentinel before k = 1)"""
    support.assert_claims(ps.REGIMES, case)
    lib = _lib.load()
    O, keep_t = _batch_out(case["batch"])
    B, K = len(case["ms"]), case["K"]
    T = int(case["offsets"][-1])
    tag, off = support.dev_np(case["tag"], np.int64), support.dev_np(case["offsets"], np.int64)
    grads = ps.scatter_grads(case)
    sentinel = np.asarray([0x7f80dead], np.int32).view(np.float32)[0]
    out = support.filled(T, 0.0, torch.float32, GUARD)
    out.view(torch.int32).fill_(0x7f80dead)
    rec = _records(T)
    outs, wr, want_err = ps.scatter_reference(case, grads, sentinel, S32)
    written = wr[0] != S32
    for k in range(K):
        g = support.dev_np(grads[k], np.float32)
        _lib.check(lib.igmc_edge_grad_scatter(C.byref(O), B, tag.data_ptr(), g.data_ptr(), off.data_ptr(), k, K,
                                              out.data_ptr(), rec[0].data_ptr(), rec[1].data_ptr(), rec[2].data_ptr(),
                                              err.data_ptr(), _stream_ptr()), "igmc_edge_grad_scatter")
        assert _take_err(err) == want_err, k
        got = out.cpu().numpy()
        assert same_f32(got[:T], outs[k]), (k, np.argwhere(got[:T].view(np.int32) != outs[k].view(np.int32))[:5])
        assert (got.view(np.int32)[:T][~written] == 0x7f80dead).all() and (got.view(np.int32)[T:] == 0x7f80dead).all()
        for r, w in zip(rec, wr if k == 0 else np.full_like(wr, S32)):
            assert np.array_equal(r[:T].cpu().numpy(), w) and _guard_ok(r, T, S32), k
        for r in rec:
            r.fill_(S32)


# ---- engine streams -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    from igmc_b200.models import IGMC
    A = make_synthetic_dataset("tiny", seed=0)["adj_train"]
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    return A, m


def _record(eng, start):
    """start the run, then step it; after each call the slot run["done"] & 1 as (phase, done, steps, arrays)"""
    recs = []

    def read():
        torch.cuda.synchronize()
        run = eng.run
        slot = run["done"] & 1
        s = eng.slots[slot]
        d = {k: s[k].cpu().numpy().copy() for k in ("u", "v", "pid", "tag", "sess") if k in s}
        if run.get("phase") == "occlude":
            ep = eng.batches[slot]._priv["edge_ptr"].cpu().numpy().astype(np.int64)
            d["j"], d["edge_ptr"] = s["j"].cpu().numpy().copy(), ep
            d["keep"] = s["keep"][:int(ep[-1])].cpu().numpy().copy()
        recs.append((run.get("phase"), run["done"], run["steps"], d))
    start()
    read()
    while eng.step():
        read()
    read()
    return recs


def _passes(recs):
    """records split into passes: [(phase, steps, [batch 0 .. steps-1 arrays], the batch past the end or None)]"""
    out = []
    for phase, done, steps, d in recs:
        if done == 0:
            out.append([phase, steps, [], None])
        assert out[-1][0] == phase and out[-1][1] == steps
        if done < steps:
            assert done == len(out[-1][2])
            out[-1][2].append(d)
        else:
            out[-1][3] = d
    return out


def _check_pass(ps_, B, want, P, extra=()):
    """the batches of a pass are the enumeration ``want`` (u, v, pid, tag[, extra...]) in position order, each real
    position once, and the tail duplicates of the last position with tag -1"""
    phase, steps, batches, past = ps_
    assert steps == (P + B - 1) // B
    keys = ("u", "v", "pid", "tag") + tuple(extra)
    got = {k: np.concatenate([b[k] for b in batches]).astype(np.int64) for k in keys}
    c = np.arange(steps * B)
    real = c < P
    c = np.minimum(c, P - 1)
    for i, k in enumerate(keys):
        w = want[i][c]
        if k == "tag":
            w = np.where(real, w, -1)
        assert np.array_equal(got[k], w), (phase, k, np.argwhere(got[k] != w)[:5].ravel())
    if past is not None:                         # the batch past the end: all padding, every key the last position's
        for i, k in enumerate(keys):
            w = -1 if k == "tag" else want[i][P - 1]
            assert (past[k] == w).all(), (phase, "past the end", k)


def _engine(m, A, B, use_graph):
    return rc.InferenceEngine(m, A, batch_size=B, use_graph=use_graph)


def _finish_clean(eng):
    eng.finish()
    assert int(eng.extractor.err.item()) == 0


RUNS = ("recommend", "shared", "rows", "retrieve", "pairs", "session_pairs", "session_recommend")


@pytest.mark.parametrize("use_graph", (True, False), ids=("graph", "eager"))
@pytest.mark.parametrize("kind", RUNS)
def test_engine_candidate_stream(tiny, kind, use_graph):
    A, m = tiny
    nu, ni = A.shape
    rng = np.random.default_rng(len(kind))
    users = np.concatenate([np.arange(nu), [3, 3, 17]])
    B = {"recommend": 700, "session_recommend": 513}.get(kind, 64)
    eng = _engine(m, A, B, use_graph)
    extra = ()
    if kind in ("recommend", "shared", "rows", "retrieve"):
        items, cand = None, None
        if kind == "shared":
            cand = items = np.sort(rng.choice(ni, 25, replace=False))
            sets = ps.candidate_sets(A, users, cand, True)
        elif kind == "recommend":
            sets = ps.candidate_sets(A, users, None, True)
        else:
            if kind == "rows":
                items = rng.integers(-1, ni, (len(users), 30))
                items[0] = -1
                rows = items
            else:
                items = None
                rows = ps.corated_rows(A, users, 10)
            sets = ps.list_sets(A, users, rows, True)
        want = ps.enumerate_positions(sets, users, ni)
        recs = _record(eng, lambda: eng.start_recommend(users, 5, items=items,
                                                        retrieve=10 if kind == "retrieve" else None))
    elif kind == "pairs":
        pu, pv = rng.integers(0, nu, 150), rng.integers(0, ni, 150)
        want = (pu, pv, pu * ni + pv, np.arange(150))
        recs = _record(eng, lambda: eng.start_pairs(pu, pv))
    else:
        s_users = np.asarray([3, nu, 3, 7, nu + 40], np.int64)       # a new id, a shared id
        session, it = rng.integers(0, 5, 40), rng.integers(0, ni, 40)
        val = rng.integers(0, 6, 40)
        S = rc.RatingSessions(eng.graph, s_users, session, it, val)
        if kind == "session_pairs":
            sp, iv = rng.integers(0, 5, 200), rng.integers(0, ni, 200)
            u = s_users[sp]
            want = (u, iv, u * ni + iv, np.arange(200), sp)
            recs = _record(eng, lambda: eng.start_session_pairs(S, sp, iv))
        else:
            rows = []
            for s, u in enumerate(s_users):
                r = set(ps.row(A, int(u)).tolist()) if u < nu else set()      # the base row, then the edits
                for a, b, x in zip(session, it, val):
                    if a == s:
                        if x == 0:
                            r.discard(int(b))
                        else:
                            r.add(int(b))
                rows.append(sorted(set(range(ni)) - set(r)))
            st = ps.enumerate_positions(rows, s_users, ni)
            want = st + (st[3],)
            recs = _record(eng, lambda: eng.start_session_recommend(S, 5))
        extra = ("sess",)
    P = len(want[0])
    (ps_,) = _passes(recs)
    assert P % B or kind != "recommend"
    _check_pass(ps_, B, want, P, extra)
    _finish_clean(eng)
    eng.close()


@pytest.mark.parametrize("use_graph", (True, False), ids=("graph", "eager"))
@pytest.mark.parametrize("kind", ("explain", "attribute"))
def test_engine_rating_stream(tiny, kind, use_graph):
    """both passes: the base pass over the pairs, then the occlusion positions (q, j) or the pairs again; the rating
    counts from the numpy oracle's subgraphs; every occlusion slot's keep is the mask of its own edge_ptr"""
    A, m = tiny
    nu, ni = A.shape
    pu, pv = np.asarray([0, 5, 5, 33, 59]), np.asarray([1, 39, 2, 20, 0])
    B = 600 if kind == "explain" else 64
    eng = _engine(m, A, B, use_graph)
    g = extract_np.RatingCSR(A)
    ne = np.asarray([len(extract_np.extract_subgraph(g, u, v)["r"]) for u, v in zip(pu, pv)], np.int64)
    off = ps.prefix(ne)
    T = int(off[-1])
    start = eng.start_explain if kind == "explain" else eng.start_attribute
    recs = _record(eng, lambda: start(pu, pv))
    base, second = _passes(recs)
    pairs = (pu, pv, pu * ni + pv, np.arange(5))
    _check_pass(base, B, pairs, 5)
    if kind == "attribute":
        assert second[0] == "grad"
        _check_pass(second, B, pairs, 5)
    else:
        assert second[0] == "occlude" and T % B
        c = np.arange(T)
        q = ps.owner_linear(off, c)
        _check_pass(second, B, (pu[q], pv[q], pu[q] * ni + pv[q], c, c - off[q]), T, ("j",))
        for d in second[2] + ([second[3]] if second[3] is not None else []):
            ep = d["edge_ptr"]
            want = np.ones(int(ep[-1]), np.uint8)
            for i in range(B):
                mm = int(ep[i + 1] - ep[i]) // 2
                if d["tag"][i] >= 0:
                    jj = int(d["j"][i])
                    assert 0 <= jj < mm and mm == ne[q[d["tag"][i]]]
                    want[ep[i] + jj] = want[ep[i] + mm + jj] = 0
            assert np.array_equal(d["keep"], want)
    _finish_clean(eng)
    eng.close()
