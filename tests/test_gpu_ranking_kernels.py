"""The inference path's ranking and selection kernels against brute-force orders (tests/ranking_cases.py).

* igmc_topk_merge, igmc_score_scatter, igmc_influence_topk, igmc_occlusion_order, igmc_corated_items and
  igmc_corated_sessions called directly on tensors built here: ties at and across the k-th place, signed zeros,
  infinities, NaN payloads, subnormals, neighbouring floats, all-equal and all-NaN keys; shuffled ids up to 2^31 - 1;
  runs longer than a CTA's threads, batches past 48 KB and at the 227 KB shared-memory limit, streams cut in different
  places, the retriever's radix select on every byte and its ties over several chunks of its tie scan.  Scores compare
  bit for bit (NaN as NaN; its payload too where the kernel copies the value), ids exactly;
* end to end: a catalogue with never-rated items, whose identical scores fill the tail of a top-k by the tie rule, and
  an ensemble with a NaN checkpoint, through recommend and explain_pairs;
* igmc_topk_fits at its boundary, and the engine refusing a batch size the merge cannot run before any launch."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.data import make_synthetic_dataset
from igmc_b200.util_functions import RatingGraph, _stream_ptr
from tests import ranking_cases as rcs

pytestmark = pytest.mark.gpu

CASES = rcs.all_cases()


def _id(c):
    return c["name"]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _assert_claims(case, extra=None):
    got = rcs.REGIMES[case["kernel"]](case) if extra is None else extra
    assert case["claims"] <= got, ("the case no longer reaches", case["claims"] - got)


def _sync():
    torch.cuda.synchronize()


# ---- igmc_topk_merge ----------------------------------------------------------------------------------------------------
def _run_merge(lib, case, cuts):
    k, K, n_slots = case["k"], case["K"], len(case["segs"])
    ts = torch.full((n_slots, k), -np.inf, dtype=torch.float32, device="cuda")
    ti = torch.full((n_slots, k), -1, dtype=torch.int64, device="cuda")
    for pr, tag, it, (a, b) in rcs.merge_calls(case, cuts):
        B = len(tag)
        assert lib.igmc_topk_fits(k, B) == 1
        p, t, i = _dev(pr), _dev(tag), _dev(it)
        _lib.check(lib.igmc_topk_merge(p.data_ptr(), K, B, t.data_ptr(), i.data_ptr(), k, ts.data_ptr(),
                                       ti.data_ptr(), _stream_ptr()), "igmc_topk_merge")
        ws, wi = rcs.merge_reference(case, b)
        gs, gi = ts.cpu().numpy(), ti.cpu().numpy()
        assert np.array_equal(gi, wi), (cuts, b, np.argwhere(gi != wi)[:5])
        assert rcs.same_f32(gs, ws, keep_nan_bits=K == 1), (cuts, b)
    return ts, ti


@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "merge"], ids=_id)
def test_topk_merge(case):
    _assert_claims(case)
    lib = _lib.load()
    finals = [_run_merge(lib, case, cuts) for cuts in case["cuts"]]
    for ts, ti in finals[1:]:     # independent of where the batches were cut
        assert torch.equal(ti, finals[0][1])
        assert torch.equal(ts.view(torch.int32), finals[0][0].view(torch.int32))


def test_topk_merge_refuses_past_227_kb():
    """k = 256: B = 19 113 fits (the B=19113 merge case runs it), 19 114 is refused with -2 before anything is written;
    k = 1: 19 368 / 19 369.  The merge takes 16 + (k + B) * 12 bytes: a launch at k = 256, B = 19 114 failed when the
    limit was taken as (k + B) * 12"""
    lib = _lib.load()
    assert lib.igmc_topk_fits(256, 19113) == 1 and lib.igmc_topk_fits(256, 19114) == 0
    assert lib.igmc_topk_fits(1, 19368) == 1 and lib.igmc_topk_fits(1, 19369) == 0
    assert lib.igmc_topk_fits(0, 10) == 0 and lib.igmc_topk_fits(257, 10) == 0 and lib.igmc_topk_fits(1, 0) == 0
    B, k = 19114, 256
    preds = torch.zeros(B, dtype=torch.float32, device="cuda")
    tag = torch.zeros(B, dtype=torch.int64, device="cuda")
    items = torch.arange(B, dtype=torch.int32, device="cuda")
    ts = torch.full((1, k), 7.0, dtype=torch.float32, device="cuda")
    ti = torch.full((1, k), -1, dtype=torch.int64, device="cuda")
    assert lib.igmc_topk_merge(preds.data_ptr(), 1, B, tag.data_ptr(), items.data_ptr(), k, ts.data_ptr(),
                               ti.data_ptr(), _stream_ptr()) == -2
    S = torch.zeros(B, 1, dtype=torch.float32, device="cuda")
    assert lib.igmc_influence_topk(S.data_ptr(), B, 1, tag.data_ptr(), k, ts.data_ptr(), ti.data_ptr(),
                                   ts.data_ptr(), ti.data_ptr(), _stream_ptr()) == -20
    _sync()
    assert (ts == 7.0).all() and (ti == -1).all()


# ---- igmc_score_scatter -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "scatter"], ids=_id)
def test_score_scatter(case):
    _assert_claims(case)
    lib = _lib.load()
    preds, tag, n = rcs.scatter_data(case)
    sentinel = rcs.f32_bits([0x7f80dead])[0]
    out = torch.full((n,), float(sentinel), dtype=torch.float32, device="cuda")
    out.view(torch.int32).fill_(0x7f80dead)
    p, t = _dev(preds), _dev(tag)
    _lib.check(lib.igmc_score_scatter(p.data_ptr(), case["K"], len(tag), t.data_ptr(), out.data_ptr(), _stream_ptr()),
               "igmc_score_scatter")
    got = out.cpu().numpy()
    want = np.full(n, sentinel, np.float32)
    want.view(np.int32)[:] = 0x7f80dead
    want[tag[tag >= 0]] = rcs.ckpt_mean(preds)[tag >= 0]
    untouched = np.ones(n, bool)
    untouched[tag[tag >= 0]] = False
    assert (got.view(np.int32)[untouched] == 0x7f80dead).all()
    assert rcs.same_f32(got, want, keep_nan_bits=case["K"] == 1)


# ---- igmc_influence_topk ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "influence"], ids=_id)
def test_influence_topk(case):
    _assert_claims(case)
    lib = _lib.load()
    T, k = case["T"], case["k"]
    finals = []
    for cuts in case["cuts"]:
        pv = torch.full((T, k), -np.inf, dtype=torch.float32, device="cuda")
        cv = torch.full((T, k), np.inf, dtype=torch.float32, device="cuda")
        pi = torch.full((T, k), -1, dtype=torch.int64, device="cuda")
        ci = torch.full((T, k), -1, dtype=torch.int64, device="cuda")
        calls = rcs.influence_calls(case, cuts)
        for c, (S, tag, (a, b)) in enumerate(calls):
            B = len(tag)
            assert lib.igmc_topk_fits(k, B) == 1
            s, t = _dev(S), _dev(tag)
            _lib.check(lib.igmc_influence_topk(s.data_ptr(), B, T, t.data_ptr(), k, pv.data_ptr(), pi.data_ptr(),
                                               cv.data_ptr(), ci.data_ptr(), _stream_ptr()), "igmc_influence_topk")
            if c == len(calls) - 1 or T <= 3:
                want = rcs.influence_reference(case, b)
                got = [x.cpu().numpy() for x in (pv, pi, cv, ci)]
                assert np.array_equal(got[1], want[1]), (cuts, b, "pro index")
                assert np.array_equal(got[3], want[3]), (cuts, b, "con index")
                assert rcs.same_f32(got[0], want[0], True) and rcs.same_f32(got[2], want[2], True), (cuts, b)
        finals.append((pi, ci))
    for pi, ci in finals[1:]:
        assert torch.equal(pi, finals[0][0]) and torch.equal(ci, finals[0][1])


# ---- igmc_occlusion_order -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "occlusion"], ids=_id)
def test_occlusion_order(case):
    _assert_claims(case)
    lib = _lib.load()
    score, occluded, offsets, user, item, rating = rcs.occlusion_data(case)
    P, T, m = len(offsets) - 1, int(offsets[-1]), case["m"]
    nbytes = C.c_int64(0)
    _lib.check(lib.igmc_occlusion_order_ws_bytes(P, T, C.byref(nbytes)), "igmc_occlusion_order_ws_bytes")
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device="cuda")
    n = P * m if m else T
    outs = [torch.full((max(n, 1),), 12345, dtype=torch.int32, device="cuda") for _ in range(3)]
    od = torch.full((max(n, 1),), 12345.0, dtype=torch.float32, device="cuda")
    d_score = None if score is None else _dev(score)
    d_occ, d_off = _dev(occluded if T else np.zeros(1, np.float32)), _dev(offsets)
    d_u, d_i, d_r = (_dev(x if T else np.zeros(1, np.int32)) for x in (user, item, rating))
    _lib.check(lib.igmc_occlusion_order(_lib.ptr(d_score), d_occ.data_ptr(), d_off.data_ptr(), P, T, d_u.data_ptr(),
                                        d_i.data_ptr(), d_r.data_ptr(), m, ws.data_ptr(), ws.numel(),
                                        outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), od.data_ptr(),
                                        _stream_ptr()), "igmc_occlusion_order")
    order, delta = rcs.occlusion_reference(case)
    order = order.reshape(-1)
    pad = order < 0
    got = [o.cpu().numpy()[:n] for o in outs] + [od.cpu().numpy()[:n]]
    for g, src in zip(got[:3], (user, item, rating)):
        want = np.where(pad, -1, src[np.where(pad, 0, order)] if T else -1)
        assert np.array_equal(g, want)
    want_d = np.where(pad, np.float32(0), delta[np.where(pad, 0, order)] if T else np.float32(0)).astype(np.float32)
    assert rcs.same_f32(got[3], want_d, keep_nan_bits=score is None)


# ---- igmc_corated_items / igmc_corated_sessions -------------------------------------------------------------------------
_GRAPHS = {}


def _graph(name):
    if name not in _GRAPHS:
        _GRAPHS.clear()                     # one device graph at a time: the 2^24 graph holds 17 M ratings
        A = rcs.GRAPHS[name]()
        _GRAPHS[name] = (A, RatingGraph(A))
    return _GRAPHS[name]


def _corated_call(lib, g, users, m, exclude, slack=0):
    """igmc_corated_items with the workspace it asks for plus `slack` sentinel bytes; (items, paths, err, ws tail)"""
    U = len(users)
    nbytes = C.c_int64(0)
    _lib.check(lib.igmc_corated_ws_bytes(g.num_users, g.num_items, U, m, C.byref(nbytes)), "igmc_corated_ws_bytes")
    ws = torch.full((nbytes.value + slack + 1,), 0xA5, dtype=torch.uint8, device="cuda")
    items = torch.full((U, m), 777, dtype=torch.int32, device="cuda")
    paths = torch.full((U, m), 777, dtype=torch.int32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    du = _dev(np.asarray(users, np.int32))
    _lib.check(lib.igmc_corated_items(C.byref(g._c), du.data_ptr(), U, m, int(exclude), ws.data_ptr(), nbytes.value,
                                      items.data_ptr(), paths.data_ptr(), err.data_ptr(), _stream_ptr()),
               "igmc_corated_items")
    return items.cpu().numpy(), paths.cpu().numpy(), int(err.item()), nbytes.value, ws[nbytes.value:].cpu().numpy()


@pytest.mark.parametrize("case", [c for c in CASES if c["kernel"] == "corated"], ids=_id)
def test_corated_items(case):
    A, g = _graph(case["graph"])
    _assert_claims(case, rcs.corated_regimes(case, A))
    lib = _lib.load()
    nu, ni = A.shape
    items, paths, err, nbytes, tail = _corated_call(lib, g, case["users"], case["m"], case["exclude"], slack=1 << 16)
    shared = rcs.retriever_shared(nu, ni, case["m"])
    assert (nbytes == 0) == shared                       # the regime the case claims is the one the library takes
    wi, wp, _ = rcs.corated_reference(case, A)
    bad = [u for u in case["users"] if not 0 <= u < nu]
    assert err == (7 if bad else 0)                     # IGMC_ERR_CANDIDATES
    assert np.array_equal(items, wi), np.argwhere(items != wi)[:5]
    assert np.array_equal(paths, wp)
    if not shared:
        assert (tail == 0xA5).all(), "the retriever wrote past the workspace it asked for"


def test_corated_sessions():
    """sessions on the tie graph: a new user id, an unchanged user, existing users with deleted and inserted ratings
    and an empty session; both regimes of exclude_rated"""
    A, g = _graph("chunk_ties")
    lib = _lib.load()
    S = rc.RatingSessions(g, list(rcs.SESSIONS["users"]), list(rcs.SESSIONS["session"]), list(rcs.SESSIONS["items"]),
                          list(rcs.SESSIONS["values"]))
    rows = rcs.session_rows(A)
    hr = S.rows()
    for s, r in enumerate(rows):                          # the rows the kernel reads are the definition's
        assert np.array_equal(hr[1][hr[0][s]:hr[0][s + 1]], r)
    assert len(rows[4]) == 0 and rcs.SESSIONS["users"][0] >= A.shape[0]
    P = rcs.corated_paths(A, rows, rcs.SESSIONS["users"])
    for m in (1200, 7, 4000):
        for exclude in (True, False):
            wi, wp, thr = rcs.corated_select(P, rows, m, exclude)
            if m == 1200:
                assert any(t[2] and len(t[1]) > 1500 for t in thr)    # ties over several chunks
            items = torch.full((len(rows), m), 777, dtype=torch.int32, device="cuda")
            paths = torch.full((len(rows), m), 777, dtype=torch.int32, device="cuda")
            err = torch.zeros(1, dtype=torch.int32, device="cuda")
            nbytes = C.c_int64(0)
            _lib.check(lib.igmc_corated_ws_bytes(g.num_users, g.num_items, len(rows), m, C.byref(nbytes)), "ws")
            assert nbytes.value == 0
            ws = torch.empty(1, dtype=torch.uint8, device="cuda")
            _lib.check(lib.igmc_corated_sessions(C.byref(g._c), C.byref(S._c), m, int(exclude), ws.data_ptr(), 0,
                                                 items.data_ptr(), paths.data_ptr(), err.data_ptr(), _stream_ptr()),
                       "igmc_corated_sessions")
            assert int(err.item()) == 0
            assert np.array_equal(items.cpu().numpy(), wi), (m, exclude)
            assert np.array_equal(paths.cpu().numpy(), wp), (m, exclude)


def test_corated_global_regime_many_users():
    """more query users than the global-memory grid has CTAs, duplicates among them: every row its own reference"""
    A, g = _graph("bytes")
    lib = _lib.load()
    users = tuple(np.random.default_rng(5).choice(np.arange(65539), 400).tolist()) + (0, 0)
    case = dict(graph="bytes", users=users, m=10, exclude=True)
    items, paths, err, nbytes, _ = _corated_call(lib, g, users, 10, True)
    assert nbytes > 0 and err == 0
    wi, wp, _ = rcs.corated_reference(case, A)
    assert np.array_equal(items, wi) and np.array_equal(paths, wp)


# ---- end to end through InferenceEngine ---------------------------------------------------------------------------------
def _model(R, seed=0):
    from igmc_b200.models import IGMC
    torch.manual_seed(seed)
    return IGMC(4, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True).cuda()


def _cold_catalogue():
    A = make_synthetic_dataset("ml_100k", seed=0)["adj_train"]
    nu, ni = A.shape
    return ssp.csr_matrix(ssp.hstack([A, ssp.csr_matrix((nu, 320), dtype=A.dtype)])), ni


def test_cold_catalogue_ties_fill_the_tail():
    A, warm = _cold_catalogue()
    nu, ni = A.shape
    cold = np.arange(warm, ni)
    m = _model(5)
    m.kernel_plan = 1                 # the same plan at every batch size
    mnph = 100
    users = np.array([3, 400, 942])
    rng = np.random.default_rng(1)
    # the full catalogue, and a list of 100 warm and every cold item: 320 equal scores straddle the 256th place
    lists = [None, np.sort(np.concatenate([rng.choice(warm, 100, replace=False), cold]))]
    for cand in lists:
        per_user = []
        for u in users:
            rated = A.indices[A.indptr[u]:A.indptr[u + 1]]
            base = np.arange(ni) if cand is None else cand
            c = base[~np.isin(base, rated)]
            per_user.append(c)
        pu = np.concatenate([np.full(len(c), u) for u, c in zip(users, per_user)])
        pv = np.concatenate(per_user)
        flat = rc.predict_pairs(m, A, pu, pv, max_nodes_per_hop=mnph, batch_size=256).cpu().numpy()
        scores = np.split(flat, np.cumsum([len(c) for c in per_user])[:-1])
        for j, c in enumerate(per_user):       # precondition: every cold item of a user scores bit-identically
            sc = scores[j][np.isin(c, cold)]
            assert len(np.unique(sc.view(np.int32))) == 1, (users[j], "cold scores differ")
        if cand is not None:
            assert all(rcs.ties_at(s, c, 256) for s, c in zip(scores, per_user))
        for B in (50, 256):
            for use_graph in (True, False):
                eng = rc.InferenceEngine(m, A, max_nodes_per_hop=mnph, batch_size=B, use_graph=use_graph)
                ti, ts = eng.recommend(users, 256, items=cand)
                eng.close()
                ti, ts = ti.cpu().numpy(), ts.cpu().numpy()
                for j, c in enumerate(per_user):
                    ws, wi = rcs.top_list(scores[j], c, 256, rcs.order_desc, -np.inf)
                    assert np.array_equal(ti[j], wi), (B, use_graph, j)
                    assert rcs.same_f32(ts[j], ws, True), (B, use_graph, j)


def test_nan_checkpoint():
    """an ensemble with a checkpoint whose lin2.bias is NaN: every score is NaN, so each top-k is the first k
    candidates by item and each explanation is in rating order, as a model whose every delta is 0 orders it"""
    A = make_synthetic_dataset("ml_100k", seed=0)["adj_train"]
    m = _model(5)
    users = np.array([5, 6])
    with tempfile.TemporaryDirectory() as tmp:
        good, bad, flat = (os.path.join(tmp, n) for n in ("good.pth", "nan.pth", "flat.pth"))
        torch.save(m.state_dict(), good)
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        sd["lin2.bias"].fill_(float("nan"))
        torch.save(sd, bad)
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        sd["lin2.weight"].zero_()
        torch.save(sd, flat)
        ti, ts = rc.recommend(m, A, users, 20, items=np.arange(0, 300, 7), max_nodes_per_hop=200, batch_size=50,
                              checkpoints=[good, bad])
        ti, ts = ti.cpu().numpy(), ts.cpu().numpy()
        assert np.isnan(ts).all()
        for j, u in enumerate(users):
            rated = A.indices[A.indptr[u]:A.indptr[u + 1]]
            c = np.arange(0, 300, 7)
            assert np.array_equal(ti[j], c[~np.isin(c, rated)][:20])
        pu, pv = np.array([5, 6, 7]), np.array([10, 20, 30])
        ex = rc.explain_pairs(m, A, pu, pv, max_nodes_per_hop=200, batch_size=50, checkpoints=[good, bad])
        zero = rc.explain_pairs(m, A, pu, pv, max_nodes_per_hop=200, batch_size=50, checkpoints=[flat])
    assert torch.isnan(ex.score).all() and torch.isnan(ex.delta).all()
    assert (zero.delta == 0).all() and not torch.signbit(zero.delta).any()
    for f in ("offsets", "user", "item", "rating"):
        assert torch.equal(getattr(ex, f), getattr(zero, f)), f


def test_engine_refuses_unrunnable_batch_before_launch():
    """batch_size 19 114: k = 256 does not fit the merge and is refused with ValueError before any launch (recommend,
    sessions, influence, the public functions); the engine then serves k = 255 and an explicit-pair run"""
    ds = make_synthetic_dataset("tiny", seed=0)
    A = ds["adj_train"]
    m = _model(5)
    eng = rc.InferenceEngine(m, A, batch_size=19114)
    with pytest.raises(ValueError, match="top-k merge"):
        eng.recommend([0, 1], 256)
    sess = rc.RatingSessions(eng.graph, [0, 1])
    with pytest.raises(ValueError, match="top-k merge"):
        eng.recommend_sessions(sess, 256)
    tr = (np.array([0, 1]), np.array([2, 3]), np.array([1.0, 2.0]))
    with pytest.raises(ValueError, match="top-k merge"):
        eng.influence(tr, (np.array([0]), np.array([4])), 256)
    for call in (lambda: rc.recommend(m, A, [0], 256, batch_size=19114),
                 lambda: rc.recommend_sessions(m, sess, 256, batch_size=19114),
                 lambda: rc.influence(m, A, tr, (np.array([0]), np.array([4])), 256, batch_size=19114)):
        with pytest.raises(ValueError, match="top-k merge"):
            call()
    ti, ts = eng.recommend([0, 1], 255)
    nu, ni = A.shape
    for j, u in enumerate([0, 1]):
        rated = A.indices[A.indptr[u]:A.indptr[u + 1]]
        c = np.setdiff1d(np.arange(ni), rated)
        s = eng.predict_pairs(np.full(len(c), u), c).cpu().numpy()
        ws, wi = rcs.top_list(s, c, 255, rcs.order_desc, -np.inf)
        assert np.array_equal(ti[j].cpu().numpy(), wi) and rcs.same_f32(ts[j].cpu().numpy(), ws, True)
    eng.close()
