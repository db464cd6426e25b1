"""Rating sessions on the GPU (RatingSessions, predict_sessions, recommend_sessions, corated_items_sessions).

The oracle is the contract's equivalence: session s's subgraphs, scores, top-k lists and retrieved items are bit for
bit those of the graph functions on RatingGraph(A_s), A_s = the graph with session s's edits applied to users[s]'s
row, at the same kernel plan and batch size."""
import functools
import os
import tempfile

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import recommend as rc
from igmc_b200.data import build_adj, make_synthetic_dataset, synth_ratings
from igmc_b200.util_functions import RatingGraph, SubgraphExtractor
from oracle import extract_np

pytestmark = pytest.mark.gpu

ARRAYS = ("row_ptr", "col_idx", "rating", "col_ptr", "row_idx")


@functools.lru_cache(maxsize=None)
def _ds(name):
    return make_synthetic_dataset(name, seed=0)


@functools.lru_cache(maxsize=None)
def _r13():
    nu, ni = 400, 300
    u, v, lab = synth_ratings(nu, ni, 9000, 13, seed=4)
    return build_adj(u, v, lab, nu, ni)


def _model(R, rgcn="pyg-1.4", dgcnn=False, seed=0, h=1):
    from igmc_b200.models import DGCNN_RS, IGMC
    torch.manual_seed(seed)
    if dgcnn:
        m = DGCNN_RS(2 * h + 2, latent_dim=[32, 32, 32, 1], k=30, num_relations=R, num_bases=4, regression=True,
                     rgcn=rgcn)
    else:
        m = IGMC(2 * h + 2, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True, rgcn=rgcn)
    return m.cuda()


def _rows(A, users, session, items, values):
    """per session the dict item -> value (label + 1) of its user's row after its edits"""
    A = ssp.csr_matrix(A)
    out = []
    for s, u in enumerate(users):
        d = {}
        if u < A.shape[0]:
            d = {int(c): int(round(x)) for c, x in zip(A.indices[A.indptr[u]:A.indptr[u + 1]],
                                                      A.data[A.indptr[u]:A.indptr[u + 1]])}
        for ss, it, x in zip(session, items, values):
            if ss == s:
                if x > 0:
                    d[int(it)] = int(x)
                else:
                    d.pop(int(it), None)
        out.append(d)
    return out


def _A_s(A, u, row):
    """A with user u's row replaced by ``row`` (item -> value), grown to hold u"""
    coo = ssp.coo_matrix(A)
    keep = coo.row != u
    r = np.r_[coo.row[keep], np.full(len(row), u)]
    c = np.r_[coo.col[keep], np.array(list(row.keys()), np.int64)]
    d = np.r_[coo.data[keep], np.array(list(row.values()), np.float64)]
    return ssp.csr_matrix((d.astype(np.float32), (r, c)), shape=(max(A.shape[0], u + 1), A.shape[1]))


def _edits(rng, A, users, D, R=5):
    S, ni = len(users), A.shape[1]
    session = rng.integers(0, S, D)
    items = rng.integers(0, ni, D)
    for k in range(0, D, 3):
        u = users[session[k]]
        if u < A.shape[0] and A.indptr[u + 1] > A.indptr[u]:
            items[k] = A.indices[rng.integers(A.indptr[u], A.indptr[u + 1])]
    values = np.where(rng.random(D) < 0.3, 0, rng.integers(1, R + 1, D))
    return session, items, values


def _batch_arrays(b):
    b.check()
    adj = b.adjacency()[1]
    return [t.cpu() for t in (b.x, b.edge_index, b.edge_type, b.node_label, b.node_gid, b.y, b.batch)] + \
        [b._priv["node_ptr"].cpu(), b._priv["edge_ptr"].cpu()] + \
        [adj[k][:int(b._priv["node_ptr"][-1]) + 1 if k == "adj_in_ptr" else int(b._priv["edge_ptr"][-1])].cpu()
         for k in ("adj_in_ptr", "adj_in", "adj_eid")]


# ---- 1. the session rows --------------------------------------------------------------------------------------------
def test_session_rows_match_twin_and_invalid_input_raises():
    A = _ds("ml_100k")["adj_train"]
    g = RatingGraph(A)
    rng = np.random.default_rng(0)
    nu = A.shape[0]
    users = np.r_[rng.integers(0, nu, 20), [nu, nu + 3, 5, 5]]
    session, items, values = _edits(rng, A, users, 300)
    sess = rc.RatingSessions(g, users, session, items, values)
    got = sess.rows()
    want = rc.session_rows_host(g.host, g.shape, users, session, items, values)
    for a, b in zip(got, want):
        assert np.array_equal(a, b) and a.dtype == b.dtype
    assert sess.max_row_deg == int(np.diff(want[0]).max())
    # device inputs are checked by the kernel: RuntimeError, the graph untouched
    before = {k: g.dev[k].clone() for k in ARRAYS}
    dev = g.device
    for bad in ((0, nu, 1), (0, 0, 300), (len(users), 0, 1)):
        t = [torch.tensor([x], dtype=torch.int32, device=dev) for x in bad]
        t[1] = torch.tensor([bad[1] if bad[1] != nu else A.shape[1]], dtype=torch.int32, device=dev)
        with pytest.raises(RuntimeError, match="rating sessions"):
            rc.RatingSessions(g, users, *t)
    with pytest.raises(RuntimeError, match="rating sessions"):
        rc.RatingSessions(g, torch.tensor([-1], dtype=torch.int32, device=dev))
    for k in ARRAYS:
        assert torch.equal(before[k], g.dev[k])
    with pytest.raises(IndexError):
        rc.RatingSessions(g, users, [0], [A.shape[1]], [1])
    with pytest.raises(ValueError):
        rc.RatingSessions(g, users, [0], [0], [257])


# ---- 2. extraction ---------------------------------------------------------------------------------------------------
EXTRACT_CASES = [(1, None, 1.0, True), (1, None, 1.0, False), (1, 30, 1.0, True), (1, None, 0.6, True),
                 (1, 30, 0.7, False), (2, 30, 1.0, True), (2, None, 0.8, True), (3, 10, 1.0, True)]


@pytest.mark.parametrize("h,mnph,ratio,fast", EXTRACT_CASES)
def test_extraction_equals_graph_with_edits(h, mnph, ratio, fast):
    A = _ds("ml_100k")["adj_train"]
    nu, ni = A.shape
    g = RatingGraph(A)
    rng = np.random.default_rng(h * 10 + (mnph or 0))
    u_long = int(np.argmax(np.diff(A.indptr)))
    users = np.array([3, nu, 17, u_long])
    session, items, values = _edits(rng, A, users[:3], 60)
    # session 1 (a new user) and 2 hold the target item of their pairs; session 2 deletes ratings; session 3 grows the
    # longest row beyond the graph's longest
    r2 = A.indices[A.indptr[17]:A.indptr[17 + 1]][:5]
    unrated = np.setdiff1d(np.arange(ni), A.indices[A.indptr[u_long]:A.indptr[u_long + 1]])[:40]
    session = np.r_[session, [1, 2], np.full(len(r2), 2), np.full(len(unrated), 3)]
    items = np.r_[items, [7, 8], r2, unrated]
    values = np.r_[values, [3, 4], np.zeros(len(r2), np.int64), rng.integers(1, 6, len(unrated))]
    sess = rc.RatingSessions(g, users, session, items, values)
    if mnph is None:
        assert sess.max_row_deg > g.max_row_deg
    rows = _rows(A, users, session, items, values)
    cv = np.arange(1, 6, dtype=np.float32)
    ex = SubgraphExtractor(g, [0], [0], [0], cv, h, ratio, mnph, max_batch=16, seed=3, fast=fast)
    ex.serve_sessions(sess.max_row_deg)
    for s, u in enumerate(users):
        pv = np.r_[[7, 8], rng.integers(0, ni, 6), list(rows[s].keys())[:2]].astype(np.int64)
        pu = np.full(len(pv), u)
        pid = pu * ni + pv
        got = _batch_arrays(ex.extract(pairs=(pu, pv, np.zeros(len(pv), np.int64)), pair_ids=pid, sessions=sess,
                                       sess=np.full(len(pv), s, np.int32)))
        As = _A_s(A, u, rows[s])
        fresh = SubgraphExtractor(RatingGraph(As), [0], [0], [0], cv, h, ratio, mnph, max_batch=16, seed=3,
                                  fast=fast)
        want = _batch_arrays(fresh.extract(pairs=(pu, pv, np.zeros(len(pv), np.int64)), pair_ids=pid))
        for k, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), (s, k)
        # the oracle's canonical form of the first pair
        sub = extract_np.extract_subgraph(extract_np.RatingCSR(As), u, pv[0], h, ratio, mnph, seed=3,
                                          pair_id=int(pid[0]))
        n0 = int(got[7][1])
        assert np.array_equal(got[4][:n0].numpy(), np.r_[sub["u_nodes"], sub["v_nodes"]])
    assert int(ex.err.item()) == 0


# ---- 3. scores -------------------------------------------------------------------------------------------------------
def _session_case(A, rng, S=6, D=80):
    nu = A.shape[0]
    users = np.r_[rng.integers(0, nu, S - 2), [nu, nu + 1]]
    session, items, values = _edits(rng, A, users, D)
    return users, session, items, values


def _scores_equal(A, m, plan, mnph, B, checkpoints=None, seed=5):
    rng = np.random.default_rng(seed)
    g = RatingGraph(A)
    users, session, items, values = _session_case(A, rng)
    sess = rc.RatingSessions(g, users, session, items, values)
    rows = _rows(A, users, session, items, values)
    P = 70
    ps = rng.integers(0, len(users), P)
    pi = rng.integers(0, A.shape[1], P)
    m.kernel_plan = plan
    try:
        got = rc.predict_sessions(m, sess, ps, pi, max_nodes_per_hop=mnph, batch_size=B, checkpoints=checkpoints)
        for s in range(len(users)):
            sel = ps == s
            if not sel.any():
                continue
            want = rc.predict_pairs(m, RatingGraph(_A_s(A, users[s], rows[s])), np.full(sel.sum(), users[s]), pi[sel],
                                    max_nodes_per_hop=mnph, batch_size=B, checkpoints=checkpoints)
            assert torch.equal(got[torch.from_numpy(np.flatnonzero(sel)).cuda()], want), s
    finally:
        m.kernel_plan = "auto"
    return got


@pytest.mark.parametrize("case", ["ml_1m plan 2", "ml_100k plan 4", "r13 plan 0", "ml_100k L2", "pyg-2", "dgcnn"])
def test_scores_equal_graph_with_edits(case):
    from igmc_b200 import _lib
    if case == "ml_1m plan 2":
        A, m, plan, mnph = _ds("ml_1m")["adj_train"], _model(5), 2, 100
    elif case == "ml_100k plan 4":
        A, m, plan, mnph = _ds("ml_100k")["adj_train"], _model(5), 4, 200
    elif case == "r13 plan 0":
        A, m, plan, mnph = _r13(), _model(13), 0, 50
    elif case == "ml_100k L2":
        A, m, plan, mnph = _ds("ml_100k")["adj_train"], _model(5), _lib.plan_l2(2), 100
    elif case == "pyg-2":
        A, m, plan, mnph = _ds("ml_100k")["adj_train"], _model(5, rgcn="pyg-2"), 2, 100
    else:
        A, m, plan, mnph = _ds("ml_100k")["adj_train"], _model(5, dgcnn=True), "auto", 100
    _scores_equal(A, m, plan, mnph, 50)


def test_three_checkpoints():
    A = _ds("ml_100k")["adj_train"]
    m = _model(5)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for c in range(3):
            paths.append(os.path.join(tmp, "c%d.pth" % c))
            torch.save(_model(5, seed=c + 1).state_dict(), paths[-1])
        _scores_equal(A, m, 2, 100, 50, checkpoints=paths)


# ---- 4. ranking and retrieval ----------------------------------------------------------------------------------------
def test_recommend_and_retrieval_equal_graph_with_edits():
    A = _ds("ml_100k")["adj_train"]
    m = _model(5)
    m.kernel_plan = 2
    rng = np.random.default_rng(2)
    g = RatingGraph(A)
    users, session, items, values = _session_case(A, rng, S=5, D=60)
    sess = rc.RatingSessions(g, users, session, items, values)
    rows = _rows(A, users, session, items, values)
    ni = A.shape[1]
    lst = np.sort(rng.choice(ni, 80, replace=False))
    per = rng.integers(-1, ni, (len(users), 30))
    kw = dict(max_nodes_per_hop=100, batch_size=64)
    try:
        runs = [dict(), dict(items=lst), dict(items=lst, exclude_rated=False), dict(items=per), dict(retrieve=40)]
        got = [rc.recommend_sessions(m, sess, 10, **r, **kw) for r in runs]
        ci, cp = rc.corated_items_sessions(sess, 25)
        for s, u in enumerate(users):
            gs = RatingGraph(_A_s(A, u, rows[s]))
            for r, (ti, ts) in zip(runs, got):
                r = dict(r)
                if "items" in r and np.ndim(r["items"]) == 2:
                    r["items"] = r["items"][s:s + 1]
                wi, ws = rc.recommend(m, gs, [u], 10, **r, **kw)
                assert torch.equal(ti[s], wi[0]) and torch.equal(ts[s], ws[0]), (s, sorted(r))
            wi, wp = rc.corated_items(gs, [u], 25)
            assert torch.equal(ci[s], wi[0]) and torch.equal(cp[s], wp[0]), s
    finally:
        m.kernel_plan = "auto"


def test_empty_edits_equal_plain_functions():
    A = _ds("ml_100k")["adj_train"]
    m = _model(5)
    g = RatingGraph(A)
    users = np.array([4, 9, 4])
    sess = rc.RatingSessions(g, users)
    pi = np.arange(0, 60, 3)
    got = rc.predict_sessions(m, sess, np.full(len(pi), 1), pi, max_nodes_per_hop=100, batch_size=50)
    want = rc.predict_pairs(m, g, np.full(len(pi), 9), pi, max_nodes_per_hop=100, batch_size=50)
    assert torch.equal(got, want)
    ti, ts = rc.recommend_sessions(m, sess, 10, max_nodes_per_hop=100, batch_size=50)
    wi, ws = rc.recommend(m, g, users, 10, max_nodes_per_hop=100, batch_size=50)
    assert torch.equal(ti, wi) and torch.equal(ts, ws)


# ---- 5. independence, the graph untouched, failure and scale ---------------------------------------------------------
def test_independence_and_graph_untouched():
    from igmc_b200.models import IGMC
    from igmc_b200.train_eval import FusedAdam, TrainEngine
    from igmc_b200.util_functions import MyDynamicDataset
    ds = make_synthetic_dataset("tiny", seed=0)
    A = _ds("ml_100k")["adj_train"]
    g = RatingGraph(A)
    m = _model(5)
    m.kernel_plan = 2
    rng = np.random.default_rng(7)
    users, session, items, values = _session_case(A, rng, S=8, D=120)
    before = {k: g.dev[k].clone() for k in ARRAYS}
    state = (g.version, g.shape, g.nnz)
    sess = rc.RatingSessions(g, users, session, items, values)
    alone = rc.RatingSessions(g, users[2:3], session[session == 2] * 0, items[session == 2], values[session == 2])
    pi = rng.integers(0, A.shape[1], 90)
    try:
        outs = []
        for B, use_graph in ((50, True), (256, True), (50, False), (50, True)):
            eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=B, use_graph=use_graph)
            outs.append((eng.predict_sessions(sess, np.full(len(pi), 2), pi), eng.recommend_sessions(sess, 8)))
            eng.close()
        for o in outs[1:]:
            assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1][0], outs[0][1][0])
            assert torch.equal(o[1][1], outs[0][1][1])
        one = rc.predict_sessions(m, alone, np.zeros(len(pi), np.int64), pi, max_nodes_per_hop=100, batch_size=50)
        assert torch.equal(one, outs[0][0])
    finally:
        m.kernel_plan = "auto"
    for k in ARRAYS:
        assert torch.equal(before[k], g.dev[k]), k
    assert (g.version, g.shape, g.nnz) == state
    # a train engine on a graph that served sessions still steps
    tu, tv, tl = ds["train"]
    gt = RatingGraph(ds["adj_train"])
    rc.RatingSessions(gt, [0, gt.num_users], [0, 1], [0, 1], [2, 3])
    d = MyDynamicDataset(None, gt, (tu, tv), tl, 1, 1.0, 10, None, None, ds["class_values"])
    torch.manual_seed(0)
    mt = IGMC(d, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    te = TrainEngine(d, mt, FusedAdam(mt, lr=1e-3), 8)
    te.step(np.arange(8))
    te.step(np.arange(8, 16))
    te.close()


def test_stale_sessions_raise_and_steady_state_at_scale():
    A = _ds("ml_1m")["adj_train"]
    g = RatingGraph(A, reserve_nnz=10)
    m = _model(5)
    rng = np.random.default_rng(3)
    nu = A.shape[0]
    S = 1100
    users = np.r_[rng.integers(0, nu, S // 2), nu + np.arange(S - S // 2)]
    session = rng.integers(0, S - 50, 6000)              # the last 50 sessions have no edits
    items = rng.integers(0, A.shape[1], 6000)
    values = rng.integers(1, 6, 6000)
    session = np.r_[session, [S - 1]]                    # ... and one new user with a single delete: zero ratings
    items, values = np.r_[items, [0]], np.r_[values, [0]]
    users[S - 1] = nu + 5000
    sess = rc.RatingSessions(g, users, session, items, values)
    assert int(np.diff(sess.rows()[0])[-1]) == 0
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=256)
    try:
        outs = []
        for rep in range(2):
            P = eng.start_session_recommend(sess, 5, retrieve=20)
            assert P > 4 * 256
            for _ in range(4):
                eng.step()
            torch.cuda.set_sync_debug_mode("error")
            try:
                while eng.step():
                    pass
            finally:
                torch.cuda.set_sync_debug_mode("default")
            outs.append(eng.finish())
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
        assert (outs[0][0][S - 1] == -1).all()               # no ratings: no bridge, no candidate
        free = np.setdiff1d(np.arange(A.shape[1]), A.indices[A.indptr[1]:A.indptr[2]])[0]
        g.update([1], [free], [3])
        with pytest.raises(RuntimeError, match="updated"):
            eng.recommend_sessions(sess, 5)
        with pytest.raises(RuntimeError, match="updated"):
            rc.corated_items_sessions(sess, 5)
    finally:
        eng.close()
