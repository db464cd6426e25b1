"""Counterfactual explanations on the GPU (counterfactual, InferenceEngine.start_counterfactual).

The oracle is the contract: every trial score is ``predict_sessions`` of a session that deletes the trial's ratings
(bit for bit, at the same kernel plan and batch size), and the whole greedy path is ``counterfactual_host`` driven by
``predict_sessions``.  The kernels are checked byte for byte against their numpy twins."""
import ctypes as C
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.util_functions import RatingGraph
from tests import support

pytestmark = pytest.mark.gpu

SENT32, SENT8, SENTF = -77, 0xAB, -7.5
GUARD = 16


def _host(cf):
    return rc.Counterfactual(*(t.cpu().numpy() for t in cf))


def _equal(a, b):
    for f in rc.Counterfactual._fields:
        x, y = getattr(a, f), getattr(b, f)
        if f in ("score", "rival_score"):
            assert support.same(x, y), f
        else:
            assert np.array_equal(np.asarray(x), np.asarray(y)), f


def _queries(m, g, n, seed, lo=8, hi=60, **kw):
    """n queries (u, X, Y): users of degree lo..hi, X and Y their first two recommended items"""
    rng = np.random.default_rng(seed)
    deg = np.diff(g.host["row_ptr"])
    users = rng.choice(np.flatnonzero((deg >= lo) & (deg <= hi)), n, replace=False)
    top, _ = rc.recommend(m, g, users, 2, **kw)
    top = top.cpu().numpy()
    return users, top[:, 0], top[:, 1]


def _session_scorer(m, g, **kw):
    """scorer(users, deleted, targets) of counterfactual_host: one RatingSessions and one predict_sessions call"""
    def score(users, deleted, targets):
        sess = np.array([s for s, d in enumerate(deleted) for _ in d], np.int64)
        items = np.array([i for d in deleted for i in d], np.int64)
        S = rc.RatingSessions(g, np.asarray(users, np.int64), sess, items, np.zeros(len(items), np.int64))
        return rc.predict_sessions(m, S, np.arange(len(users)), targets, **kw).cpu().numpy()
    return score


# ---- 1. kernels against their twins ---------------------------------------------------------------------------------
def _kernel_state(g, users, M, step, rng):
    """a mid-run state: R of step - 1 random positions per query, counts of the next pass"""
    Q = len(users)
    deg = np.diff(g.host["row_ptr"])[users]
    removed = np.zeros((Q, M), np.int32)
    size = np.zeros(Q, np.int32)
    count = np.ones(Q, np.int32)
    for q in range(Q):
        if step > 0:
            t = min(step - 1, int(deg[q]))
            size[q] = t
            removed[q, :t] = np.sort(rng.choice(int(deg[q]), t, replace=False))
            count[q] = deg[q] - t
    count[1] = 0                                                        # a query already done
    return removed, size, count


@pytest.mark.parametrize("B,step", [(1, 0), (7, 0), (1, 2), (7, 1), (64, 3), (256, 2)])
def test_kernels_match_twins(B, step):
    A = support.adj("ml_100k")
    g = RatingGraph(A)
    rng = np.random.default_rng(B + step)
    h = g.host
    rp, ci, rt = h["row_ptr"], h["col_idx"], h["rating"]
    deg = np.diff(rp)
    users = np.r_[rng.choice(np.flatnonzero((deg > 0) & (deg < 40)), 5), [int(np.argmax(deg))]]
    users[3] = users[2]                                                 # a duplicated query
    Q, M, ni = len(users), 4, A.shape[1]
    items = rng.integers(0, ni, Q)
    rivals = (items + 1) % ni
    removed, size, count = _kernel_state(g, users, M, step, rng)
    offsets = rc.explain_offsets_host(count)
    P2 = 2 * int(offsets[-1])
    L = max(g.max_row_deg, 1)
    lib = _lib.load()
    du, dx, dy = support.dev(users, torch.int32), support.dev(items, torch.int32), support.dev(rivals, torch.int32)
    dsize, drem = support.dev(size, torch.int32), support.dev(removed, torch.int32)
    Qd = _lib.Counterfactual(du.data_ptr(), dx.data_ptr(), dy.data_ptr(), dsize.data_ptr(), drem.data_ptr(), Q, M)
    doff = support.dev(offsets, torch.int64)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    cursor = torch.zeros(1, dtype=torch.int64, device="cuda")
    for pos in list(range(0, P2, B))[:6] + [P2 + 5]:                    # the last: an all-padding batch
        cursor.fill_(pos)
        lu, lv, ru, sess = (torch.full((B + GUARD,), SENT32, dtype=torch.int32, device="cuda") for _ in range(4))
        rptr = torch.full((B + 1 + GUARD,), SENT32, dtype=torch.int32, device="cuda")
        pid, tag = (torch.full((B + GUARD,), SENT32, dtype=torch.int64, device="cuda") for _ in range(2))
        rcol = torch.full((B * L + GUARD,), SENT32, dtype=torch.int32, device="cuda")
        rrat = torch.full((B * L + GUARD,), SENT8, dtype=torch.uint8, device="cuda")
        assert lib.igmc_counterfactual_pairs(C.byref(g._c), C.byref(Qd), doff.data_ptr(), step, cursor.data_ptr(), B,
                                             lu.data_ptr(), lv.data_ptr(), pid.data_ptr(), tag.data_ptr(),
                                             ru.data_ptr(), rptr.data_ptr(), rcol.data_ptr(), rrat.data_ptr(), B * L,
                                             sess.data_ptr(), err.data_ptr(), None) == 0
        out, (wu, wptr, wcol, wrat) = rc.counterfactual_pairs_host(rp, ci, rt, ni, users, items, rivals, removed, size,
                                                                   offsets, step, pos, B)
        assert int(err.item()) == 0 and int(cursor.item()) == pos + B
        assert np.array_equal(lu.cpu().numpy()[:B], out[0]) and np.array_equal(lv.cpu().numpy()[:B], out[1])
        assert np.array_equal(pid.cpu().numpy()[:B], out[2]) and np.array_equal(tag.cpu().numpy()[:B], out[3])
        assert np.array_equal(ru.cpu().numpy()[:B], wu) and np.array_equal(sess.cpu().numpy()[:B], np.arange(B))
        assert np.array_equal(rptr.cpu().numpy()[:B + 1], wptr)
        n = int(wptr[-1])
        assert np.array_equal(rcol.cpu().numpy()[:n], wcol) and np.array_equal(rrat.cpu().numpy()[:n], wrat)
        for t, k, sent in ((lu, B, SENT32), (lv, B, SENT32), (ru, B, SENT32), (sess, B, SENT32), (rptr, B + 1, SENT32),
                           (pid, B, SENT32), (tag, B, SENT32), (rcol, B * L, SENT32), (rrat, B * L, SENT8)):
            assert (t[k:] == sent).all()                               # guard entries untouched
    # the selection after a pass, scores with ties and NaN
    scores = rng.choice(np.array([0.25, 0.5, 0.5, 1.0, np.nan], np.float32), max(P2, 1))
    st = dict(removed=removed.copy(), size=size.copy(), count=count.copy(), found=np.zeros(Q, bool),
              items=np.full((Q, M), SENT32, np.int32), ratings=np.full((Q, M), SENT32, np.int32),
              score=np.full((Q, M + 1), SENTF, np.float32), rival_score=np.full((Q, M + 1), SENTF, np.float32))
    dev = {k: support.dev(v, torch.uint8 if k == "found" else torch.from_numpy(v).dtype) for k, v in st.items()}
    Qd.size, Qd.removed = dev["size"].data_ptr(), dev["removed"].data_ptr()
    dscores = support.dev(scores, torch.float32)
    assert lib.igmc_counterfactual_select(C.byref(g._c), C.byref(Qd), doff.data_ptr(), dscores.data_ptr(), step,
                                          dev["count"].data_ptr(), dev["found"].data_ptr(), dev["items"].data_ptr(),
                                          dev["ratings"].data_ptr(), dev["score"].data_ptr(),
                                          dev["rival_score"].data_ptr(), err.data_ptr(), None) == 0
    rc.counterfactual_select_host(rp, ci, rt, users, items, rivals, offsets, scores, step, st)
    assert int(err.item()) == 0
    for k, v in st.items():
        got = dev[k].cpu().numpy()
        if k in ("score", "rival_score"):
            assert support.same(got, v), k
        else:
            assert np.array_equal(got.astype(v.dtype), v), k


# ---- 2. every trial score is predict_sessions' ----------------------------------------------------------------------
def test_trial_scores_equal_predict_sessions():
    A = support.adj("ml_1m")
    g = RatingGraph(A)
    m = support.model(5)
    m.kernel_plan = 2
    B, kw = 64, dict(max_nodes_per_hop=100)
    try:
        users, items, rivals = _queries(m, g, 4, 0, hi=30, **kw)
        eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=B)
        passes = []
        select = eng._select_trials

        def snapshot():
            run = eng.run
            passes.append((run["step"], run["offsets"].cpu().numpy(), run["scores"].cpu().numpy(),
                           run["removed"].cpu().numpy(), run["out"].size.cpu().numpy()))
            return select()
        eng._select_trials = snapshot
        try:
            eng.counterfactual(users, items, rivals, 3)
        finally:
            eng.close()
        rp, ci = g.host["row_ptr"], g.host["col_idx"]
        scorer = _session_scorer(m, g, batch_size=B, **kw)
        assert len(passes) >= 2 and [p[0] for p in passes[:3]] == list(range(min(len(passes), 3)))
        for step, offsets, scores, removed, size in passes[:3]:
            tu, dl, tt = [], [], []
            for q in range(len(users)):
                u, n = int(users[q]), int(offsets[q + 1] - offsets[q])
                if n == 0:                                              # done before this pass
                    continue
                R = list(removed[q, :size[q]])
                free = [p for p in range(int(rp[u + 1] - rp[u])) if p not in R] if step else [None] * n
                assert len(free) == n
                for c in range(n):
                    d = list(ci[rp[u] + np.array(R + ([free[c]] if step else []), np.int64)])
                    tu += [u, u]
                    dl += [d, d]
                    tt += [items[q], rivals[q]]
            assert support.same(scorer(tu, dl, tt), scores)
    finally:
        m.kernel_plan = "auto"


# ---- 3. the whole path is the host loop over predict_sessions ---------------------------------------------------------
CASES = {
    # name: (dataset, h, mnph, model kwargs, forced kernel plan, checkpoints); the automatic plans are those
    # tests/test_gpu_draws.py checks for the same cases
    "plan 2 ml_1m": ("ml_1m", 1, 100, {}, "auto", 0),
    "plan 4 ml_100k": ("ml_100k", 1, 200, {}, "auto", 0),
    "plan 0 R=13": ("r13", 1, 50, {}, "auto", 0),
    "L2 plan ml_100k uncapped": ("ml_100k", 1, None, {}, "auto", 0),
    "pyg-2": ("ml_1m", 1, 100, dict(rgcn="pyg-2"), "auto", 0),
    "DGCNN_RS": ("ml_1m", 1, 100, dict(dgcnn=True), "auto", 0),
    "NB 2": ("ml_1m", 1, 100, dict(nb=2), "auto", 0),
    "NB 4 plan 4": ("ml_1m", 1, 100, dict(nb=4), 4, 0),
    "h=2 sampled": ("ml_1m", 2, 20, {}, "auto", 0),
    "K=3 checkpoints": ("ml_1m", 1, 100, {}, "auto", 3),
}


@pytest.mark.parametrize("name", list(CASES))
def test_path_equals_host_loop(name):
    dsn, h, mnph, kw, plan, K = CASES[name]
    A = support.adj(dsn)
    R = 13 if dsn == "r13" else 5
    g = RatingGraph(A)
    m = support.model(R, h=h, **kw)
    m.kernel_plan = plan
    B = 50
    try:
        with tempfile.TemporaryDirectory() as d:
            ck = support.checkpoints(m, K, d) if K else None
            opts = dict(h=h, max_nodes_per_hop=mnph, batch_size=B, checkpoints=ck, sample_seed=3)
            users, items, rivals = _queries(m, g, 3, len(name), hi=25, **opts)
            M = 4
            got = _host(rc.counterfactual(m, g, users, items, rivals, M, **opts))
            rp, ci, rt = g.host["row_ptr"], g.host["col_idx"], g.host["rating"]
            want = rc.counterfactual_host(rp, ci, rt, users, items, rivals, M, _session_scorer(m, g, **opts))
            _equal(got, want)
            # through the graph path: the removals applied to a fresh graph
            for q in range(len(users)):
                t = int(got.size[q])
                if t == 0:
                    continue
                g2 = RatingGraph(A)
                g2.update(np.full(t, users[q]), got.items[q, :t], np.zeros(t, np.int64))
                s = rc.predict_pairs(m, g2, [users[q]] * 2, [items[q], rivals[q]], **opts).cpu().numpy()
                assert support.same(s, [got.score[q, t], got.rival_score[q, t]])
                if got.found[q]:
                    assert rc._before(s[1], rivals[q], s[0], items[q])
    finally:
        m.kernel_plan = "auto"


# ---- 4. independence, determinism and no stray syncs ------------------------------------------------------------------
def _run(m, g, users, items, rivals, M, B, use_graph=True, sync_check=False):
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=B, use_graph=use_graph)
    try:
        eng.start_counterfactual(users, items, rivals, M)
        while True:
            run = eng.run
            inside = run["steps"] > 0 and 2 <= run["done"] < run["steps"] - 1   # captured, not the pass's last step
            if sync_check and inside:
                torch.cuda.set_sync_debug_mode("error")
            try:
                more = eng.step()
            finally:
                torch.cuda.set_sync_debug_mode("default")
            if not more:
                break
        out = _host(eng.finish())
        assert int(eng.extractor.err.item()) == 0
        return out
    finally:
        eng.close()


def test_independent_of_batch_replay_and_other_queries():
    A = support.adj("ml_1m")
    g = RatingGraph(A)
    m = support.model(5)
    users, items, rivals = _queries(m, g, 101, 5, hi=200, max_nodes_per_hop=100)
    M = 3
    base = _run(m, g, users[:2], items[:2], rivals[:2], M, 50)
    for B in (1, 256):
        _equal(_run(m, g, users[:2], items[:2], rivals[:2], M, B), base)
    _equal(_run(m, g, users[:2], items[:2], rivals[:2], M, 50, use_graph=False), base)
    _equal(_run(m, g, users[:2], items[:2], rivals[:2], M, 50), base)          # a second run
    among = _run(m, g, users, items, rivals, M, 256)
    alone = _run(m, g, users[50:51], items[50:51], rivals[50:51], M, 256)
    _equal(rc.Counterfactual(*(f[50:51] for f in among)), alone)
    _equal(rc.Counterfactual(*(f[:2] for f in among)), base)


def test_steps_inside_a_pass_do_not_sync():
    A = support.adj("ml_1m")
    g = RatingGraph(A)
    m = support.model(5)
    users, items, rivals = _queries(m, g, 6, 9, lo=40, hi=120, max_nodes_per_hop=100)
    a = _run(m, g, users, items, rivals, 2, 16, sync_check=True)
    _equal(a, _run(m, g, users, items, rivals, 2, 16))


# ---- 5. validation ------------------------------------------------------------------------------------------------------
def test_validation_and_updates():
    A = support.adj("ml_100k")
    g = RatingGraph(A, reserve_nnz=10)
    m = support.model(5)
    nu, ni = A.shape
    eng = rc.InferenceEngine(m, g, batch_size=32)
    try:
        with pytest.raises(IndexError):
            eng.start_counterfactual([nu], [0], [1])
        with pytest.raises(ValueError):
            eng.start_counterfactual([0], [3], [3])
        with pytest.raises(NotImplementedError):
            eng.start_counterfactual([0], [0], [1], 300)
        empty = eng.counterfactual([], [], [], 5)
        assert empty.items.shape == (0, 5) and empty.score.shape == (0, 6)
        deg = np.diff(g.host["row_ptr"])
        u = int(np.flatnonzero(deg > 20)[0])
        eng.start_counterfactual([u], [0], [1], 3)
        g.update([u], [int(g.host["col_idx"][g.host["row_ptr"][u]])], [0])     # delete one of u's ratings
        with pytest.raises(RuntimeError, match="updated during this run"):
            while eng.step():
                pass
        # after the update the engine serves the new graph
        cf = _host(eng.counterfactual([u], [0], [1], 3))
        rp, ci, rt = g.host["row_ptr"], g.host["col_idx"], g.host["rating"]
        want = rc.counterfactual_host(rp, ci, rt, [u], [0], [1], 3, _session_scorer(m, g, batch_size=32))
        _equal(cf, want)
    finally:
        eng.close()
