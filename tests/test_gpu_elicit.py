"""Question impact on the GPU (elicit, question_impact, InferenceEngine.start_elicit / start_question_impact).

The oracle is the contract: every score x_a(t) is ``predict_sessions`` of a session with the session's edits plus the
edit (q, a + 1) (bit for bit, at the same kernel plan and batch size), aggregated by ``question_impact_host``; the
ranking is a stable sort of ``question_impact``'s keys in ``recommend``'s order."""
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import recommend as rc
from igmc_b200.util_functions import RatingGraph
from tests import support

pytestmark = pytest.mark.gpu


def _specs(g, R, seed):
    """session specs (user, [(item, value)]): two new users (5 ratings, and none), a graph user with an insert, a
    change and a delete, and the user with the graph's longest row (its row + 1 is longer than any graph row)"""
    rng = np.random.default_rng(seed)
    rp, ci, rt = g.host["row_ptr"], g.host["col_idx"], g.host["rating"]
    nu, ni = g.shape
    deg = np.diff(rp)[:nu]
    u = int(rng.choice(np.flatnonzero((deg >= 5) & (deg <= 30))))
    row = ci[rp[u]:rp[u + 1]]
    free = np.setdiff1d(np.arange(ni), row)
    edits = [(int(rng.choice(free)), 1), (int(row[0]), int((rt[rp[u]] + 1) % R) + 1), (int(row[1]), 0)]
    new = [(int(i), int(rng.integers(1, R + 1))) for i in rng.choice(ni, 5, replace=False)]
    return [(nu + 3, new), (nu + 7, []), (u, edits), (int(np.argmax(deg)), [])]


def _sessions(g, specs):
    sess = [s for s, (_, e) in enumerate(specs) for _ in e]
    items = [i for _, e in specs for i, _ in e]
    values = [v for _, e in specs for _, v in e]
    return rc.RatingSessions(g, [u for u, _ in specs], sess, items, values)


def _scorer(m, g, specs, **kw):
    """scorer(session, question, answer, target) of question_impact_host: one RatingSessions of a session per (s, q,
    a) with s's edits plus (q, a + 1), one predict_sessions call"""
    def score(session, question, answer, target):
        keys = sorted(set(zip(session.tolist(), question.tolist(), answer.tolist())))
        idx = {k: j for j, k in enumerate(keys)}
        S2 = _sessions(g, [(specs[s][0], specs[s][1] + [(q, a + 1)]) for s, q, a in keys])
        j = [idx[k] for k in zip(session.tolist(), question.tolist(), answer.tolist())]
        return rc.predict_sessions(m, S2, j, target, **kw).cpu().numpy()
    return score


def _units(S, rows, ni, per, seed):
    """per session `per` questions not in its row (one at the row's ends where possible)"""
    rng = np.random.default_rng(seed)
    us, uq = [], []
    for s in range(S):
        free = np.setdiff1d(np.arange(ni), rows[s])
        pick = list(rng.choice(free, per, replace=False))
        pick[0] = int(free[0])
        us += [s] * per
        uq += [int(q) for q in pick]
    return np.array(us), np.array(uq)


def _rows(S):
    rp, ci, _ = S.rows()
    return [ci[rp[s]:rp[s + 1]] for s in range(S.num_sessions)]


CASES = {
    # name: (dataset, h, mnph, sample_ratio, model kwargs, forced kernel plan, checkpoints)
    "plan 2 ml_1m": ("ml_1m", 1, 100, 1.0, {}, 2, 0),
    "plan 4 ml_100k": ("ml_100k", 1, 200, 1.0, {}, 4, 0),
    "plan 0 R=13": ("r13", 1, 50, 1.0, {}, "auto", 0),
    "L2 plan ml_100k uncapped": ("ml_100k", 1, None, 1.0, {}, "auto", 0),
    "pyg-2": ("ml_1m", 1, 100, 1.0, dict(rgcn="pyg-2"), "auto", 0),
    "DGCNN_RS": ("ml_1m", 1, 100, 1.0, dict(dgcnn=True), "auto", 0),
    "NB 2": ("ml_1m", 1, 100, 1.0, dict(nb=2), "auto", 0),
    "NB 4 plan 4": ("ml_1m", 1, 100, 1.0, dict(nb=4), 4, 0),
    "h=2 sampled": ("ml_1m", 2, 20, 0.7, {}, "auto", 0),
    "K=3 checkpoints": ("ml_1m", 1, 100, 1.0, {}, "auto", 3),
}


# ---- 1. every impact and answer mean is the host aggregation over predict_sessions ----------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_impacts_equal_host_aggregation(name):
    dsn, h, mnph, ratio, kw, plan, K = CASES[name]
    A = support.adj(dsn)
    R = 13 if dsn == "r13" else 5
    g = RatingGraph(A)
    m = support.model(R, h=h, **kw)
    m.kernel_plan = plan
    try:
        with tempfile.TemporaryDirectory() as d:
            ck = support.checkpoints(m, K, d) if K else None
            B = max(64, 4 * R)
            opts = dict(h=h, max_nodes_per_hop=mnph, sample_ratio=ratio, batch_size=B, checkpoints=ck, sample_seed=3)
            specs = _specs(g, R, len(name))
            S = _sessions(g, specs)
            rows = _rows(S)
            assert max(len(r) for r in rows) + 1 > g.max_row_deg
            us, uq = _units(len(specs), rows, g.shape[1], 2, len(name))
            scorer = _scorer(m, g, specs, **opts)
            ni = g.shape[1]
            shared = np.array([int(rows[2][0]), 5, 5, ni - 1])               # a rated target and a duplicate
            per = np.array([[1, -1, 2, 3], [-1, -1, -1, 4], [int(rows[2][1]), 0, -1, -1], [7, 8, 9, -1]])
            for targets in (shared, per):
                got = rc.question_impact(m, S, us, uq, targets, **opts)
                imp, mean = rc.question_impact_host(R, targets, us, uq, scorer)
                assert support.same(got.impact.cpu().numpy(), imp) and support.same(got.answer_mean.cpu().numpy(), mean)
                assert np.isfinite(imp).all()
    finally:
        m.kernel_plan = "auto"


# ---- 2. the ranking is a stable sort of question_impact's keys --------------------------------------------------------
def _ranked(impact, us, uq, S, n):
    items, top = np.full((S, n), -1, np.int64), np.full((S, n), -np.inf, np.float32)
    for s in range(S):
        top[s], items[s] = rc.rank_host(impact[us == s], uq[us == s], n)
    return items, top


def test_ranking_equals_stable_sort_of_impacts():
    A = support.adj("ml_100k")
    g = RatingGraph(A)
    m = support.model(5)
    ni = g.shape[1]
    specs = _specs(g, 5, 1)
    S = _sessions(g, specs)
    rows = _rows(S)
    opts = dict(max_nodes_per_hop=100, batch_size=64)
    targets = [3, 50, 400]
    rng = np.random.default_rng(2)
    shared = rng.choice(ni, 40, replace=False)
    per_rows = np.full((4, 30), -1, np.int64)
    for s in range(4):
        k = 3 if s == 1 else 30                                           # session 1: fewer questions than n
        per_rows[s, :k] = rng.choice(ni, k, replace=False)
        if len(rows[s]):
            per_rows[s, 0] = rows[s][0]                                   # a rated item in the row
    for questions, n in ((None, 1), (None, 10), (shared, 256), (per_rows, 10)):
        items, top = rc.elicit(m, S, n, targets, questions=questions, **opts)
        cand = []
        for s in range(4):
            q = np.arange(ni) if questions is None else np.unique(questions if questions.ndim == 1 else questions[s])
            q = q[(q >= 0) & ~np.isin(q, rows[s])]
            cand.append(q)
        us = np.concatenate([[s] * len(c) for s, c in enumerate(cand)]).astype(np.int64)
        uq = np.concatenate(cand).astype(np.int64)
        imp = rc.question_impact(m, S, us, uq, targets, **opts).impact.cpu().numpy()
        want_i, want_s = _ranked(imp, us, uq, 4, n)
        assert np.array_equal(items.cpu().numpy(), want_i) and support.same(top.cpu().numpy(), want_s)
    assert (items.cpu().numpy()[1, 3:] == -1).all()


# ---- 3. independence, determinism and no stray syncs ------------------------------------------------------------------
def _run(m, g, S, n, targets, questions, B, use_graph=True, sync_check=False):
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=B, use_graph=use_graph)
    try:
        eng.start_elicit(S, n, targets, questions)
        while True:
            run = eng.run
            inside = run["steps"] > 0 and 2 <= run["done"] < run["steps"] - 1
            if sync_check and inside:
                torch.cuda.set_sync_debug_mode("error")
            try:
                more = eng.step()
            finally:
                torch.cuda.set_sync_debug_mode("default")
            if not more:
                break
        items, top = eng.finish()
        return items.cpu().numpy(), top.cpu().numpy()
    finally:
        eng.close()


def test_independent_of_batch_replay_and_other_sessions():
    A = support.adj("ml_1m")
    g = RatingGraph(A)
    m = support.model(5)
    specs = _specs(g, 5, 4)
    S = _sessions(g, specs)
    targets = [11, 12, 13]                                                 # W = 3, U = 15
    questions = np.arange(0, 400, 3)
    base = _run(m, g, S, 10, targets, questions, 64)
    for B in (15, 16, 256):                                                # B = U exactly, and padded tails
        got = _run(m, g, S, 10, targets, questions, B)
        assert np.array_equal(got[0], base[0]) and support.same(got[1], base[1])
    for got in (_run(m, g, S, 10, targets, questions, 64, use_graph=False), _run(m, g, S, 10, targets, questions, 64)):
        assert np.array_equal(got[0], base[0]) and support.same(got[1], base[1])
    more = _sessions(g, specs + [(5, []), (g.shape[0] + 1, [(3, 2)])])    # added sessions
    got = _run(m, g, more, 10, targets, questions, 64)
    assert np.array_equal(got[0][:4], base[0]) and support.same(got[1][:4], base[1])
    sync = _run(m, g, S, 10, targets, questions, 32, sync_check=True)
    assert np.array_equal(sync[0], base[0]) and support.same(sync[1], base[1])


# ---- 4. validation ------------------------------------------------------------------------------------------------------
def test_validation_and_updates():
    A = support.adj("ml_100k")
    g = RatingGraph(A, reserve_nnz=10)
    m = support.model(5)
    nu, ni = A.shape
    S = _sessions(g, [(0, []), (nu + 1, [(4, 2)])])
    rated = int(g.host["col_idx"][g.host["row_ptr"][0]])
    with pytest.raises(ValueError):
        rc.elicit(m, S, 0, [1])
    with pytest.raises(NotImplementedError):
        rc.elicit(m, S, 257, [1])
    with pytest.raises(ValueError, match="raise batch_size"):
        rc.elicit(m, S, 3, list(range(20)), batch_size=64)
    with pytest.raises(ValueError):
        rc.elicit(m, S, 3, [])
    with pytest.raises(ValueError, match="no target"):
        rc.elicit(m, S, 3, [[1, 2], [-1, -1]])
    with pytest.raises(IndexError):
        rc.elicit(m, S, 3, [ni])
    with pytest.raises(IndexError):
        rc.elicit(m, S, 3, [1], questions=[ni])
    with pytest.raises(TypeError):
        rc.elicit(m, [0], 3, [1])
    with pytest.raises(ValueError, match="already rated"):
        rc.question_impact(m, S, [0], [rated], [1])
    with pytest.raises(ValueError, match="already rated"):
        rc.question_impact(m, S, [1], [4], [1])
    with pytest.raises(IndexError):
        rc.question_impact(m, S, [2], [1], [1])
    with pytest.raises(ValueError, match="same length"):
        rc.question_impact(m, S, [0, 1], [1], [1])
    e = rc.question_impact(m, S, [], [], [1])
    assert e.impact.shape == (0,) and e.answer_mean.shape == (0, 5)
    items, _ = rc.elicit(m, S, 4, [1], questions=[rated, 4])              # session 1 rated 4, session 0 rated
    row0 = g.host["col_idx"][g.host["row_ptr"][0]:g.host["row_ptr"][1]]
    assert items.cpu().numpy()[0].tolist() == ([-1] if 4 in row0 else [4]) + [-1] * 3
    assert items.cpu().numpy()[1].tolist() == [rated, -1, -1, -1]
    eng = rc.InferenceEngine(m, g, batch_size=32)
    try:
        eng.start_elicit(S, 3, [1, 2])
        g.update([0], [rated], [0])
        with pytest.raises(RuntimeError, match="updated during this run"):
            while eng.step():
                pass
        with pytest.raises(RuntimeError):                                  # the sessions belong to the old graph
            eng.start_elicit(S, 3, [1, 2])
        S2 = _sessions(g, [(0, []), (nu + 1, [(4, 2)])])
        got = eng.question_impact(S2, [0], [rated], [1, 2])                # now a question
        want = rc.question_impact(m, S2, [0], [rated], [1, 2], batch_size=32)
        assert support.same(got.impact.cpu().numpy(), want.impact.cpu().numpy())
    finally:
        eng.close()
