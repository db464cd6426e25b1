"""Group recommendation on the GPU (recommend_groups, predict_groups, InferenceEngine.start_recommend_groups /
start_group_pairs; csrc/groups.cu).

* igmc_group_rows, igmc_group_pairs and igmc_group_stats byte for byte against their host twins
  (tests/test_group_host.py), with guard entries past the outputs and the error word read, bad ids included;
* every list and every GroupScores bit for bit the host composition (recommend_groups_host / predict_groups_host) of
  ``predict_pairs`` scores from the same engine, on plans 2 / 4 / 0 (R = 13) / L2, rgcn="pyg-2", DGCNN_RS and three
  checkpoints, over the catalogue, a shared list and per-group rows, with and without exclusion;
* a group of one is ``recommend``; a group that rated every candidate gets -1 / -inf; k beyond the candidates pads;
* results do not depend on the other groups or on graph replay, two runs are bit-identical, steps make no host sync,
  and a graph.update between runs is served while one during a run raises."""
import ctypes as C
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.util_functions import RatingGraph, _stream_ptr
from tests import support

pytestmark = pytest.mark.gpu

SENT32, SENTF = -77, -7.5
GUARD = 16


def _groups(g, seed, sizes=(1, 2, 3, 5)):
    """groups of the given sizes from users with 5-60 ratings, the last one sharing a member with the second"""
    rng = np.random.default_rng(seed)
    deg = np.diff(g.host["row_ptr"])[:g.num_users]
    pool = np.flatnonzero((deg >= 5) & (deg <= 60))
    out = [list(rng.choice(pool, n, replace=False)) for n in sizes]
    if len(out) > 2 and out[1][1] not in out[-1]:
        out[-1][0] = out[1][1]
    return [[int(u) for u in grp] for grp in out]


# ---- 1. the kernels against their twins --------------------------------------------------------------------------------
def _toy_csr():
    rows = [[1, 4, 7], [], [0, 4, 9, 11], [2, 7], [4], [1, 3, 5, 7, 9, 11], list(range(0, 300, 2))]
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    ci = np.concatenate([np.asarray(r, np.int64) for r in rows]).astype(np.int32)
    keep = [support.dev(rp), support.dev(ci)]
    G = _lib.CSR(keep[0].data_ptr(), keep[1].data_ptr(), None, None, None, len(rows), 300)
    return G, keep, rp, ci


def _group_rows(G, members, cap):
    Gn, M = members.shape
    row_ptr = torch.full((Gn + 1 + GUARD,), SENT32, dtype=torch.int32, device="cuda")
    col = torch.full((max(cap, 1) + GUARD,), SENT32, dtype=torch.int32, device="cuda")
    ws = torch.empty(2 * Gn + 1 + cap, dtype=torch.int32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    dm = support.dev(members)
    code = _lib.load().igmc_group_rows(C.byref(G), dm.data_ptr(), Gn, M, row_ptr.data_ptr(), col.data_ptr(), cap,
                                       ws.data_ptr(), err.data_ptr(), _stream_ptr())
    torch.cuda.synchronize()
    return code, int(err.item()), row_ptr.cpu().numpy(), col.cpu().numpy()


@pytest.mark.parametrize("M", [1, 3, 64])
def test_group_rows_kernel_matches_twin(M):
    G, keep, rp, ci = _toy_csr()
    rng = np.random.default_rng(M)
    members = np.full((300, M), -1, np.int32)                                # > 256 groups: two scan chunks
    for j in range(300):
        n = int(rng.integers(1, M + 1))
        members[j, :n] = rng.choice(7, n, replace=True) if M > 7 else rng.choice(7, n, replace=False)
    members[0, :] = -1
    members[0, 0] = 1                                                        # only the empty row
    cap = int(sum(rp[u + 1] - rp[u] for u in members[members >= 0]))
    code, err, got_rp, got_ci = _group_rows(G, members, cap)
    assert code == 0 and err == 0
    want_rp, want_ci = rc.group_rows_host(rp, ci, members)
    assert np.array_equal(got_rp[:301], want_rp) and (got_rp[301:] == SENT32).all()
    n = int(want_rp[-1])
    assert np.array_equal(got_ci[:n], want_ci) and (got_ci[n:] == SENT32).all()


def test_group_rows_kernel_flags_bad_ids_and_capacity():
    G, keep, rp, ci = _toy_csr()
    members = np.array([[0, 2], [3, 99], [5, -3]], np.int32)                 # ids outside [-1, num_users)
    code, err, got_rp, got_ci = _group_rows(G, members, 64)
    assert code == 0 and err == 7                                            # IGMC_ERR_CANDIDATES
    want_rp, want_ci = rc.group_rows_host(rp, ci, np.where((members < -1) | (members >= 7), -1, members))
    assert np.array_equal(got_rp[:4], want_rp) and np.array_equal(got_ci[:int(want_rp[-1])], want_ci)
    code, err, got_rp, got_ci = _group_rows(G, np.array([[0, 2], [5, 3]], np.int32), 9)    # 7 + 8 entries > 9
    assert code == 0 and err == 7 and (got_ci[9:] == SENT32).all() and got_rp[2] <= 9
    lib = _lib.load()
    p = keep[0].data_ptr()
    for Gn, M in ((0, 1), (1, 0), (1, 65)):
        assert lib.igmc_group_rows(C.byref(G), p, Gn, M, p, p, 4, p, p, None) == -1


@pytest.mark.parametrize("B", [12, 13, 256])
def test_group_pairs_kernel_matches_twin(B):
    members = np.array([[5, 2, -1], [0, -1, -1], [3, 1, 4]], np.int32)
    ni, nu = 3_000_000_000 // 6, 6                                           # pair ids past 2^31
    Gu = B // 3
    rng = np.random.default_rng(B)
    ug = rng.integers(0, 3, Gu).astype(np.int32)
    ug[0] = 0
    uv = rng.integers(0, ni, Gu).astype(np.int32)
    ut = np.arange(Gu, dtype=np.int64)
    ut[-1] = -1                                                              # a tail unit
    out = {k: torch.full((B + GUARD,), SENT32, dtype=dt, device="cuda")
           for k, dt in (("u", torch.int32), ("v", torch.int32), ("pid", torch.int64), ("tag", torch.int64))}
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    lib = _lib.load()
    keep = [support.dev(members), support.dev(ug), support.dev(uv), support.dev(ut, torch.int64)]
    assert lib.igmc_group_pairs(keep[0].data_ptr(), 3, 3, nu, ni, keep[1].data_ptr(), keep[2].data_ptr(),
                                keep[3].data_ptr(), B, out["u"].data_ptr(), out["v"].data_ptr(),
                                out["pid"].data_ptr(), out["tag"].data_ptr(), err.data_ptr(), None) == 0
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    want = rc.group_pairs_host(members, ni, ug, uv, ut, B)
    for r, k in enumerate(("u", "v", "pid", "tag")):
        o = out[k].cpu().numpy()
        assert np.array_equal(o[:B], want[r]) and (o[B:] == SENT32).all(), k
    for bad in (dict(ug=np.full(Gu, 3, np.int32)), dict(uv=np.full(Gu, ni, np.int32)),
                dict(members=np.array([[5, 6, -1], [0, -1, -1], [3, 1, 4]] * 1, np.int32))):
        args = dict(members=members, ug=ug, uv=uv)
        args.update(bad)
        keep = [support.dev(args["members"]), support.dev(args["ug"]), support.dev(args["uv"]),
                support.dev(ut, torch.int64)]
        err.zero_()
        assert lib.igmc_group_pairs(keep[0].data_ptr(), 3, 3, nu, ni, keep[1].data_ptr(), keep[2].data_ptr(),
                                    keep[3].data_ptr(), B, out["u"].data_ptr(), out["v"].data_ptr(),
                                    out["pid"].data_ptr(), out["tag"].data_ptr(), err.data_ptr(), None) == 0
        torch.cuda.synchronize()
        assert int(err.item()) == 7
        u, v = out["u"][:B].cpu().numpy(), out["v"][:B].cpu().numpy()
        assert (u >= 0).all() and (u < nu).all() and (v >= 0).all() and (v < ni).all()   # valid pairs regardless
    p = keep[0].data_ptr()
    assert lib.igmc_group_pairs(p, 3, 4, nu, ni, p, p, p, 3, p, p, p, p, p, None) == -1     # width > B


@pytest.mark.parametrize("agg", ["mean", "min", "max"])
@pytest.mark.parametrize("form", ["key", "scatter"])
def test_group_stats_kernel_matches_twin(agg, form):
    rng = np.random.default_rng(7)
    K, M, B = 3, 4, 203                                                       # Gu = 50, 3 padding positions
    preds = rng.standard_normal((K, B)).astype(np.float32)
    preds[:, 5] = [0.0, -0.0, 0.0]
    preds[:, 6] = [-0.0, 0.0, -0.0]
    preds[:, 9] = [np.inf, 1.0, 1.0]
    preds[:, 13] = [np.nan, 1.0, 1.0]
    preds[:, 20:24] = 1.25                                                     # ties
    tag = np.full(B, -1, np.int64)
    sizes = rng.integers(0, M + 1, B // M)
    sizes[:6] = [4, 2, 3, 4, 4, 0]
    for u in range(B // M):
        tag[u * M:u * M + sizes[u]] = u if sizes[u] else -1
    key, xs, utag = rc.group_stats_host(preds, K, B, M, agg, tag)
    Gu, T = B // M, B // M
    dk = torch.full((Gu + GUARD,), SENTF, device="cuda")
    ds = torch.full((T + GUARD,), SENTF, device="cuda")
    dm = torch.full((T * M + GUARD,), SENTF, device="cuda")
    outs = (dk.data_ptr(), None, None) if form == "key" else (None, ds.data_ptr(), dm.data_ptr())
    assert _lib.load().igmc_group_stats(support.dev(preds, torch.float32).data_ptr(), K, B, M,
                                        _lib.GROUP_AGGREGATES.index(agg), support.dev(tag, torch.int64).data_ptr(),
                                        *outs, None) == 0
    torch.cuda.synchronize()
    if form == "key":
        got = dk.cpu().numpy()
        assert support.same(got[:Gu], key) and (got[Gu:] == SENTF).all()
    else:
        want_s, want_m = np.full(T, SENTF, np.float32), np.full((T, M), SENTF, np.float32)
        for g in np.flatnonzero(utag >= 0):
            want_s[utag[g]], want_m[utag[g]] = key[g], xs[g]
        got_s, got_m = ds.cpu().numpy(), dm.cpu().numpy()
        assert support.same(got_s[:T], want_s) and support.same(got_m[:T * M], want_m.reshape(-1))
        assert (got_s[T:] == SENTF).all() and (got_m[T * M:] == SENTF).all()
    p = dk.data_ptr()
    lib = _lib.load()
    assert lib.igmc_group_stats(p, 1, 8, 2, 3, p, p, None, None, None) == -1             # unknown aggregate
    assert lib.igmc_group_stats(p, 1, 8, 65, 0, p, p, None, None, None) == -1
    assert lib.igmc_group_stats(p, 1, 8, 2, 0, p, None, p, None, None) == -1             # no key, no member scores


def test_engine_raises_on_bad_device_ids():
    g = RatingGraph(support.adj("ml_100k"))
    m = support.model(5)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=50, batch_size=64)
    try:
        eng.start_group_pairs([[1, 2], [3]], [0, 1, 1], [4, 5, 6])
        eng.run["groups"][1, 0] = g.num_users + 5                           # corrupted on the device
        with pytest.raises(RuntimeError, match="kernel error 7"):
            eng.finish()
        got = eng.predict_groups([[1, 2], [3]], [0, 1], [4, 5])             # the engine serves on
        assert got.score.shape == (2,)
    finally:
        eng.close()


# ---- 2. the lists are the host composition of predict_pairs scores -----------------------------------------------------
CASES = {
    # name: (dataset, mnph, model kwargs, forced kernel plan, checkpoints)
    "plan 2 ml_1m": ("ml_1m", 100, {}, 2, 0),
    "plan 4 ml_100k": ("ml_100k", 200, {}, 4, 0),
    "plan 0 R=13": ("r13", 50, {}, "auto", 0),
    "L2 plan ml_100k uncapped": ("ml_100k", None, {}, "auto", 0),
    "pyg-2": ("ml_1m", 100, dict(rgcn="pyg-2"), "auto", 0),
    "DGCNN_RS": ("ml_1m", 100, dict(dgcnn=True), "auto", 0),
    "K=3 checkpoints": ("ml_1m", 100, {}, "auto", 3),
}


def _table_scorer(eng, members, ni):
    """scorer(users, items) of the host twins: every (member, item) score from one predict_pairs on ``eng``"""
    us = np.unique(members[members >= 0]).astype(np.int64)
    u = np.repeat(us, ni)
    v = np.tile(np.arange(ni, dtype=np.int64), len(us))
    table = eng.predict_pairs(u, v).cpu().numpy().reshape(len(us), ni)
    return lambda uu, vv: table[np.searchsorted(us, np.asarray(uu, np.int64)), np.asarray(vv, np.int64)]


@pytest.mark.parametrize("name", list(CASES))
def test_lists_equal_host_composition(name):
    dsn, mnph, kw, plan, K = CASES[name]
    A = support.adj(dsn)
    g = RatingGraph(A)
    m = support.model(13 if dsn == "r13" else 5, **kw)
    m.kernel_plan = plan
    try:
        with tempfile.TemporaryDirectory() as d:
            ck = support.checkpoints(m, K, d) if K else None
            eng = rc.InferenceEngine(m, g, max_nodes_per_hop=mnph, batch_size=64, checkpoints=ck, sample_seed=3)
            try:
                ni = g.num_items
                groups = _groups(g, len(name))
                members = rc._group_members(groups, g.num_users, 64)
                scorer = _table_scorer(eng, members, ni)
                hp = g.host
                rng = np.random.default_rng(1)
                shared = np.unique(np.r_[rng.choice(ni, 60, replace=False), hp["col_idx"][hp["row_ptr"][groups[1][0]]]])
                rows = np.full((len(groups), 40), -1, np.int64)
                for j in range(len(groups)):
                    rows[j, :30] = rng.choice(ni, 30)                          # duplicates and -1 slots
                runs = [(None, True, a) for a in ("mean", "min", "max")] + \
                       [(shared, True, "mean"), (shared, False, "min"), (rows, True, "max"), (rows, False, "mean")]
                for items, excl, agg in runs:
                    ti, ts = eng.recommend_groups(groups, 10, agg, items, excl)
                    wi, ws = rc.recommend_groups_host(hp["row_ptr"], hp["col_idx"], ni, members, 10, agg, scorer,
                                                      items, excl)
                    assert np.array_equal(ti.cpu().numpy(), wi), (items is None, excl, agg)
                    assert support.same(ts.cpu().numpy(), ws)
                    q = np.repeat(np.arange(len(groups)), 10)
                    top = ti.cpu().numpy().reshape(-1)
                    ok = top >= 0
                    got = eng.predict_groups(groups, q[ok], top[ok], agg)
                    want_s, want_m = rc.predict_groups_host(members, q[ok], top[ok], agg, scorer)
                    assert support.same(got.score.cpu().numpy(), want_s)
                    assert support.same(got.members.cpu().numpy(), want_m)
                    assert support.same(got.score.cpu().numpy(), ts.cpu().numpy().reshape(-1)[ok])
            finally:
                eng.close()
    finally:
        m.kernel_plan = "auto"


# ---- 3. edge cases ------------------------------------------------------------------------------------------------------
def test_group_of_one_rated_everything_and_short_lists():
    g = RatingGraph(support.adj("ml_100k"))
    m = support.model(5)
    opts = dict(max_nodes_per_hop=100, batch_size=64)
    users = [3, 17, 250]
    want_i, want_s = rc.recommend(m, g, users, 10, **opts)
    for agg in ("mean", "min", "max"):
        ti, ts = rc.recommend_groups(m, g, [[u] for u in users], 10, aggregate=agg, **opts)
        assert torch.equal(ti, want_i) and torch.equal(ts, want_s)
    hp = g.host
    a, b = 3, 17
    rated = np.union1d(hp["col_idx"][hp["row_ptr"][a]:hp["row_ptr"][a + 1]],
                       hp["col_idx"][hp["row_ptr"][b]:hp["row_ptr"][b + 1]])
    ti, ts = rc.recommend_groups(m, g, [[a, b]], 5, items=rated[:20], **opts)     # every candidate rated
    assert (ti.cpu().numpy() == -1).all() and (ts.cpu().numpy() == -np.inf).all()
    free = np.setdiff1d(np.arange(g.num_items), rated)[:3]
    ti, ts = rc.recommend_groups(m, g, [[a, b], [250]], 10, items=np.r_[free, rated[:4]], **opts)
    assert sorted(ti.cpu().numpy()[0, :3].tolist()) == free.tolist()         # k past the candidates: padded
    assert (ti.cpu().numpy()[0, 3:] == -1).all() and (ts.cpu().numpy()[0, 3:] == -np.inf).all()
    e = rc.predict_groups(m, g, [[a, b]], [], [], **opts)
    assert e.score.shape == (0,) and e.members.shape == (0, 2)
    ti, _ = rc.recommend_groups(m, g, [], 4, **opts)
    assert ti.shape == (0, 4)


# ---- 4. independence, determinism, syncs and updates ---------------------------------------------------------------------
def _run(m, g, groups, k, agg, B=64, use_graph=True, sync_check=False):
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=B, use_graph=use_graph)
    try:
        eng.start_recommend_groups(groups, k, agg)
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
        ti, ts = eng.finish()
        return ti.cpu().numpy(), ts.cpu().numpy()
    finally:
        eng.close()


def test_independent_of_other_groups_and_replay_and_sync_free():
    g = RatingGraph(support.adj("ml_1m"))
    m = support.model(5)
    groups = _groups(g, 5)
    for agg in ("mean", "min"):
        base = _run(m, g, groups, 10, agg)
        for got in (_run(m, g, groups, 10, agg), _run(m, g, groups, 10, agg, use_graph=False),
                    _run(m, g, groups, 10, agg, sync_check=True)):
            assert np.array_equal(got[0], base[0]) and support.same(got[1], base[1])
        more = _groups(g, 9, sizes=(4, 2)) + groups + [[7]]                   # other groups around them, M = 5 still
        got = _run(m, g, more, 10, agg)
        assert np.array_equal(got[0][2:-1], base[0]) and support.same(got[1][2:-1], base[1])


def test_served_across_updates():
    A = support.adj("ml_100k")
    g = RatingGraph(A, reserve_nnz=50)
    m = support.model(5)
    groups = [[1, 2, 3], [40, 41]]
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=64)
    try:
        eng.recommend_groups(groups, 5)
        free = np.setdiff1d(np.arange(20), g.host["col_idx"][g.host["row_ptr"][1]:g.host["row_ptr"][2]])
        g.update([1, 40], [int(free[0]), 3], [4, 2])
        ti, ts = eng.recommend_groups(groups, 5, "min")
        members = rc._group_members(groups, g.num_users, 64)
        scorer = _table_scorer(eng, members, g.num_items)
        hp = g.host
        wi, ws = rc.recommend_groups_host(hp["row_ptr"], hp["col_idx"], g.num_items, members, 5, "min", scorer)
        assert np.array_equal(ti.cpu().numpy(), wi) and support.same(ts.cpu().numpy(), ws)
        assert int(free[0]) not in ti.cpu().numpy()[0]                         # newly rated by a member: excluded
        eng.start_recommend_groups(groups, 5)
        g.update([2], [int(free[1])], [3])
        with pytest.raises(RuntimeError, match="updated during this run"):
            while eng.step():
                pass
        got = eng.predict_groups(groups, [0], [int(free[1])])
        want = rc.predict_groups(m, g, groups, [0], [int(free[1])], max_nodes_per_hop=100, batch_size=64)
        assert support.same(got.score.cpu().numpy(), want.score.cpu().numpy())
    finally:
        eng.close()
