"""Ranking users for items on the GPU (igmc_b200/recommend.py: recommend_users, corated_users; csrc/retrieve.cu,
csrc/recommend.cu).

* corated_users against its host twin (tests/test_recommend_users_host.py) byte for byte on tiny, ml_100k*, ml_1m*, the
  real flixster split, a 60 000 x 2 000 graph and its transpose (global-memory histograms either way), after a chain of
  graph updates; invalid item ids; the dense counts of corated_users and corated_items agree entry for entry;
* igmc_item_query_pairs called directly: batch sizes 1 / 512 / 513 / 5 000, a tag -1 tail, pair ids past 2^31, guard
  entries, the error word after each case;
* recommend_users scores bit for bit predict_pairs of the same (user, item) on plans 2, 4, 0 (R = 13) and L2, h = 2,
  rgcn="pyg-2", DGCNN_RS and a three-checkpoint ensemble; lists against a stable sort of those scores for every user,
  a shared list, per-item rows and retrieve=M; bit-identical across batch sizes and CUDA graphs on / off;
* an item nobody rated, a new item added by graph.update, recommend and recommend_users interleaved on one engine;
  steady-state steps without a host synchronisation."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.data import build_adj, synth_ratings
from igmc_b200.util_functions import RatingGraph, _stream_ptr
from tests import support

pytestmark = pytest.mark.gpu


def _twin(g, items, m, exclude):
    h = g.host
    return rc.corated_users_host(h["row_ptr"], h["col_idx"], g.num_users, g.num_items, items, m, exclude)


def _query_items(A, n, seed):
    """the most and least rated items, the first and last, and n random ones"""
    rng = np.random.default_rng(seed)
    ni = A.shape[1]
    deg = np.diff(ssp.csc_matrix(A).indptr)
    items = [int(np.argmax(deg)), int(np.argmin(deg)), 0, ni - 1]
    return np.array(items + rng.choice(ni, min(n, ni), replace=False).tolist(), np.int64)


def _tie_m(paths):
    """an m whose m-th and (m+1)-th counts tie in some row of a full (m = num_users) result, or None"""
    for row in paths:
        for p in range(1, len(row) - 1):
            if row[p] > 0 and row[p] == row[p - 1] and row[p + 1] == row[p]:
                return p
    return None


def _raters(A, v):
    return ssp.csc_matrix(A)[:, int(v)].nonzero()[0]


# ---- 1. the item-side retriever against its twin ----------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny", "ml_100k", "ml_1m", "flixster"])
def test_corated_users_match_twin(name):
    A = support.adj(name)
    g = RatingGraph(A)
    nu, ni = g.shape
    items = _query_items(A, 60, seed=1)
    full = _twin(g, items, nu, False)
    tie = _tie_m(full[1])
    ms = sorted(({1, 50, 500, nu} | ({tie} if tie else set())) & set(range(1, nu + 1)))
    for m in ms:
        for exclude in (True, False):
            users, paths = rc.corated_users(g, items, m, exclude_rated=exclude)
            assert users.shape == (len(items), m) and users.dtype == torch.int32 and paths.dtype == torch.int32
            wu, wp = _twin(g, items, m, exclude)
            assert np.array_equal(users.cpu().numpy(), wu), (name, m, exclude)
            assert np.array_equal(paths.cpu().numpy(), wp), (name, m, exclude)
            again = rc.corated_users(g, items, m, exclude_rated=exclude)
            assert torch.equal(users, again[0]) and torch.equal(paths, again[1])
            if exclude:
                for j, v in enumerate(items[:6]):
                    assert not np.isin(wu[j], _raters(A, v)).any()


@pytest.mark.parametrize("transpose", [False, True])
def test_corated_users_global_memory_regime(transpose):
    """60 000 users x 2 000 items and its transpose: the item-side histograms (the transposed shape's) do not fit in
    shared memory with either axis large"""
    u, v, lab = synth_ratings(60000, 2000, 150000, 5, seed=9)
    A = build_adj(u, v, lab, 60000, 2000)
    if transpose:
        A = ssp.csr_matrix(A.T)
        A.sort_indices()
    g = RatingGraph(A)
    nu, ni = g.shape
    items = _query_items(A, 300, seed=2)          # more items than the global-memory grid has CTAs
    lib = _lib.load()
    for m, n in ((1, len(items)), (100, len(items)), (nu, 40)):
        nbytes = C.c_int64(0)
        assert lib.igmc_corated_ws_bytes(ni, nu, n, m, C.byref(nbytes)) == 0
        assert nbytes.value > 0, (transpose, m)
        for exclude in (True, False):
            users, paths = rc.corated_users(g, items[:n], m, exclude_rated=exclude)
            wu, wp = _twin(g, items[:n], m, exclude)
            assert np.array_equal(users.cpu().numpy(), wu), (transpose, m, exclude)
            assert np.array_equal(paths.cpu().numpy(), wp), (transpose, m, exclude)
        assert torch.equal(users, rc.corated_users(g, items[:n], m, exclude_rated=False)[0])


def test_corated_users_invalid_ids_set_the_error_word():
    """an item id outside G: IGMC_ERR_CANDIDATES and a padding row; the other rows are the twin's"""
    A = support.adj("ml_100k")
    g = RatingGraph(A)
    nu, ni = g.shape
    lib = _lib.load()
    items = torch.tensor([3, -1, ni, 7], dtype=torch.int32, device="cuda")
    m = 20
    users = torch.full((4, m), 99, dtype=torch.int32, device="cuda")
    paths = torch.full((4, m), 99, dtype=torch.int32, device="cuda")
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    _lib.check(lib.igmc_corated_users(C.byref(g._ct), items.data_ptr(), 4, m, 1, None, 0, users.data_ptr(),
                                      paths.data_ptr(), err.data_ptr(), _stream_ptr()), "igmc_corated_users")
    assert int(err.item()) == 7
    got_u, got_p = users.cpu().numpy(), paths.cpu().numpy()
    assert (got_u[1:3] == -1).all() and (got_p[1:3] == 0).all()
    wu, wp = _twin(g, [3, 7], m, True)
    assert np.array_equal(got_u[[0, 3]], wu) and np.array_equal(got_p[[0, 3]], wp)
    with pytest.raises(IndexError):
        rc.corated_users(g, [ni], 3)
    assert lib.igmc_corated_users(C.byref(g._ct), items.data_ptr(), 4, nu + 1, 1, None, 0, users.data_ptr(),
                                  paths.data_ptr(), err.data_ptr(), _stream_ptr()) == -1


def _apply_chain(g, cur, rng, steps, n):
    """``steps`` random deltas of inserts, relabels and deletes with ids up to the capacity (new users and items); the
    graph is updated in place and the scipy result returned"""
    for _ in range(steps):
        cu, ci, _ = g.capacity
        coo = cur.tocoo()
        e = rng.integers(0, cur.nnz, n)
        kind = rng.integers(0, 3, n)
        u = np.where(kind == 0, rng.integers(0, cu, n), coo.row[e]).astype(np.int64)
        v = np.where(kind == 0, rng.integers(0, ci, n), coo.col[e]).astype(np.int64)
        x = np.where(kind == 2, 0, rng.integers(1, 6, n)).astype(np.int64)
        g.update(u, v, x)
        o = np.lexsort((v, u))
        keep = np.r_[(u[o][1:] != u[o][:-1]) | (v[o][1:] != v[o][:-1]), True]
        su, sv, sx = u[o][keep], v[o][keep], x[o][keep]
        lil = ssp.lil_matrix((g.num_users, g.num_items), dtype=np.float32)
        c2 = cur.tocoo()
        lil[c2.row, c2.col] = c2.data
        lil[su, sv] = sx.astype(np.float32)
        cur = ssp.csr_matrix(lil)
        cur.eliminate_zeros()
        cur.sort_indices()
    return cur


def test_corated_users_follow_graph_updates():
    """a chain of inserts, relabels, deletes and new users / items: the same bytes as a fresh graph of the result"""
    A = ssp.csr_matrix(support.adj("ml_100k"))
    g = RatingGraph(A, reserve_nnz=20000, reserve_users=50, reserve_items=40)
    old = g.shape
    cur = _apply_chain(g, A.copy(), np.random.default_rng(5), 4, 3000)
    assert g.shape == cur.shape and g.nnz == cur.nnz and g.shape != old
    fresh = RatingGraph(cur)
    items = np.concatenate([_query_items(cur, 40, seed=3), np.arange(old[1], g.num_items)])
    for m in (20, g.num_users):
        for exclude in (True, False):
            got = rc.corated_users(g, items, m, exclude_rated=exclude)
            want = rc.corated_users(fresh, items, m, exclude_rated=exclude)
            assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (m, exclude)
            wu, wp = _twin(fresh, items, m, exclude)
            assert np.array_equal(got[0].cpu().numpy(), wu) and np.array_equal(got[1].cpu().numpy(), wp)


@pytest.mark.parametrize("exclude", [True, False])
def test_item_and_user_side_counts_agree(exclude):
    """m = num_users and m = num_items: the dense count matrices of corated_users and corated_items are transposes"""
    A = support.adj("ml_100k")
    g = RatingGraph(A)
    nu, ni = g.shape
    iu, ip = (x.cpu().numpy() for x in rc.corated_items(g, np.arange(nu), ni, exclude_rated=exclude))
    uu, up = (x.cpu().numpy() for x in rc.corated_users(g, np.arange(ni), nu, exclude_rated=exclude))
    by_user = np.zeros((nu, ni), np.int64)
    by_item = np.zeros((ni, nu), np.int64)
    for D, ids, paths in ((by_user, iu, ip), (by_item, uu, up)):
        rows = np.repeat(np.arange(ids.shape[0]), ids.shape[1])
        keep = ids.reshape(-1) >= 0
        D[rows[keep], ids.reshape(-1)[keep]] = paths.reshape(-1)[keep]
    assert by_user.sum() > 0
    assert np.array_equal(by_user, by_item.T)


# ---- 2. the pair post-pass --------------------------------------------------------------------------------------------
def test_item_query_pairs_direct():
    """the swap and the int64 pair id at B = 1, 512, 513 and 5 000 (ids past 2^31 with many items), guard entries past
    B untouched, the error word after each case (an item id outside [0, num_items) sets it)"""
    lib = _lib.load()
    rng = np.random.default_rng(0)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    G = 16
    for B, ni, nu in ((1, 5, 7), (512, 3706, 6040), (513, 3_000_000, 1000), (5000, 3_000_000, 70_000)):
        items = rng.integers(0, ni, B + G).astype(np.int32)
        users = rng.integers(0, nu, B + G).astype(np.int32)
        lu = torch.from_numpy(items).cuda()
        lv = torch.from_numpy(users).cuda()
        pid = torch.full((B + G,), -5, dtype=torch.int64, device="cuda")
        _lib.check(lib.igmc_item_query_pairs(ni, B, lu.data_ptr(), lv.data_ptr(), pid.data_ptr(), err.data_ptr(),
                                             _stream_ptr()), "igmc_item_query_pairs")
        wu, wv, wp = rc.item_query_pairs_host(ni, items[:B], users[:B])
        assert np.array_equal(lu[:B].cpu().numpy(), wu) and np.array_equal(lv[:B].cpu().numpy(), wv), B
        assert np.array_equal(pid[:B].cpu().numpy(), wp), B
        assert np.array_equal(lu[B:].cpu().numpy(), items[B:]) and np.array_equal(lv[B:].cpu().numpy(), users[B:])
        assert (pid[B:].cpu().numpy() == -5).all()
        if ni == 3_000_000:
            assert wp.max() >= 2 ** 31
        assert int(err.item()) == 0, B
    lu = torch.tensor([2, 5, -1], dtype=torch.int32, device="cuda")
    lv = torch.tensor([1, 1, 1], dtype=torch.int32, device="cuda")
    pid = torch.zeros(3, dtype=torch.int64, device="cuda")
    _lib.check(lib.igmc_item_query_pairs(5, 3, lu.data_ptr(), lv.data_ptr(), pid.data_ptr(), err.data_ptr(),
                                         _stream_ptr()), "igmc_item_query_pairs")
    assert int(err.item()) == 7
    assert lu.tolist() == [1, 0, 0] and lv.tolist() == [2, 0, 0] and pid.tolist() == [7, 0, 0]
    assert lib.igmc_item_query_pairs(5, 0, lu.data_ptr(), lv.data_ptr(), pid.data_ptr(), err.data_ptr(),
                                     _stream_ptr()) == -1


@pytest.mark.parametrize("which", ["all", "list", "rows"])
def test_item_side_batches_match_the_twins(which):
    """the candidate kernels on the transposed view then igmc_item_query_pairs, every batch of a run and one past its
    end (the tag -1 tail), against the host twins on the transposed arrays"""
    A = support.adj("ml_100k")
    m = support.model(5)
    nu, ni = A.shape
    items = np.array([0, 50, 50, ni - 1, 7], np.int64)
    users = None if which == "all" else np.unique(np.random.default_rng(1).choice(nu, 200))
    if which == "rows":
        users = np.random.default_rng(2).integers(-1, nu, (len(items), 30))
    eng = rc.InferenceEngine(m, A, batch_size=64, max_nodes_per_hop=10)
    g = eng.graph
    trp, tci = g.host["col_ptr"].astype(np.int64), g.host["row_idx"].astype(np.int64)
    if which == "rows":
        off, lists = rc.candidate_lists_host(trp, tci, nu, items, users, True)
        cand, exclude = None, True
    else:
        cand, exclude = users, True
        plan = rc.candidate_plan_host(trp, tci, nu, items, cand, exclude)
    P = eng.start_recommend_users(items, 5, users=users)
    run = eng.run
    assert run["by_item"]
    if which == "rows":
        assert np.array_equal(run["user_off"].cpu().numpy(), off)
    else:
        assert P == int(plan[0][-1]) and np.array_equal(run["user_off"].cpu().numpy(), plan[0])
    B = 64
    cursor = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = eng.slots[0]
    err = eng.extractor.err
    for pos in range(0, P + B, B):
        _lib.check(eng.lib.igmc_candidate_pairs(C.byref(g._ct), C.byref(run["Cd"]), cursor.data_ptr(), B,
                                                s["u"].data_ptr(), s["v"].data_ptr(), s["pid"].data_ptr(),
                                                s["tag"].data_ptr(), err.data_ptr(), _stream_ptr()),
                   "igmc_candidate_pairs")
        _lib.check(eng.lib.igmc_item_query_pairs(ni, B, s["u"].data_ptr(), s["v"].data_ptr(), s["pid"].data_ptr(),
                                                 err.data_ptr(), _stream_ptr()), "igmc_item_query_pairs")
        if which == "rows":
            # per-item lists: the twin enumerates the compacted lists directly
            g_ = np.minimum(np.arange(pos, pos + B), P - 1)
            j = np.searchsorted(off, g_, side="right") - 1
            lu, lv = items[j], lists[g_].astype(np.int64)
            tag = np.where(np.arange(pos, pos + B) < P, j, -1)
        else:
            lu, lv, _, tag = rc.candidate_pairs_host(trp, tci, nu, items, cand, exclude, plan, pos, B)
        wu, wv, wp = rc.item_query_pairs_host(ni, lu, lv)
        got = np.stack([s[k].cpu().numpy().astype(np.int64) for k in ("u", "v", "pid", "tag")])
        assert np.array_equal(got, np.stack([wu, wv, wp, tag])), pos
        assert int(err.item()) == 0, pos
    eng.close()


# ---- 3. scores: recommend_users == predict_pairs ---------------------------------------------------------------------
def _item_lists(A, items, users, exclude):
    """per query item its candidate users (every user or the sorted list), without its raters when exclude"""
    nu = A.shape[0]
    base = np.arange(nu) if users is None else np.unique(users)
    return [base[~np.isin(base, _raters(A, v))] if exclude else base for v in items]


def _pair_scores(m, A, items, lists, **kw):
    """predict_pairs over every (u, v) of the lists, split per item"""
    pu = np.concatenate(lists).astype(np.int64)
    pv = np.concatenate([np.full(len(l_), v) for v, l_ in zip(items, lists)]).astype(np.int64)
    flat = rc.predict_pairs(m, A, pu, pv, **kw).cpu().numpy()
    return np.split(flat, np.cumsum([len(l_) for l_ in lists])[:-1])


def _check_lists(lists, scores, k, res):
    tu, ts = (x.cpu().numpy() for x in res)
    assert tu.shape == (len(lists), k) and res[0].dtype == torch.int64 and res[1].dtype == torch.float32
    for j in range(len(lists)):
        ws, wu = rc.rank_host(scores[j], lists[j], k)
        assert np.array_equal(tu[j], wu), (k, j)
        assert np.array_equal(ts[j], ws, equal_nan=True), (k, j)


PLANS = {
    # name: (dataset, h, mnph, model kwargs, expected plan)
    "plan 2 ml_1m": ("ml_1m", 1, 100, {}, 2),
    "plan 4 ml_100k": ("ml_100k", 1, 200, {}, 4),
    "plan 0 R=13": ("r13", 1, 50, {}, 0),
    "L2 plan ml_1m uncapped": ("ml_1m", 1, None, {}, "l2"),
    "h=2": ("ml_1m", 2, 20, {}, None),
    "pyg-2": ("ml_1m", 1, 100, dict(rgcn="pyg-2"), 2),
    "DGCNN_RS": ("ml_1m", 1, 100, dict(dgcnn=True), None),
}


@pytest.mark.parametrize("name", list(PLANS))
def test_recommend_users_scores_equal_predict_pairs(name):
    """k = 256 keeps every candidate of a 120-user list: the lists show every score, each bit for bit predict_pairs'
    at the same B and plan; rated pairs (exclude_rated=False) are scored without their target edge, as there"""
    dsn, h, mnph, kw, plan = PLANS[name]
    ds = support.dataset(dsn)
    A = ds["adj_train"]
    nu = A.shape[0]
    m = support.model(ds["num_relations"], h=h, **kw, pyg2_bias=True)
    items = _query_items(A, 2, seed=4)[[0, 2, 4, 5]]
    rng = np.random.default_rng(6)
    users = np.unique(np.concatenate([rng.choice(nu, 100, replace=False), _raters(A, items[2])[:20]]))
    opts = dict(h=h, max_nodes_per_hop=mnph, batch_size=50, sample_seed=7)
    for exclude in (True, False):
        lists = _item_lists(A, items, users, exclude)
        assert max(len(l_) for l_ in lists) <= 256
        scores = _pair_scores(m, A, items, lists, **opts)
        res = rc.recommend_users(m, A, items, 256, users=users, exclude_rated=exclude, **opts)
        _check_lists(lists, scores, 256, res)
    cl = next(iter(m._plans.values()))
    if plan == "l2":
        assert _lib.l2_csize(cl) > 0, cl
    elif plan is not None:
        assert cl == plan, (name, cl)


def test_recommend_users_three_checkpoints():
    """the ensemble score of every pair is the fp32 mean, in checkpoint order, of three single-checkpoint runs"""
    A = support.adj("ml_100k")
    m = support.model(5)
    items = np.array([0, 10, 200], np.int64)
    users = np.arange(0, 943, 9)
    opts = dict(max_nodes_per_hop=200, batch_size=50, sample_seed=3)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for c in range(3):
            paths.append(os.path.join(tmp, "model_checkpoint%d.pth" % c))
            torch.save(support.model(5, seed=c + 1).state_dict(), paths[-1])
        ens = rc.recommend_users(m, A, items, 256, users=users, checkpoints=paths, **opts)
        single = [rc.recommend_users(m, A, items, 256, users=users, checkpoints=[p], **opts) for p in paths]
    lists = _item_lists(A, items, users, True)

    def by_user(res, j):
        tu, ts = res[0][j].cpu().numpy(), res[1][j].cpu().numpy()
        keep = tu >= 0
        return dict(zip(tu[keep].tolist(), ts[keep].tolist()))
    for j in range(len(items)):
        e = by_user(ens, j)
        s = [by_user(r, j) for r in single]
        assert sorted(e) == lists[j].tolist()
        want = np.array([((np.float32(s[0][u]) + np.float32(s[1][u])) + np.float32(s[2][u])) / np.float32(3)
                         for u in lists[j]], np.float32)
        ws, wu = rc.rank_host(want, lists[j], 256)
        assert np.array_equal(ens[0][j].cpu().numpy(), wu) and np.array_equal(ens[1][j].cpu().numpy(), ws), j


# ---- 4. lists -------------------------------------------------------------------------------------------------------------
def test_recommend_users_lists_and_determinism():
    """ml_1m*: every user (an item spans many batches), a shared 300-user list and per-item rows (several items per
    batch), exclude_rated on and off, k = 1, 10 and 256; B = 50 and 256 on one plan, CUDA graphs on and off"""
    A = support.adj("ml_1m")
    nu, ni = A.shape
    m = support.model(5)
    m.kernel_plan = 1                       # the same plan at both batch sizes
    mnph = 100
    rng = np.random.default_rng(8)
    items = np.array([1, 77, 3000], np.int64)
    shared = rng.choice(nu, 300, replace=False)
    rows = rng.integers(0, nu, (len(items), 60))
    for j, v in enumerate(items):
        r = _raters(A, v)
        rows[j, :3] = r[:3][np.arange(3) % len(r)]      # raters
        rows[j, 3:6] = rows[j, 6]                       # duplicates
        rows[j, rng.choice(60, 5, replace=False)] = -1  # empty slots
    cases = [("every user", None, True, (1, 10, 256)), ("every user", None, False, (256,)),
             ("shared", shared, True, (1, 10, 256)), ("shared", shared, False, (10,)),
             ("rows", rows, True, (1, 10, 256)), ("rows", rows, False, (10,))]
    for what, users, exclude, ks in cases:
        if what == "rows":
            C_ = ssp.csc_matrix(A)
            C_.sort_indices()
            off, flat = rc.candidate_lists_host(C_.indptr, C_.indices, nu, items, users, exclude)
            lists = [flat[off[j]:off[j + 1]].astype(np.int64) for j in range(len(items))]
        else:
            lists = _item_lists(A, items, users, exclude)
        scores = _pair_scores(m, A, items, lists, max_nodes_per_hop=mnph, batch_size=50, sample_seed=3)
        first = None
        for B in (50, 256):
            for use_graph in (True, False):
                if what != "every user" and B == 256 and not use_graph:
                    continue
                eng = rc.InferenceEngine(m, A, max_nodes_per_hop=mnph, batch_size=B, sample_seed=3,
                                         use_graph=use_graph)
                res = {k: eng.recommend_users(items, k, users=users, exclude_rated=exclude) for k in ks}
                eng.close()
                for k in ks:
                    _check_lists(lists, scores, k, res[k])
                    if exclude:
                        for j, v in enumerate(items):
                            tu = res[k][0][j].cpu().numpy()
                            assert not np.isin(tu[tu >= 0], _raters(A, v)).any()
                if first is None:
                    first = res
                for k in ks:
                    assert torch.equal(res[k][0], first[k][0]) and torch.equal(res[k][1], first[k][1]), \
                        (what, exclude, B, use_graph)


def test_recommend_users_retrieve_equals_retrieved_rows():
    """retrieve=M ranks exactly the rows corated_users returns; a device tensor of rows gives the same lists"""
    A = support.adj("ml_1m")
    m = support.model(5)
    items = np.array([2, 40, 41, 1000], np.int64)
    opts = dict(max_nodes_per_hop=100, batch_size=128, sample_seed=2)
    for M in (60, 300):
        for exclude in (True, False):
            rows, _ = rc.corated_users(A, items, M, exclude_rated=exclude)
            a = rc.recommend_users(m, A, items, 20, retrieve=M, exclude_rated=exclude, **opts)
            b = rc.recommend_users(m, A, items, 20, users=rows, exclude_rated=exclude, **opts)
            c = rc.recommend_users(m, A, items, 20, users=rows.cpu().numpy(), exclude_rated=exclude, **opts)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), (M, exclude)
            assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1]), (M, exclude)
            assert (a[0] >= 0).all()
            tu = a[0].cpu().numpy()
            for j in range(len(items)):
                assert np.isin(tu[j], rows[j].cpu().numpy()).all()


# ---- 5. edge cases -------------------------------------------------------------------------------------------------------
def test_item_nobody_rated_and_a_new_item():
    """an item without ratings has no bridge (corated_users is all padding) and is still ranked against every user by
    the model; a new item added by graph.update with three ratings is ranked by an engine kept across the update as a
    fresh engine ranks it, and an update during a run makes the next step raise"""
    A = ssp.csr_matrix(support.adj("ml_100k"))
    nu, ni = A.shape
    g = RatingGraph(A, reserve_nnz=100, reserve_items=4)
    m = support.model(5)
    opts = dict(max_nodes_per_hop=200, batch_size=64, sample_seed=1)
    g.update([], [], [], shape=(nu, ni + 1))          # item ni: nobody rated it
    users, paths = rc.corated_users(g, [ni], 10)
    assert (users.cpu().numpy() == -1).all() and (paths.cpu().numpy() == 0).all()
    eng = rc.InferenceEngine(m, g, **opts)
    res = eng.recommend_users([ni], 30)
    scores = _pair_scores(m, g, [ni], [np.arange(nu)], **opts)
    _check_lists([np.arange(nu)], scores, 30, res)
    # a new item ni + 1 rated by three users; the engine serves across the update
    before = eng.recommend_users([5], 20)
    raters = np.array([3, 100, 500])
    g.update(raters, np.full(3, ni + 1), np.array([5, 4, 1]))
    kept = eng.recommend_users([ni + 1, 5], 20)
    fresh_eng = rc.InferenceEngine(m, g, **opts)
    fresh = fresh_eng.recommend_users([ni + 1, 5], 20)
    fresh_eng.close()
    assert torch.equal(kept[0], fresh[0]) and torch.equal(kept[1], fresh[1])
    h = g.host
    cur = ssp.csr_matrix((np.ones(g.nnz, np.float32), h["col_idx"], h["row_ptr"]), shape=g.shape)
    lists = _item_lists(cur, [ni + 1, 5], None, True)
    assert not np.isin(kept[0][0].cpu().numpy(), raters).any()
    _check_lists(lists, _pair_scores(m, g, [ni + 1, 5], lists, **opts), 20, kept)
    assert before[0].shape == (1, 20)
    assert (rc.corated_users(g, [ni + 1], 5)[0].cpu().numpy()[0] >= 0).any()
    eng.start_recommend_users([1, 2], 10)
    assert eng.step()
    g.update([7], [1], [3])
    with pytest.raises(RuntimeError, match="updated during this run"):
        eng.step()
    eng.close()


def test_recommend_and_recommend_users_interleaved():
    """one engine alternating user-side and item-side runs gives what separate engines give"""
    A = support.adj("ml_100k")
    m = support.model(5)
    opts = dict(max_nodes_per_hop=200, batch_size=64, sample_seed=2)
    users, items = np.array([1, 2, 300]), np.array([4, 5, 900])
    eng = rc.InferenceEngine(m, A, **opts)
    got = [eng.recommend(users, 15), eng.recommend_users(items, 15), eng.recommend(users, 15, retrieve=100),
           eng.recommend_users(items, 15, retrieve=100)]
    eng.close()
    want = []
    for call in (lambda e: e.recommend(users, 15), lambda e: e.recommend_users(items, 15),
                 lambda e: e.recommend(users, 15, retrieve=100), lambda e: e.recommend_users(items, 15, retrieve=100)):
        e = rc.InferenceEngine(m, A, **opts)
        want.append(call(e))
        e.close()
    for a, b in zip(got, want):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_recommend_users_steady_state_steps_do_not_sync():
    A = support.adj("ml_1m")
    m = support.model(5)
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=50, sample_seed=1)
    outs = []
    try:
        for retrieve in (None, None, 500):
            P = eng.start_recommend_users([11, 12], 25, retrieve=retrieve)
            assert P > 8 * 50
            for _ in range(4):          # eager warm-up and capture of both batch slots
                eng.step()
            assert len(eng.graphs) == 2
            torch.cuda.set_sync_debug_mode("error")
            try:
                while eng.step():
                    pass
            finally:
                torch.cuda.set_sync_debug_mode("default")
            outs.append(eng.finish())
            assert int(eng.extractor.err.item()) == 0
    finally:
        eng.close()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
