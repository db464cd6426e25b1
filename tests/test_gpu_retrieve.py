"""Candidate retrieval by bridge count and per-user candidate lists on the GPU (csrc/retrieve.cu, csrc/recommend.cu).

* corated_items against its host twin (tests/test_retrieve_host.py) byte for byte on ml_100k*, ml_1m*, the real
  flixster split and tiny, on a shape whose histograms do not fit in shared memory, and after a chain of graph
  updates; two runs are bit-identical;
* recommend(items=<2-D>) against a stable sort of predict_pairs over each user's deduplicated unrated list, on the
  relation-space, generic (R = 13) and L2 plans, B = 50 and 256, CUDA graphs on and off;
* recommend(retrieve=M) against recommend(items=corated_items(...)), and retrieve=num_items against the full
  catalogue restricted to the items with a bridge;
* steady-state steps of a retrieve run do not synchronise."""
import ctypes

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.data import build_adj, synth_ratings
from igmc_b200.util_functions import RatingGraph
from tests import support

pytestmark = pytest.mark.gpu


def _twin(g, users, m, exclude):
    h = g.host
    return rc.corated_host(h["row_ptr"], h["col_idx"], g.num_users, g.num_items, users, m, exclude)


def _query_users(nu, A, n, seed):
    rng = np.random.default_rng(seed)
    deg = np.diff(A.indptr)
    users = [int(np.argmax(deg)), int(np.argmin(deg)), 0, nu - 1]
    return np.array(users + rng.choice(nu, n, replace=False).tolist(), np.int64)


# ---- 1. the retriever against its twin ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["ml_100k", "ml_1m", "flixster", "tiny"])
def test_corated_items_match_twin(name):
    A = support.adj(name)
    g = RatingGraph(A)
    nu, ni = g.shape
    users = _query_users(nu, A, min(60, nu - 4), seed=1)
    for m in sorted({1, 50, 500, ni} & set(range(1, ni + 1))):
        for exclude in (True, False):
            items, paths = rc.corated_items(g, users, m, exclude_rated=exclude)
            assert items.shape == (len(users), m) and items.dtype == torch.int32 and paths.dtype == torch.int32
            wi, wp = _twin(g, users, m, exclude)
            assert np.array_equal(items.cpu().numpy(), wi), (name, m, exclude)
            assert np.array_equal(paths.cpu().numpy(), wp), (name, m, exclude)
            again = rc.corated_items(g, users, m, exclude_rated=exclude)
            assert torch.equal(items, again[0]) and torch.equal(paths, again[1])


def test_corated_items_global_memory_regime():
    """60 000 users x 2 000 items: the histograms (248 KB) do not fit in shared memory"""
    nu, ni = 60000, 2000
    u, v, lab = synth_ratings(nu, ni, 150000, 5, seed=9)
    A = build_adj(u, v, lab, nu, ni)
    g = RatingGraph(A)
    users = _query_users(nu, A, 300, seed=2)        # more users than the global-memory grid has CTAs
    for m in (1, 100, ni):
        nbytes = ctypes.c_int64(0)
        assert _lib.load().igmc_corated_ws_bytes(nu, ni, len(users), m, ctypes.byref(nbytes)) == 0
        assert nbytes.value > 0
        items, paths = rc.corated_items(g, users, m)
        wi, wp = _twin(g, users, m, True)
        assert np.array_equal(items.cpu().numpy(), wi), m
        assert np.array_equal(paths.cpu().numpy(), wp), m
        assert torch.equal(items, rc.corated_items(g, users, m)[0])


def test_corated_items_follow_graph_updates():
    """a chain of inserts, relabels, deletes and new users / items: the same bytes as a fresh graph of the result"""
    A = ssp.csr_matrix(support.adj("ml_100k"))
    g = RatingGraph(A, reserve_nnz=20000, reserve_users=50, reserve_items=40)
    rng = np.random.default_rng(5)
    cur = A.copy()
    for step in range(4):
        cu, ci, _ = g.capacity
        n = 3000
        coo = cur.tocoo()
        e = rng.integers(0, cur.nnz, n)
        kind = rng.integers(0, 3, n)
        u = np.where(kind == 0, rng.integers(0, cu, n), coo.row[e]).astype(np.int64)
        v = np.where(kind == 0, rng.integers(0, ci, n), coo.col[e]).astype(np.int64)
        x = np.where(kind == 2, 0, rng.integers(1, 6, n)).astype(np.int64)
        g.update(u, v, x)
        # the scipy result of the same delta (last occurrence wins, 0 deletes)
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
    assert g.shape == cur.shape and g.nnz == cur.nnz
    fresh = RatingGraph(cur)
    users = _query_users(g.num_users, cur, 40, seed=3)
    for m in (20, g.num_items):
        got = rc.corated_items(g, users, m)
        want = rc.corated_items(fresh, users, m)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), m
        wi, _ = _twin(fresh, users, m, True)
        assert np.array_equal(got[0].cpu().numpy(), wi)


# ---- 2. per-user candidate lists in the ranking engine ----------------------------------------------------------------
def _rows(A, users, width, seed):
    """per-user rows with duplicates, rated items and -1 slots"""
    rng = np.random.default_rng(seed)
    ni = A.shape[1]
    rows = rng.integers(0, ni, (len(users), width)).astype(np.int64)
    for j, u in enumerate(users):
        rated = A.indices[A.indptr[u]:A.indptr[u + 1]]
        if len(rated):
            rows[j, :3] = rated[:3][np.arange(3) % len(rated)]
        rows[j, 3:6] = rows[j, 6]                     # duplicates
        rows[j, rng.choice(width, 4, replace=False)] = -1
    rows[-1] = -1                                     # a user with no candidate at all
    return rows


def _check_against_predict(m, A, users, rows, exclude, k, ti_ts, mnph, seed):
    """the ranked lists equal a stable sort of predict_pairs over each user's deduplicated (unrated) list"""
    off, lists = rc.candidate_lists_host(A.indptr, A.indices, A.shape[1], users, rows, exclude)
    per = [lists[off[j]:off[j + 1]].astype(np.int64) for j in range(len(users))]
    pu = np.concatenate([np.full(len(p), u) for u, p in zip(users, per)])
    pv = np.concatenate(per)
    flat = rc.predict_pairs(m, A, pu, pv, max_nodes_per_hop=mnph, batch_size=64, sample_seed=seed).cpu().numpy() \
        if len(pu) else np.zeros(0, np.float32)
    scores = np.split(flat, np.cumsum([len(p) for p in per])[:-1])
    ti, ts = (x.cpu().numpy() for x in ti_ts)
    for j in range(len(users)):
        ws, wi = rc.rank_host(scores[j], per[j], k)
        assert np.array_equal(ti[j], wi), j
        assert np.array_equal(ts[j], ws, equal_nan=True), j


PLANS = {
    # name: (dataset, mnph, expected plan)
    "relation-space ml_1m": ("ml_1m", 100, 2),
    "plan 0 R=13": ("r13", 50, 0),
    "L2 plan ml_100k uncapped": ("ml_100k", None, "l2"),
}


@pytest.mark.parametrize("name", list(PLANS))
def test_recommend_per_user_lists(name):
    dsn, mnph, plan = PLANS[name]
    ds = support.dataset(dsn)
    A = ds["adj_train"]
    m = support.model(ds["num_relations"])
    users = np.array([3, 10, 10, 25, 7], np.int64)
    rows = _rows(A, users, 40, seed=4)
    first = None
    for B in (50, 256):
        for use_graph in (True, False):
            eng = rc.InferenceEngine(m, A, max_nodes_per_hop=mnph, batch_size=B, sample_seed=5, use_graph=use_graph)
            res = eng.recommend(users, 10, items=rows)
            eng.close()
            if first is None:
                first = res
                _check_against_predict(m, A, users, rows, True, 10, res, mnph, 5)
            assert torch.equal(res[0], first[0]) and torch.equal(res[1], first[1]), (B, use_graph)
    cl = next(iter(m._plans.values()))
    if plan == "l2":
        assert _lib.l2_csize(cl) > 0
    else:
        assert cl == plan, (name, cl)
    # rated items compete when exclude_rated is False; a device tensor gives the same lists as the host array
    res = rc.recommend(m, A, users, 25, items=rows, exclude_rated=False, max_nodes_per_hop=mnph, batch_size=50,
                       sample_seed=5)
    _check_against_predict(m, A, users, rows, False, 25, res, mnph, 5)
    dev = rc.recommend(m, A, users, 25, items=torch.as_tensor(rows, device="cuda"), exclude_rated=False,
                       max_nodes_per_hop=mnph, batch_size=50, sample_seed=5)
    assert torch.equal(res[0], dev[0]) and torch.equal(res[1], dev[1])


def test_recommend_retrieve_equals_retrieved_lists():
    ds = support.dataset("ml_1m")
    A, mnph = ds["adj_train"], 100
    m = support.model(5)
    users = np.array([2, 40, 41, 1000], np.int64)
    items, _ = rc.corated_items(A, users, 60)
    a = rc.recommend(m, A, users, 20, retrieve=60, max_nodes_per_hop=mnph, batch_size=128, sample_seed=2)
    b = rc.recommend(m, A, users, 20, items=items, max_nodes_per_hop=mnph, batch_size=128, sample_seed=2)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert (a[0] >= 0).all()


def test_retrieve_all_items_equals_bridged_full_catalogue():
    """retrieve=num_items ranks exactly the unrated items with at least one bridge"""
    ds = support.dataset("ml_100k")
    A, mnph = ds["adj_train"], 200
    m = support.model(5)
    g = RatingGraph(A)
    ni = g.num_items
    users = np.array([5, 300], np.int64)
    ti, ts = rc.recommend(m, A, users, 50, retrieve=ni, max_nodes_per_hop=mnph, batch_size=256, sample_seed=4)
    wi_all, wp_all = _twin(g, users, ni, True)
    for j, u in enumerate(users):
        unrated = np.setdiff1d(np.arange(ni), A.indices[A.indptr[u]:A.indptr[u + 1]])
        full = rc.predict_pairs(m, A, np.full(len(unrated), u), unrated, max_nodes_per_hop=mnph, batch_size=256,
                                sample_seed=4).cpu().numpy()
        bridged = set(wi_all[j][wp_all[j] > 0].tolist())
        keep = np.array([v in bridged for v in unrated])
        assert keep.sum() == len(bridged)
        ws, wi = rc.rank_host(full[keep], unrated[keep], 50)
        assert np.array_equal(ti[j].cpu().numpy(), wi), j
        assert np.array_equal(ts[j].cpu().numpy(), ws, equal_nan=True), j


def test_retrieve_steady_state_steps_do_not_sync():
    ds = support.dataset("ml_1m")
    A = ds["adj_train"]
    m = support.model(5)
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=50, sample_seed=1)
    outs = []
    try:
        for rep in range(2):
            P = eng.start_recommend([11, 12, 13], 25, retrieve=500)
            assert P > 20 * 50
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


def test_invalid_device_rows_set_the_error_word():
    """device rows are checked by the kernel: an id outside [-1, num_items) is a kernel error, nothing is scored"""
    ds = support.dataset("tiny")
    A = ds["adj_train"]
    m = support.model(5)
    rows = torch.tensor([[0, 1, A.shape[1]]], device="cuda")
    with pytest.raises(RuntimeError, match="kernel error 7"):
        rc.recommend(m, A, [0], 3, items=rows, max_nodes_per_hop=10, batch_size=16)
