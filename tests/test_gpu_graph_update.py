"""In-place updates of the device rating graph (RatingGraph.update, csrc/graph_update.cu).

* the kernels against the numpy twin (tests/test_graph_update_host.py) and against RatingGraph(A_updated), byte for
  byte, on ml_100k*, ml_1m* and the flixster fixture with deltas of 1, 1 000 and 100 000 entries; a chain of 20
  updates; users and items grown up to the capacity;
* capacity overflow and invalid device input leave the graph unchanged; the five device pointers never change;
* an extractor and an InferenceEngine kept across updates give the bits a fresh one on RatingGraph(A_updated) gives;
* an update during an engine run, and a TrainEngine whose graph changed after its first step, raise."""

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import recommend as rc
from igmc_b200.data import make_synthetic_dataset
from igmc_b200.util_functions import RatingGraph, SubgraphExtractor, graph_update_host
from tests import support

pytestmark = pytest.mark.gpu

ARRAYS = ("row_ptr", "col_idx", "rating", "col_ptr", "row_idx")


def _apply_scipy(A, u, v, x, shape):
    """A with the delta applied (last occurrence of a pair wins, value 0 deletes), at ``shape``"""
    A = ssp.csr_matrix(A)
    M = np.int64(max(shape[1], 1))
    o = np.lexsort((v, u))
    su, sv, sx = u[o], v[o], x[o]
    keep = np.r_[(su[1:] != su[:-1]) | (sv[1:] != sv[:-1]), True]
    su, sv, sx = su[keep], sv[keep], sx[keep]
    coo = A.tocoo()
    okey = coo.row.astype(np.int64) * M + coo.col
    stay = ~np.isin(okey, su * M + sv)
    ins = sx > 0
    r = np.concatenate([coo.row[stay], su[ins]])
    c = np.concatenate([coo.col[stay], sv[ins]])
    d = np.concatenate([coo.data[stay], sx[ins].astype(np.float32)])
    return ssp.csr_matrix((d, (r, c)), shape=shape, dtype=np.float32)


def _random_delta(rng, A, n, cap_users, cap_items, R):
    """inserts (new users / items up to the capacity included), overwrites, deletes, deletes of absent pairs and
    repeated pairs"""
    coo = A.tocoo()
    k = rng.integers(0, 4, n)
    e = rng.integers(0, max(A.nnz, 1), n)
    u = np.where(k < 2, coo.row[e] if A.nnz else 0, rng.integers(0, cap_users, n)).astype(np.int64)
    v = np.where(k < 2, coo.col[e] if A.nnz else 0, rng.integers(0, cap_items, n)).astype(np.int64)
    x = np.where((k == 0) | (k == 2), rng.integers(1, R + 1, n), 0).astype(np.int64)
    if n >= 5:
        dup = rng.integers(0, n, n // 5)
        u, v = np.concatenate([u, u[dup]]), np.concatenate([v, v[dup]])
        x = np.concatenate([x, rng.integers(0, R + 1, len(dup))])
    return u, v, x


def _assert_graph_equal(g, A_want):
    """g's arrays (cut to nnz and shape) and fields are those of a graph built from A_want"""
    f = RatingGraph(A_want)
    for k in ARRAYS:
        assert np.array_equal(g.host[k], f.host[k]) and g.host[k].dtype == f.host[k].dtype, k
        n = len(f.host[k])
        assert torch.equal(g.dev[k][:n], f.dev[k][:n]), k
    assert g.shape == f.shape and g.nnz == f.nnz
    assert (g.num_users, g.num_items, g.max_row_deg, g.max_col_deg) == \
        (f.num_users, f.num_items, f.max_row_deg, f.max_col_deg)
    assert (g._c.num_users, g._c.num_items) == g.shape


@pytest.mark.parametrize("name", ["ml_100k", "ml_1m", "flixster"])
def test_update_matches_twin_and_rebuild(name):
    ds = support.dataset(name)
    A, R = ds["adj_train"], ds["num_relations"]
    rng = np.random.default_rng(5)
    for n in (1, 1000, 100000):
        g = RatingGraph(A, reserve_nnz=n, reserve_users=7, reserve_items=5)
        cu, ci, _ = g.capacity
        u, v, x = _random_delta(rng, A, n, cu, ci, R)
        before = g.host
        want_h, hdr = graph_update_host(before, g.shape, u, v, x)
        counts = g.update(u, v, x)
        assert counts == dict(inserted=hdr["inserted"], changed=hdr["changed"], removed=hdr["removed"])
        for k in ARRAYS:
            assert np.array_equal(g.host[k], want_h[k]), (name, n, k)
        assert (g.nnz, g.num_users, g.num_items, g.max_row_deg, g.max_col_deg) == \
            (hdr["nnz"], hdr["num_users"], hdr["num_items"], hdr["max_row_deg"], hdr["max_col_deg"])
        _assert_graph_equal(g, _apply_scipy(A, u, v, x, g.shape))
        assert g.version == (1 if any(counts.values()) or g.shape != A.shape else 0)


def test_chain_of_updates_and_growth_to_capacity():
    ds = support.dataset("ml_100k")
    A = ds["adj_train"]
    g = RatingGraph(A, reserve_nnz=20000, reserve_users=40, reserve_items=30)
    cu, ci, _ = g.capacity
    ptrs = [g.dev[k].data_ptr() for k in ARRAYS]
    rng = np.random.default_rng(9)
    for step in range(20):
        u, v, x = _random_delta(rng, A, int(rng.integers(1, 3000)), g.num_users + 2, g.num_items + 2, 5)
        shape = (g.num_users + 1, g.num_items) if step == 7 else None
        g.update(u, v, x, shape=shape)
        A = _apply_scipy(A, u, v, x, g.shape)
        _assert_graph_equal(g, A)
    # the last user and item of the capacity; shape= with an empty delta adds empty rows / columns
    g.update([cu - 1, 0], [3, ci - 1], [4, 2])
    A = _apply_scipy(A, np.array([cu - 1, 0]), np.array([3, ci - 1]), np.array([4, 2]), (cu, ci))
    _assert_graph_equal(g, A)
    assert g.shape == (cu, ci)
    assert [g.dev[k].data_ptr() for k in ARRAYS] == ptrs


def test_shape_only_and_noop_updates():
    A = support.adj("ml_100k")
    g = RatingGraph(A, reserve_users=3, reserve_items=2)
    v0 = g.version
    coo = A.tocoo()
    # the same labels again and deletes of absent pairs: nothing changes, the version stays
    assert g.update(coo.row[:5], coo.col[:5], coo.data[:5].astype(np.int64)) == dict(inserted=0, changed=0, removed=0)
    dense_free = (0, int(np.setdiff1d(np.arange(A.shape[1]), A.indices[A.indptr[0]:A.indptr[1]])[0]))
    g.update([dense_free[0]], [dense_free[1]], [0])
    assert g.version == v0
    g.update([], [], [], shape=(A.shape[0] + 2, A.shape[1] + 1))
    assert g.version == v0 + 1
    coo = A.tocoo()
    _assert_graph_equal(g, ssp.csr_matrix((coo.data, (coo.row, coo.col)), shape=(A.shape[0] + 2, A.shape[1] + 1)))


def test_overflow_and_invalid_device_input_leave_the_graph():
    A = support.adj("ml_100k")
    g = RatingGraph(A, reserve_nnz=10, reserve_users=2)
    snap = {k: t.clone() for k, t in g.dev.items()}
    fields = (g.shape, g.nnz, g.max_row_deg, g.max_col_deg, g.version)
    free = np.setdiff1d(np.arange(A.shape[1]), A.indices[A.indptr[0]:A.indptr[1]])[:11]
    with pytest.raises(ValueError, match="capacity"):
        g.update(np.zeros(11, np.int64), free, np.full(11, 3))
    bad = torch.tensor([1, A.shape[0] + 2], dtype=torch.int32, device="cuda")        # beyond the user capacity
    with pytest.raises(RuntimeError, match="graph update"):
        g.update(bad, torch.tensor([0, 0], dtype=torch.int32, device="cuda"),
                 torch.tensor([1, 1], dtype=torch.int32, device="cuda"))
    with pytest.raises(RuntimeError, match="graph update"):
        g.update(torch.tensor([1], device="cuda"), torch.tensor([0], device="cuda"), torch.tensor([300], device="cuda"))
    for k in ARRAYS:
        assert torch.equal(g.dev[k], snap[k]), k
    assert (g.shape, g.nnz, g.max_row_deg, g.max_col_deg, g.version) == fields
    # the graph still takes updates; int32 device tensors are used in place
    g.update(torch.zeros(10, dtype=torch.int32, device="cuda"), torch.as_tensor(free[:10], device="cuda").int(),
             torch.full((10,), 2, dtype=torch.int32, device="cuda"))
    assert g.nnz == A.nnz + 10


# ---- consumers --------------------------------------------------------------------------------------------------------
def _grow_delta(A, rng, n, R=5):
    """random inserts / deletes plus 300 ratings into the longest row and the longest column (the largest degree,
    and so cap without max_nodes_per_hop, grows)"""
    nu, ni = A.shape
    u, v, x = _random_delta(rng, A, n, nu, ni, R)
    hot_u, hot_i = int(np.argmax(np.diff(A.indptr))), int(np.argmax(np.diff(A.tocsc().indptr)))
    hu, hv = np.full(300, hot_u), rng.choice(ni, 300, replace=False)
    iu, iv = rng.choice(nu, 300, replace=False), np.full(300, hot_i)
    return (np.concatenate([u, hu, iu]), np.concatenate([v, hv, iv]),
            np.concatenate([x, rng.integers(1, R + 1, 600)]))


def _batch_arrays(b):
    b.check()
    return [t.cpu() for t in (b.x, b.edge_index, b.edge_type, b.node_label, b.node_gid, b.y, b.batch)] + \
        [b._priv["node_ptr"].cpu(), b._priv["edge_ptr"].cpu()]


@pytest.mark.parametrize("h,mnph,fast", [(1, None, True), (1, 100, True), (1, None, False), (1, 100, False),
                                         (2, 30, True), (2, None, True)])
def test_extractor_follows_updates(h, mnph, fast):
    A = support.adj("ml_100k")
    g = RatingGraph(A, reserve_nnz=10000)
    cv = np.arange(1, 6, dtype=np.float32)
    kept = SubgraphExtractor(g, [0], [0], [0], cv, h, 1.0, mnph, max_batch=64, seed=3, fast=fast)
    rng = np.random.default_rng(h * 7 + (mnph or 0))
    caps = [kept.cap]
    for step in range(3):
        u, v, x = _grow_delta(A, rng, 2000)
        g.update(u, v, x)
        A = _apply_scipy(A, u, v, x, g.shape)
        fresh = SubgraphExtractor(RatingGraph(A), [0], [0], [0], cv, h, 1.0, mnph, max_batch=64, seed=3, fast=fast)
        pu = np.concatenate([[10 + step, 5], rng.integers(0, A.shape[0], 62)])
        pv = np.concatenate([[3, 20 + step], rng.integers(0, A.shape[1], 62)])
        pl = rng.integers(0, 5, 64)
        pid = pu * A.shape[1] + pv
        got = _batch_arrays(kept.extract(pairs=(pu, pv, pl), pair_ids=pid))
        assert kept.cap == fresh.cap
        want = _batch_arrays(fresh.extract(pairs=(pu, pv, pl), pair_ids=pid))
        for a, b in zip(got, want):
            assert torch.equal(a, b), (h, mnph, fast, step)
        caps.append(kept.cap)
    if mnph is None and h == 1:
        assert caps[-1] > caps[0]            # the workspace was re-reserved for the grown degrees


@pytest.mark.parametrize("case", ["ml_1m plan 2", "r13 plan 0"])
def test_engine_serves_across_updates(case):
    if case == "ml_1m plan 2":
        A, R, mnph, plan = support.adj("ml_1m"), 5, 100, 2
    else:
        A, R, mnph, plan = support.adj("r13"), 13, 50, 0
    m = support.model(R)
    g = RatingGraph(A, reserve_nnz=5000, reserve_users=3, reserve_items=2)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=mnph, batch_size=50, sample_seed=5)
    rng = np.random.default_rng(1)
    try:
        for step in range(3):
            nu, ni = g.shape
            u, v, x = _random_delta(rng, A, 1500, nu, ni, R)
            if step == 1:        # a new user with a handful of ratings, and a new item
                new_u, new_i = nu, ni
                items = rng.choice(ni, 6, replace=False)
                u = np.concatenate([u, np.full(6, new_u), [3]])
                v = np.concatenate([v, items, [new_i]])
                x = np.concatenate([x, rng.integers(1, R + 1, 7)])
            g.update(u, v, x)
            A = _apply_scipy(A, u, v, x, g.shape)
            users = np.array([0, 7, g.shape[0] - 1])
            pu, pv = rng.integers(0, g.shape[0], 130), rng.integers(0, g.shape[1], 130)
            got_s = eng.predict_pairs(pu, pv)
            got_t = eng.recommend(users, 10)
            fresh = rc.InferenceEngine(m, RatingGraph(A), max_nodes_per_hop=mnph, batch_size=50, sample_seed=5)
            want_s = fresh.predict_pairs(pu, pv)
            want_t = fresh.recommend(users, 10)
            fresh.close()
            assert torch.equal(got_s, want_s), (case, step)
            assert torch.equal(got_t[0], want_t[0]) and torch.equal(got_t[1], want_t[1]), (case, step)
            assert next(iter(m._plans.values())) == plan
            if step >= 1:
                ti = got_t[0][2].cpu().numpy() if g.shape[0] - 1 == new_u else None
                if ti is not None:
                    rated = A.indices[A.indptr[new_u]:A.indptr[new_u + 1]]
                    assert (ti >= 0).all() and not np.isin(ti, rated).any()
    finally:
        eng.close()


def test_update_during_a_run_raises():
    A = support.adj("ml_100k")
    m = support.model(5)
    g = RatingGraph(A, reserve_nnz=10)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=50, batch_size=50)
    eng.start_recommend([1, 2, 3], 5)
    eng.step()
    free = np.setdiff1d(np.arange(A.shape[1]), A.indices[A.indptr[1]:A.indptr[2]])[0]
    g.update([1], [free], [3])
    with pytest.raises(RuntimeError, match="updated"):
        eng.step()
    ti, _ = eng.recommend([1, 2, 3], 5)          # the next run serves the updated graph
    assert ti.shape == (3, 5)
    eng.close()


def test_train_engine_refuses_a_changed_graph():
    from igmc_b200.models import IGMC
    from igmc_b200.train_eval import FusedAdam, TrainEngine
    from igmc_b200.util_functions import MyDynamicDataset
    ds = make_synthetic_dataset("tiny", seed=0)
    tu, tv, tl = ds["train"]
    g = RatingGraph(ds["adj_train"], reserve_nnz=4)
    d = MyDynamicDataset(None, g, (tu, tv), tl, 1, 1.0, 10, None, None, ds["class_values"])
    torch.manual_seed(0)
    m = IGMC(d, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    eng = TrainEngine(d, m, FusedAdam(m, lr=1e-3), 8)
    g.update([0], [0], [2])                      # before the first step: trained on as it is
    eng.step(np.arange(8))
    eng.step(np.arange(8, 16))
    g.update([1], [1], [0 if ds["adj_train"][1, 1] else 3])
    with pytest.raises(RuntimeError, match="updated"):
        eng.step(np.arange(8))
    eng.close()
