"""OnlineTrainer and its pair draw on the GPU (csrc/online.cu, igmc_b200/train_eval.py).

* igmc_online_draw / igmc_online_recent_append against their numpy twins, bit for bit, on ml_1m* and the tiny graph,
  B = 1 / 50 / 512, a window with deleted, changed and repeated pairs and wrap-around, users and items added by update;
* ten trainer steps against the same steps driven through the per-step calls (extract on the twin's pairs, then
  forward_backward + reduce_update or fused_step + FusedAdam.step), bit for bit in the parameters, both Adam moments and
  the loss, on the relation-space and generic plans, DGCNN_RS, rgcn="pyg-2" and without CUDA graphs;
* a trainer kept across a chain of updates (cap grows, the workspace is re-reserved) against a fresh trainer per update;
* an InferenceEngine built before fine-tuning serves the new weights; fine-tuning on held-out ratings lowers their RMSE;
* the argument checks."""
import ctypes as C
import functools

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200 import train_eval as te
from igmc_b200.data import build_adj, synth_ratings
from igmc_b200.models import IGMC, FusedAdam
from igmc_b200.train_eval import OnlineTrainer, online_draw_host, recent_append_host, recent_threshold
from igmc_b200.util_functions import RatingGraph, SubgraphExtractor, _stream_ptr
from tests import support

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _small(R=5, nu=300, ni=200, nnz=4000, seed=4):
    u, v, lab = synth_ratings(nu, ni, nnz, R, seed=seed)
    return build_adj(u, v, lab, nu, ni)


def _apply_scipy(A, u, v, x, shape):
    """A with the delta applied (last occurrence of a pair wins, value 0 deletes), at ``shape``"""
    A = ssp.csr_matrix(A)
    M = np.int64(max(shape[1], 1))
    u, v, x = (np.asarray(t, np.int64) for t in (u, v, x))
    o = np.lexsort((v, u))
    su, sv, sx = u[o], v[o], x[o]
    last = np.r_[(su[1:] != su[:-1]) | (sv[1:] != sv[:-1]), True]
    su, sv, sx = su[last], sv[last], sx[last]
    coo = A.tocoo()
    stay = ~np.isin(coo.row.astype(np.int64) * M + coo.col, su * M + sv)
    ins = sx > 0
    r = np.concatenate([coo.row[stay], su[ins]])
    c = np.concatenate([coo.col[stay], sv[ins]])
    d = np.concatenate([coo.data[stay], sx[ins].astype(np.float32)])
    return ssp.csr_matrix((d, (r, c)), shape=shape, dtype=np.float32)


def _i64(x):
    return torch.tensor([te._u64_as_i64(int(x))], dtype=torch.int64, device="cuda")


# ---- 1. the kernels against the twins ------------------------------------------------------------------------------
class _Ring(object):
    def __init__(self, cap):
        dev = "cuda"
        self.u = torch.zeros(cap, dtype=torch.int32, device=dev)
        self.v = torch.zeros(cap, dtype=torch.int32, device=dev)
        self.total = torch.zeros(1, dtype=torch.int64, device=dev)
        self.host = (np.zeros(cap, np.int32), np.zeros(cap, np.int32), 0)

    def append(self, u, v, x, err):
        t = [torch.as_tensor(np.asarray(a), dtype=torch.int32).cuda() for a in (u, v, x)]
        _lib.check(_lib.load().igmc_online_recent_append(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), len(u),
                                                         self.u.data_ptr(), self.v.data_ptr(), self.u.numel(),
                                                         self.total.data_ptr(), err.data_ptr(), _stream_ptr()), "append")
        self.host = recent_append_host(*self.host, u, v, x)
        assert np.array_equal(self.u.cpu().numpy(), self.host[0]) and np.array_equal(self.v.cpu().numpy(), self.host[1])
        assert int(self.total) == self.host[2]


def _draw_dev(g, ring, frac, count, ahead, ss, ds, B, err):
    dev = "cuda"
    out = dict(u=torch.full((B,), -7, dtype=torch.int32, device=dev), v=torch.full((B,), -7, dtype=torch.int32, device=dev),
               lab=torch.full((B,), -7, dtype=torch.int32, device=dev), pid=torch.full((B,), -7, dtype=torch.int64, device=dev),
               seeds=torch.zeros(3, dtype=torch.int64, device=dev))
    sc = torch.tensor([count, 0], dtype=torch.int64, device=dev)
    _lib.check(_lib.load().igmc_online_draw(C.byref(g._c), ring.u.data_ptr(), ring.v.data_ptr(), ring.u.numel(),
                                            ring.total.data_ptr(), recent_threshold(frac), sc.data_ptr(), ahead, ss, ds,
                                            B, out["u"].data_ptr(), out["v"].data_ptr(), out["lab"].data_ptr(),
                                            out["pid"].data_ptr(), out["seeds"].data_ptr(), err.data_ptr(),
                                            _stream_ptr()), "draw")
    return {k: t.cpu().numpy() for k, t in out.items()}


def _check_draw(g, ring, frac, count, ahead, B, err, ss=17, ds=0x1234ABCD):
    got = _draw_dev(g, ring, frac, count, ahead, ss, ds, B, err)
    h = g.host
    u, v, lab, pid, seeds, win = online_draw_host(h["row_ptr"], h["col_idx"], h["rating"], g.num_items, *ring.host,
                                                  recent_threshold(frac), count + ahead, ss, ds, B)
    assert np.array_equal(got["u"], u) and np.array_equal(got["v"], v)
    assert np.array_equal(got["lab"], lab) and np.array_equal(got["pid"], pid)
    assert np.array_equal(got["seeds"].view(np.uint64), seeds)
    return win


@pytest.mark.parametrize("name", ["ml_1m", "tiny"])
def test_draw_matches_twin(name):
    A = support.adj(name)
    g = RatingGraph(A, reserve_nnz=5000, reserve_users=4, reserve_items=3)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(2)
    cap = 64
    ring = _Ring(cap)
    for B in (1, 50, 512):
        _check_draw(g, ring, 0.5, 3, 1, B, err)          # empty window
    coo = A.tocoo()
    seen = 0
    for rnd in range(4):
        nu, ni = g.shape
        e = rng.integers(0, coo.nnz, 40)
        u, v = coo.row[e].astype(np.int64), coo.col[e].astype(np.int64)
        x = rng.integers(1, 6, 40)
        u, v, x = np.concatenate([u, u[:5]]), np.concatenate([v, v[:5]]), np.concatenate([x, x[:5]])   # repeated pairs
        if rnd == 1:        # a new user and a new item
            u, v, x = np.concatenate([u, [nu, nu, 2]]), np.concatenate([v, [0, 1, ni]]), np.concatenate([x, [3, 4, 5]])
        g.update(u, v, x)
        ring.append(u, v, x, err)
        # deletes and changes of window pairs after they were appended
        d = rng.choice(len(u), 12, replace=False)
        g.update(u[d[:6]], v[d[:6]], np.zeros(6, np.int64))
        g.update(u[d[6:]], v[d[6:]], rng.integers(1, 6, 6))
        for B in (1, 50, 512):
            for frac in (0.0, 0.6, 1.0):
                win = _check_draw(g, ring, frac, 1000 * rnd + B, rnd & 1, B, err)
                seen += int(win.sum())
    assert ring.host[2] > cap and seen > 0         # wrapped around; window draws happened
    assert int(err.item()) == 0


# ---- 2. ten trainer steps against the per-step calls -----------------------------------------------------------------
def _manual_steps(m, opt, g, mnph, B, ARR, steps, ss, window, frac, cv):
    """the trainer's steps through the per-step calls: pairs from the twin at step counter + k"""
    ex = SubgraphExtractor(g, [0], [0], [0], cv, 1, 1.0, mnph, max_batch=B, seed=ss)
    lr = torch.full((1,), float(opt.param_groups[0]["lr"]), dtype=torch.float32, device="cuda")
    acc = torch.zeros(1, dtype=torch.float32, device="cuda")
    c0 = int(opt.step_count[0])
    exchange = None
    h = g.host
    for k in range(steps):
        u, v, lab, pid, seeds, _ = online_draw_host(h["row_ptr"], h["col_idx"], h["rating"], g.num_items, *window,
                                                    recent_threshold(frac), c0 + k, ss, m.drop_seed, B)
        b = ex.extract(pairs=(u, v, lab), pair_ids=pid, seed_dev=_i64(seeds[0]))
        drop = _i64(seeds[2])
        m.stage_batch(b, True, m.make_dropout(True, seed_dev=drop))
        if m.fused_update_ok(b):
            if exchange is None:
                from igmc_b200.exchange import Exchange
                exchange = Exchange(m.flat_params.numel(), m.flat_params.device, 0, 1)
            ws = m.forward_backward(b, global_num_graphs=B, seed_dev=drop)["ws"]
            opt.reduce_update(exchange, ws, B, B * ws["cluster"], 1.0 / B, ARR, lr_dev=lr, loss_acc=acc,
                              loss_weight=float(B))
        else:
            loss = m.fused_step(b, ARR=ARR, global_num_graphs=B, seed_dev=drop)
            opt.step(grad_mul=1.0, lr_dev=lr, loss_in=loss, loss_acc=acc, loss_weight=float(B))
    torch.cuda.synchronize()
    if exchange is not None:
        exchange.close()
    return float(acc.item()) / (steps * B)


def _state(m, opt):
    return [t.detach().cpu().clone() for t in (m.flat_params, opt.exp_avg, opt.exp_avg_sq)]


CASES = {"ml_1m rs": ("ml_1m", "igmc", 5, "pyg-1.4", 100, True),
         "r13 generic": ("r13", "igmc", 13, "pyg-1.4", 50, True),
         "dgcnn": ("ml_1m", "dgcnn", 5, "pyg-1.4", 100, True),
         "pyg-2": ("ml_1m", "igmc", 5, "pyg-2", 100, True),
         "no graph": ("ml_1m", "igmc", 5, "pyg-1.4", 100, False)}


@pytest.mark.parametrize("case", list(CASES))
def test_trainer_steps_match_per_step_calls(case):
    name, kind, R, rgcn, mnph, use_graph = CASES[case]
    A = support.adj("ml_1m") if name == "ml_1m" else _small(13, 400, 300, 9000)
    B, ARR, steps, ss, frac = 50, 0.001, 10, 3, 0.5
    g = RatingGraph(A, reserve_nnz=100)
    cv = np.arange(1, R + 1, dtype=np.float32)
    m, m2 = (support.model(R, rgcn=rgcn, dgcnn=kind == "dgcnn", adj_dropout=0.2) for _ in range(2))
    opt, opt2 = FusedAdam(m, lr=1e-3), FusedAdam(m2, lr=1e-3)
    tr = OnlineTrainer(m, g, opt, batch_size=B, ARR=ARR, max_nodes_per_hop=mnph, recent_fraction=frac,
                       recent_capacity=256, sample_seed=ss, use_graph=use_graph)
    rng = np.random.default_rng(5)
    coo = A.tocoo()
    e = rng.integers(0, coo.nnz, 300)
    x = rng.integers(1, R + 1, 300)
    tr.update(coo.row[e], coo.col[e], x)
    window = recent_append_host(np.zeros(256, np.int32), np.zeros(256, np.int32), 0, coo.row[e], coo.col[e], x)
    loss = tr.train(steps)
    torch.cuda.synchronize()
    want_loss = _manual_steps(m2, opt2, g, mnph, B, ARR, steps, ss, window, frac, cv)
    for a, b in zip(_state(m, opt), _state(m2, opt2)):
        assert torch.equal(a, b), case
    assert loss == want_loss and np.isfinite(loss)
    assert int(opt.step_count[0]) == steps
    assert (len(tr.graphs) > 0) == use_graph
    tr.close()


# ---- 3. following updates ---------------------------------------------------------------------------------------------
def _copy(m, opt, kind="igmc", R=5):
    m2 = support.model(R, dgcnn=kind == "dgcnn", adj_dropout=0.2)
    m2.load_state_dict(m.state_dict())
    o2 = FusedAdam(m2, lr=opt.param_groups[0]["lr"])
    o2.load_state_dict(opt.state_dict())
    return m2, o2


@functools.lru_cache(maxsize=None)
def _uniform(nu=300, ni=200, nnz=3000, seed=6):
    """ratings at uniform random pairs: degrees stay small (subgraphs of up to 256 nodes without a node cap)"""
    rng = np.random.default_rng(seed)
    key = rng.choice(nu * ni, nnz, replace=False)
    return build_adj(key // ni, key % ni, rng.integers(0, 5, nnz), nu, ni)


def test_trainer_follows_a_chain_of_updates():
    A = _uniform()
    R, B, cap = 5, 50, 512
    g = RatingGraph(A, reserve_nnz=3000, reserve_users=10, reserve_items=10)
    m = support.model(R, adj_dropout=0.2)
    opt = FusedAdam(m, lr=1e-3)
    kw = dict(batch_size=B, ARR=0.001, max_nodes_per_hop=None, recent_fraction=0.4, recent_capacity=cap, sample_seed=9)
    tr = OnlineTrainer(m, g, opt, **kw)
    tr.train(10)
    rng = np.random.default_rng(8)
    caps = [tr.dataset.extractor.cap]
    for rnd in range(5):
        nu, ni = g.shape
        coo = A.tocoo()
        e = rng.integers(0, coo.nnz, 120)
        kind = rng.integers(0, 3, 120)          # 0 change, 1 delete, 2 insert at a random pair
        u = np.where(kind < 2, coo.row[e], rng.integers(0, nu, 120))
        v = np.where(kind < 2, coo.col[e], rng.integers(0, ni, 120))
        x = np.where(kind == 1, 0, rng.integers(1, R + 1, 120))
        if rnd in (1, 3):    # a new user whose row is longer than any, and a new item
            long = max(g.max_row_deg, g.max_col_deg) + 5 + rnd
            u = np.concatenate([u, np.full(long, nu), [0]])
            v = np.concatenate([v, rng.choice(ni, long, replace=False), [ni]])
            x = np.concatenate([x, rng.integers(1, R + 1, long + 1)])
        before = (_state(m, opt), [t.clone() for t in (tr.recent_u, tr.recent_v, tr.recent_total)])
        mf, of = _copy(m, opt)
        tr.update(u, v, x)
        A = _apply_scipy(A, u, v, x, g.shape)
        loss = tr.train(10)
        # a fresh trainer on the updated graph, from the same model / optimizer state and window
        gf = RatingGraph(A, reserve_nnz=100)
        fresh = OnlineTrainer(mf, gf, of, **kw)
        fresh.recent_u.copy_(tr.recent_u), fresh.recent_v.copy_(tr.recent_v)
        fresh.recent_total.copy_(tr.recent_total)
        loss_f = fresh.train(10)
        for a, b in zip(_state(m, opt), _state(mf, of)):
            assert torch.equal(a, b), rnd
        assert loss == loss_f
        fresh.close()
        assert not torch.equal(before[0][0], _state(m, opt)[0])
        caps.append(tr.dataset.extractor.cap)
    assert max(caps) > caps[0] and tr.dataset.extractor.__dict__.get("_retired_ws")   # cap grew: re-reserved
    tr.close()


def test_train_calls_continue_the_pipeline():
    """train(3) + train(7) gives the bits of train(10): the batch drawn beside the last step of a call is the first of
    the next.  The drawn batch's list images are rebuilt at each call, so a TrainEngine training the same model in
    between (its staged images share the model's cache) leaves the next call training on its own batch."""
    from igmc_b200.train_eval import TrainEngine
    from igmc_b200.util_functions import MyDynamicDataset
    ds = support.dataset("ml_1m")
    A = ds["adj_train"]
    tu, tv, tl = ds["train"]
    out = []
    for split in (True, False):
        m = support.model(5, adj_dropout=0.2)
        opt = FusedAdam(m, lr=1e-3)
        tr = OnlineTrainer(m, RatingGraph(A), opt, batch_size=50, max_nodes_per_hop=100)
        losses = [tr.train(3), tr.train(7)] if split else [tr.train(10)]
        out.append(_state(m, opt))
        if split:        # another engine on this model between two calls, then the trainer again
            d = MyDynamicDataset(None, tr.graph, (tu[:400], tv[:400]), tl[:400], 1, 1.0, 100, None, None,
                                 ds["class_values"])
            eng = TrainEngine(d, m, opt, 50, ARR=0.001)
            eng.prime(np.arange(50), 1)
            for s in range(7):
                eng.step_pipe(np.arange((s + 1) * 50, (s + 2) * 50) if s < 6 else None, 1)
            eng.close()
            losses.append(tr.train(5))
            assert int(opt.step_count[0]) == 22 and all(np.isfinite(losses))
            assert torch.isfinite(m.flat_params).all()
        tr.close()
    for a, b in zip(*out):
        assert torch.equal(a, b)


# ---- 4. serving --------------------------------------------------------------------------------------------------------
def test_engine_built_before_fine_tuning_serves_the_new_weights():
    A = support.adj("ml_1m")
    g = RatingGraph(A, reserve_nnz=1000)
    m = support.model(5, adj_dropout=0.2)
    opt = FusedAdam(m, lr=1e-3)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=50, sample_seed=2)
    users = np.array([0, 5, 77])
    before = eng.recommend(users, 10)
    tr = OnlineTrainer(m, g, opt, batch_size=50, max_nodes_per_hop=100)
    tr.update([1, 2], [3, 4], [5, 1])
    tr.train(20)
    got = eng.recommend(users, 10)
    fresh = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=50, sample_seed=2)
    want = fresh.recommend(users, 10)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert not torch.equal(before[1], got[1])
    # the model's own eval forward sees the new weights too (prepared weights consistent)
    pu, pv = np.arange(60) % g.num_users, np.arange(60) * 7 % g.num_items
    s1 = rc.predict_pairs(m, g, pu, pv, max_nodes_per_hop=100, batch_size=50, sample_seed=2)
    assert torch.equal(s1, fresh.predict_pairs(pu, pv))
    fresh.close(), eng.close(), tr.close()


# ---- 5. it learns --------------------------------------------------------------------------------------------------------
def _rmse(m, g, u, v, lab):
    s = rc.predict_pairs(m, g, u, v, max_nodes_per_hop=100).cpu().numpy().astype(np.float64)
    return float(np.sqrt(np.mean((s - (lab + 1)) ** 2)))


def test_fine_tuning_on_new_ratings_lowers_their_error():
    from igmc_b200.util_functions import MyDynamicDataset
    ds = support.dataset("ml_1m")
    A = ds["adj_train"].tocoo()
    rng = np.random.default_rng(0)
    users = rng.choice(ds["num_users"], 200, replace=False)
    held = np.flatnonzero(np.isin(A.row, users))
    held = rng.choice(held, 2000, replace=False)
    keep = np.ones(A.nnz, bool)
    keep[held] = False
    hu, hv, hl = A.row[held], A.col[held], (A.data[held] - 1).astype(np.int64)
    base = ssp.csr_matrix((A.data[keep], (A.row[keep], A.col[keep])), shape=A.shape)
    g = RatingGraph(base, reserve_nnz=2000)
    tu, tv = A.row[keep], A.col[keep]
    tl = (A.data[keep] - 1).astype(np.int64)
    sub = rng.choice(len(tu), 40000, replace=False)
    d = MyDynamicDataset(None, g, (tu[sub], tv[sub]), tl[sub], 1, 1.0, 100, None, None, ds["class_values"])
    torch.manual_seed(0)
    m = IGMC(d, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    te.train_multiple_epochs(d, d, m, 3, 50, 1e-3, 0.1, 50, 0, ARR=0.001, test_freq=100)
    cu, cv_, cl = ds["test"]
    other = (cu[:1000], cv_[:1000], cl[:1000])
    rmse_h0, rmse_o0 = _rmse(m, g, hu, hv, hl), _rmse(m, g, *other)
    opt = FusedAdam(m, lr=1e-4)
    tr = OnlineTrainer(m, g, opt, batch_size=50, max_nodes_per_hop=100, recent_fraction=0.5)
    tr.update(hu, hv, hl + 1)
    tr.train(200)
    rmse_h1, rmse_o1 = _rmse(m, g, hu, hv, hl), _rmse(m, g, *other)
    assert rmse_h1 < rmse_h0, (rmse_h0, rmse_h1)
    assert rmse_o1 <= 1.05 * rmse_o0, (rmse_o0, rmse_o1)
    tr.close()


# ---- 6. argument checks ------------------------------------------------------------------------------------------------
def test_argument_checks(monkeypatch):
    A = support.adj("tiny")
    g = RatingGraph(A, reserve_nnz=10)
    m = support.model(5, adj_dropout=0.2)
    opt = FusedAdam(m)
    bad = [dict(recent_fraction=-0.1), dict(recent_fraction=1.5), dict(batch_size=0), dict(h=2),
           dict(recent_capacity=0)]
    for kw in bad:
        with pytest.raises(ValueError):
            OnlineTrainer(m, g, opt, max_nodes_per_hop=10, **kw)
    with pytest.raises(ValueError, match="no ratings"):
        OnlineTrainer(m, RatingGraph(ssp.csr_matrix((5, 4), dtype=np.float32)), opt)
    monkeypatch.setattr(te, "_dist_info", lambda: (0, 2))
    with pytest.raises(NotImplementedError):
        OnlineTrainer(m, g, opt)
    monkeypatch.undo()
    tr = OnlineTrainer(m, g, opt, batch_size=8, max_nodes_per_hop=10)
    with pytest.raises(ValueError):
        tr.train(0)
    with pytest.raises(IndexError):
        tr.update([10 ** 6], [0], [3])
    with pytest.raises(ValueError):
        tr.update([0], [0], [300])
    assert int(tr.recent_total) == 0 and g.version == 0 and int(opt.step_count[0]) == 0
    coo = A.tocoo()
    tr.update(coo.row, coo.col, np.zeros(coo.nnz, np.int64))        # every rating deleted
    with pytest.raises(ValueError, match="no ratings"):
        tr.train(5)
    assert int(opt.step_count[0]) == 0
    tr.close()
