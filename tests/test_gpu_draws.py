"""Monte-Carlo-dropout draws on the GPU (igmc_b200/recommend.py predict_draws and draws= rankings, csrc/draws.cu).

* the expand, mask and stats kernels, called directly, match their numpy twins byte for byte, with guard entries;
* every draw is bit for bit the training-mode forward of the model alone on that pair's subgraph with the twin's masks,
  on plans 2, 4, 0 and L2, pyg-2, DGCNN_RS, NB 2 and 4 and h = 2, and within 1e-4 of the fp64 restated model;
* draws do not depend on the batch size, graph replay, the run or the other pairs; checkpoints average per draw;
* recommend / recommend_users / recommend_sessions with draws= rank by the keys of predict_draws; draws=None is the
  eval ranking;
* an engine kept across graph.update matches a fresh one; steady-state steps make no host synchronisation."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import scipy.sparse as ssp
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.util_functions import RatingGraph, SubgraphExtractor
from oracle import pyg_restated
from tests import pyg2_oracle
from tests import support
from tests.test_gpu_graph_update import _apply_scipy

pytestmark = pytest.mark.gpu


def _with_cold_start(A):
    """A with one more user and one more item, neither rated: the pair (new user, new item) has no ratings at all"""
    return ssp.csr_matrix(ssp.bmat([[A, None], [None, ssp.csr_matrix((1, 1), dtype=A.dtype)]]), dtype=A.dtype)


def _random_pairs(A, n, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, A.shape[0], n), rng.integers(0, A.shape[1], n)


# ---- 1. kernels against their twins ------------------------------------------------------------------------------------
SENT32, SENT8, SENTF = -77, 0xAB, -7.5
GUARD = 16


def _expand_and_extract(A, R, S, B, u, v, ptag, h=1, mnph=100, seed=3):
    """the expand kernel on G = B // S pairs (checked against its twin with guards), then the extraction of its B
    positions; returns (expanded host arrays, batch, extractor)"""
    lib = _lib.load()
    G = B // S
    ni = A.shape[1]
    pu, pv = support.dev(u[:G], torch.int32), support.dev(v[:G], torch.int32)
    ppid, pt = support.dev(u[:G].astype(np.int64) * ni + v[:G], torch.int64), support.dev(ptag[:G], torch.int64)
    out = [support.filled(B, SENT32, d) for d in (torch.int32, torch.int32, torch.int64, torch.int64, torch.int32)]
    _lib.check(lib.igmc_draws_expand(S, B, pu.data_ptr(), pv.data_ptr(), ppid.data_ptr(), pt.data_ptr(),
                                     *(t.data_ptr() for t in out), None), "igmc_draws_expand")
    want = rc.draws_expand_host(S, B, u[:G], v[:G], u[:G].astype(np.int64) * ni + v[:G], ptag[:G])
    got = [t.cpu().numpy() for t in out]
    for w, g in zip(want, got):
        assert np.array_equal(g[:B], w) and (g[B:] == SENT32).all(), (S, B)
    ex = SubgraphExtractor(RatingGraph(A), [0], [0], [0], np.arange(1, R + 1, dtype=np.float32), h, 1.0, mnph,
                           max_batch=B, seed=seed)
    b = ex.extract(pairs=(out[0][:B], out[1][:B], None), pair_ids=out[2][:B])
    return want, b, ex


@pytest.mark.parametrize("case", ["B=1", "B=50 S=8 tail", "B=256 S=8", "B=256 S=3 tail pairs", "cold start",
                                  "h=2"])
def test_kernels_match_twins(case):
    lib = _lib.load()
    A = _with_cold_start(support.adj("ml_1m"))
    R, h = 5, 1
    nu, ni = A.shape[0] - 1, A.shape[1] - 1
    u, v = _random_pairs(support.adj("ml_1m"), 256, seed=len(case))
    ptag = np.arange(256, dtype=np.int64)
    S, B = dict(zip(["B=1", "B=50 S=8 tail", "B=256 S=8", "B=256 S=3 tail pairs", "cold start", "h=2"],
                    [(1, 1), (8, 50), (8, 256), (3, 256), (4, 32), (2, 20)]))[case]
    if case == "B=256 S=3 tail pairs":
        ptag[80:] = -1                                # the pair stream's tail: pairs past the run's end
    if case == "cold start":
        u[:3], v[:3] = nu, ni                         # a subgraph without ratings
    if case == "h=2":
        h = 2
    (lu, lv, pid, tag, draw), b, ex = _expand_and_extract(A, R, S, B, u, v, ptag, h=h, mnph=20 if h == 2 else 100)
    O = b._lazy["_c"]
    edge_ptr = b._priv["edge_ptr"].cpu().numpy()
    E = int(edge_ptr[-1])
    if case == "cold start":
        assert edge_ptr[1] == edge_ptr[0]
    dpid, dtag, ddraw = support.dev(pid, torch.int64), support.dev(tag, torch.int64), support.dev(draw, torch.int32)
    for p, seed in ((0.2, 0), (0.0, 2 ** 64 - 1), (0.5, 12345)):
        ek, hk = support.filled(E, SENT8, torch.uint8), support.filled(B * 128, SENT8, torch.uint8)
        _lib.check(lib.igmc_draws_mask(C.byref(O), B, dpid.data_ptr(), dtag.data_ptr(), ddraw.data_ptr(), p, seed,
                                       ek.data_ptr(), hk.data_ptr(), None), "igmc_draws_mask")
        wek, whk = rc.draws_mask_host(edge_ptr, pid, tag, draw, p, seed)
        gek, ghk = ek.cpu().numpy(), hk.cpu().numpy()
        assert np.array_equal(gek[:E], wek) and (gek[E:] == SENT8).all(), (case, p)
        assert np.array_equal(ghk[:B * 128], whk) and (ghk[B * 128:] == SENT8).all(), (case, p)
    b.check()
    assert int(ex.err.item()) == 0
    # stats: K = 1 and 3 checkpoints, a NaN and an infinite draw among them
    rng = np.random.default_rng(1)
    G = B // S
    P = int(tag.max()) + 1 if (tag >= 0).any() else 0
    for K in (1, 3):
        preds = rng.normal(3.0, 1.0, size=(K, B)).astype(np.float32)
        if B > 8:
            preds[0, 5], preds[K - 1, S + 1] = np.nan, np.inf
        dp = support.dev(preds.reshape(-1), torch.float32)
        for beta in (0.0, 1.0, -2.5):
            key = support.filled(G, SENTF, torch.float32)
            _lib.check(lib.igmc_draws_stats(dp.data_ptr(), K, B, S, dtag.data_ptr(), beta, None, None, None,
                                            key.data_ptr(), None), "igmc_draws_stats")
            x, mean, sd, wkey = rc.draws_stats_host(preds, K, B, S, beta)
            gk = key.cpu().numpy()
            assert support.same(gk[:G], wkey), (case, K, beta)
            assert (gk[G:] == SENTF).all()
        value, mo, so = support.filled(P * S, SENTF, torch.float32), support.filled(P, SENTF, torch.float32), \
            support.filled(P, SENTF, torch.float32)
        _lib.check(lib.igmc_draws_stats(dp.data_ptr(), K, B, S, dtag.data_ptr(), 0.0, value.data_ptr(), mo.data_ptr(),
                                        so.data_ptr(), None, None), "igmc_draws_stats")
        wv = np.full(P * S + GUARD, SENTF, np.float32)
        wm, ws = np.full(P + GUARD, SENTF, np.float32), np.full(P + GUARD, SENTF, np.float32)
        for g in range(G):
            t = int(tag[g * S])
            if t >= 0:
                wv[t * S:(t + 1) * S], wm[t], ws[t] = x[g], mean[g], sd[g]
        for got, want in ((value, wv), (mo, wm), (so, ws)):
            assert support.same(got.cpu().numpy(), want), (case, K)
    # argument checks of the entry points
    assert lib.igmc_draws_expand(0, B, *([None] * 9), None) != 0
    assert lib.igmc_draws_expand(_lib.DRAWS_MAX + 1, 4096, *([None] * 9), None) != 0
    assert lib.igmc_draws_stats(dp.data_ptr(), 1, B, S, dtag.data_ptr(), float("nan"), None, None, None,
                                key.data_ptr(), None) == -2
    assert lib.igmc_draws_mask(C.byref(O), B, dpid.data_ptr(), dtag.data_ptr(), ddraw.data_ptr(), 1.5, 0,
                               ek.data_ptr(), hk.data_ptr(), None) == -2


# ---- 2. each draw is the model alone on its pair --------------------------------------------------------------------------
CASES = {
    # name: (dataset, h, mnph, model kwargs, forced kernel plan, expected plan)
    "plan 2 ml_1m": ("ml_1m", 1, 100, {}, "auto", 2),
    "plan 4 ml_100k": ("ml_100k", 1, 200, {}, "auto", 4),
    "plan 0 R=13": ("r13", 1, 50, {}, "auto", 0),
    "L2 plan ml_100k uncapped": ("ml_100k", 1, None, {}, "auto", "l2"),
    "h=2": ("ml_1m", 2, 20, {}, "auto", None),
    "pyg-2": ("ml_1m", 1, 100, dict(rgcn="pyg-2"), "auto", 2),
    "DGCNN_RS": ("ml_1m", 1, 100, dict(dgcnn=True), "auto", None),
    "NB 2": ("ml_1m", 1, 100, dict(nb=2), "auto", 2),
    "NB 4 plan 4": ("ml_1m", 1, 100, dict(nb=4), 4, 4),
}


def _case_pairs(A, n=6, seed=0):
    """n pairs of A (with a cold-start pair last): a rated pair, low-degree pairs and random ones"""
    nu, ni = A.shape[0] - 1, A.shape[1] - 1
    du, di = np.diff(A.indptr)[:nu], np.diff(A.tocsc().indptr)[:ni]
    rng = np.random.default_rng(seed)
    coo = A.tocoo()
    k = int(rng.integers(0, coo.nnz))
    lu = np.argsort(np.where(du > 0, du, du.max() + 1), kind="stable")[:n]
    li = np.argsort(np.where(di > 0, di, di.max() + 1), kind="stable")[:n]
    u = np.r_[[coo.row[k]], lu[:n - 2], [nu]]
    v = np.r_[[coo.col[k]], li[:n - 2], [ni]]
    return u.astype(np.int64), v.astype(np.int64)


def _alone(m, A, R, u, v, S, draw_seed, h, mnph, seed, plan):
    """[S] the training-mode forward of the model alone on a batch of the S draws of pair (u, v), masks from the twin,
    on kernel plan ``plan``; and the batch's (x, edge_index, edge_type) and masks for the oracle"""
    ni = A.shape[1]
    ex = SubgraphExtractor(RatingGraph(A), [0], [0], [0], np.arange(1, R + 1, dtype=np.float32), h, 1.0, mnph,
                           max_batch=S, seed=seed)
    pid = np.full(S, u * ni + v, np.int64)
    b = ex.extract(pairs=(np.full(S, u), np.full(S, v), np.zeros(S, np.int64)), pair_ids=pid)
    ek, hk = rc.draws_mask_host(b._priv["edge_ptr"].cpu().numpy(), pid, np.zeros(S, np.int64),
                                np.arange(S, dtype=np.int32), m.adj_dropout, draw_seed)
    own = m.kernel_plan
    m.kernel_plan = plan
    m.train()
    try:
        with torch.no_grad():
            out = m(b, edge_keep=torch.from_numpy(ek).cuda(), hidden_keep=torch.from_numpy(hk).cuda()).clone()
    finally:
        m.kernel_plan = own
        m.eval()
    b.check()
    return out, b, ek, hk


@pytest.mark.parametrize("name", list(CASES))
def test_each_draw_is_the_model_alone(name):
    dsn, h, mnph, kw, force, plan = CASES[name]
    A = _with_cold_start(support.adj(dsn))
    R = 13 if dsn == "r13" else 5
    m = support.model(R, h=h, **kw)
    m.kernel_plan = force
    u, v = _case_pairs(A)
    S, B, seed, ds = 8, 64, 7, 0x5EED
    d = rc.predict_draws(m, A, u, v, S, draw_seed=ds, h=h, max_nodes_per_hop=mnph, batch_size=B, sample_seed=seed)
    cl = next(iter(m._plans.values()))
    if plan == "l2":
        assert _lib.l2_csize(cl) > 0
    elif plan is not None:
        assert cl == plan, (name, cl)
    assert d.value.shape == (len(u), S)
    for p in range(len(u)):
        want = _alone(m, A, R, int(u[p]), int(v[p]), S, ds, h, mnph, seed, cl)[0]
        assert torch.equal(d.value[p], want), (name, p, (d.value[p] - want).abs().max().item())
    # the draws differ from one another (dropout acts) except on the cold-start pair's edges
    assert (d.std[:-1] > 0).all(), name


@pytest.mark.parametrize("rgcn", ["pyg-1.4", "pyg-2"])
def test_draws_against_the_fp64_oracle(rgcn):
    A = _with_cold_start(support.adj("ml_1m"))
    R, mnph, seed, S, ds = 5, 100, 7, 4, 11
    m = support.model(R, rgcn=rgcn)
    ref = pyg2_oracle.igmc_ref(rgcn, 4, (32,) * 4, R, 4, m.adj_dropout)
    ref.load_state_dict({k: v.double().cpu() for k, v in m.state_dict().items()})
    ref = pyg_restated.set_formulation(ref.double(), "transform").cuda().train()
    u, v = _case_pairs(A, 4)
    d = rc.predict_draws(m, A, u[:3], v[:3], S, draw_seed=ds, max_nodes_per_hop=mnph, batch_size=64, sample_seed=seed)
    errs = []
    for p in range(3):
        _, b, ek, hk = _alone(m, A, R, int(u[p]), int(v[p]), S, ds, 1, mnph, seed, "auto")
        with torch.no_grad():
            want = ref(b.x.double(), b.edge_index, b.edge_type, torch.from_numpy(ek).bool().cuda(),
                       torch.from_numpy(hk).bool().cuda().view(S, 128))
        errs.append((d.value[p].double() - want).cpu().numpy())
    err = float(np.abs(np.concatenate(errs)).max())
    print("%s: draws vs fp64 oracle max |err| %.2e" % (rgcn, err))
    assert err <= 1e-4, err


# ---- 3. independence of the batch, the run and the other pairs -------------------------------------------------------------
def test_draws_do_not_depend_on_batch_run_or_neighbours():
    A = support.adj("ml_1m")
    m = support.model(5)
    m.kernel_plan = 2
    u, v = _random_pairs(A, 40, seed=3)
    S, kw = 8, dict(max_nodes_per_hop=100, sample_seed=1)
    first = None
    for B in (S, 50, 256):
        for use_graph in (True, False):
            eng = rc.InferenceEngine(m, A, batch_size=B, use_graph=use_graph, **kw)
            for _ in range(2):
                got = eng.predict_draws(u, v, S, draw_seed=9)
                first = first or got
                for f in got._fields:
                    assert torch.equal(getattr(got, f), getattr(first, f)), (B, use_graph, f)
            eng.close()
    # other pairs added around them, in another order
    u2, v2 = _random_pairs(A, 100, seed=4)
    uu, vv = np.r_[u2[:30], u[::-1], u2[30:]], np.r_[v2[:30], v[::-1], v2[30:]]
    d = rc.predict_draws(m, A, uu, vv, S, draw_seed=9, batch_size=256, **kw)
    for f in d._fields:
        assert torch.equal(getattr(d, f)[30:70], getattr(first, f).flip(0)), f
    # another seed gives other draws
    other = rc.predict_draws(m, A, u, v, S, draw_seed=10, batch_size=256, **kw)
    assert not torch.equal(other.value, first.value)


def test_checkpoints_average_each_draw():
    A = support.adj("ml_100k")
    m = support.model(5)
    m.kernel_plan = 2
    u, v = _random_pairs(A, 30, seed=5)
    kw = dict(max_nodes_per_hop=100, batch_size=64, draw_seed=3)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for c in range(3):
            paths.append(os.path.join(tmp, "c%d.pth" % c))
            torch.save(support.model(5, seed=c + 1).state_dict(), paths[-1])
        got = rc.predict_draws(m, A, u, v, 4, checkpoints=paths, **kw)
        each = [rc.predict_draws(m, A, u, v, 4, checkpoints=[p], **kw).value for p in paths]
    e = [x.cpu().numpy() for x in each]
    # on the host: torch divides a CUDA tensor by a scalar as a multiplication by its reciprocal
    want = (((e[0] + e[1]).astype(np.float32) + e[2]).astype(np.float32) / np.float32(3)).astype(np.float32)
    assert np.array_equal(got.value.cpu().numpy(), want)


# ---- 4. rankings ---------------------------------------------------------------------------------------------------------
def _stable_rank(keys, cands, k):
    """key descending, candidate ascending, NaN last; padded with (-1, -inf)"""
    return rc.rank_host(keys, cands, k)


def _check_ranking(top_i, top_s, rows, keys_of, k):
    top_i, top_s = top_i.cpu().numpy(), top_s.cpu().numpy()
    for j, cands in enumerate(rows):
        ws, wi = _stable_rank(keys_of(j, cands), cands, k)
        assert np.array_equal(top_i[j], wi), (j, top_i[j][:5], wi[:5])
        assert support.same(top_s[j], ws), j


def _keys(m, A, users, items, S, beta, kw):
    """predict_draws' key mean + beta * std of every pair, from its draws by the statistics' twin"""
    d = rc.predict_draws(m, A, users, items, S, **kw)
    x = d.value.cpu().numpy()
    return np.array([rc.draws_stats_host(x[p], 1, S, S, beta)[3][0] for p in range(len(users))], np.float32)


@pytest.mark.parametrize("S", [1, 8])
def test_recommend_ranks_by_the_keys_of_predict_draws(S):
    A = support.adj("ml_100k")
    m = support.model(5)
    m.kernel_plan = 2
    ni = A.shape[1]
    users = np.array([3, 17, 250])
    kw = dict(max_nodes_per_hop=100, batch_size=256, draw_seed=21, sample_seed=2)
    rated = [set(A.indices[A.indptr[x]:A.indptr[x + 1]].tolist()) for x in users]
    for beta in (0.0, 1.0, -1.0):
        for k in (1, 10, 256):
            for mode in ("catalogue", "list", "rows", "retrieve"):
                if mode == "catalogue":
                    if k != 10:
                        continue
                    rows = [np.array([i for i in range(ni) if i not in r]) for r in rated]
                    top_i, top_s = rc.recommend(m, A, users, k, draws=S, beta=beta, **kw)
                elif mode == "list":
                    lst = np.arange(0, ni, 3)
                    rows = [np.array([i for i in lst if i not in r]) for r in rated]
                    top_i, top_s = rc.recommend(m, A, users, k, items=lst, draws=S, beta=beta, **kw)
                elif mode == "rows":
                    rr = np.random.default_rng(k).integers(-1, ni, size=(3, 40))
                    rows = [np.array(sorted(set(x for x in r if x >= 0) - rt)) for r, rt in zip(rr, rated)]
                    top_i, top_s = rc.recommend(m, A, users, k, items=rr, draws=S, beta=beta, **kw)
                else:
                    ret = rc.corated_items(RatingGraph(A), users, 100)[0].cpu().numpy()
                    rows = [np.array(sorted(x for x in r if x >= 0)) for r in ret]
                    top_i, top_s = rc.recommend(m, A, users, k, retrieve=100, draws=S, beta=beta, **kw)
                allu = np.concatenate([np.full(len(r), x) for x, r in zip(users, rows)])
                alli = np.concatenate(rows)
                keys = _keys(m, A, allu, alli, S, beta, kw)
                off = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
                _check_ranking(top_i, top_s, rows, lambda j, c: keys[off[j]:off[j + 1]], k)


def test_recommend_users_ranks_by_the_keys_of_predict_draws():
    A = support.adj("ml_100k")
    m = support.model(5)
    m.kernel_plan = 2
    items = np.array([5, 99])
    kw = dict(max_nodes_per_hop=100, batch_size=128, draw_seed=4)
    cols = A.tocsc()
    for S, beta in ((8, 1.0), (1, 0.0)):
        for k in (1, 10):
            top_i, top_s = rc.recommend_users(m, A, items, k, users=np.arange(0, A.shape[0], 2), draws=S, beta=beta,
                                              **kw)
            rows = [np.array([x for x in range(0, A.shape[0], 2)
                              if x not in set(cols.indices[cols.indptr[it]:cols.indptr[it + 1]].tolist())])
                    for it in items]
            allu = np.concatenate(rows)
            alli = np.concatenate([np.full(len(r), it) for it, r in zip(items, rows)])
            keys = _keys(m, A, allu, alli, S, beta, kw)
            off = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
            _check_ranking(top_i, top_s, rows, lambda j, c: keys[off[j]:off[j + 1]], k)


def test_recommend_sessions_equal_recommend_on_the_edited_graph():
    from tests.test_gpu_sessions import _A_s, _edits, _rows
    A = support.adj("ml_100k")
    m = support.model(5)
    m.kernel_plan = 2
    rng = np.random.default_rng(6)
    nu = A.shape[0]
    users = np.r_[rng.integers(0, nu, 3), [nu, nu + 1]]
    session, items, values = _edits(rng, A, users, 60)
    sess = rc.RatingSessions(RatingGraph(A), users, session, items, values)
    rows = _rows(A, users, session, items, values)
    kw = dict(max_nodes_per_hop=100, batch_size=128, draws=8, beta=0.5, draw_seed=7)
    got_i, got_s = rc.recommend_sessions(m, sess, 10, retrieve=50, **kw)
    lst = np.arange(0, A.shape[1], 4)
    got_li, got_ls = rc.recommend_sessions(m, sess, 10, items=lst, **kw)
    for s in range(len(users)):
        As = RatingGraph(_A_s(A, users[s], rows[s]))
        want_i, want_s = rc.recommend(m, As, [users[s]], 10, retrieve=50, **kw)
        assert torch.equal(got_i[s], want_i[0]) and torch.equal(got_s[s], want_s[0]), s
        want_i, want_s = rc.recommend(m, As, [users[s]], 10, items=lst, **kw)
        assert torch.equal(got_li[s], want_i[0]) and torch.equal(got_ls[s], want_s[0]), s


def test_draws_none_is_the_eval_ranking():
    A = support.adj("ml_100k")
    m = support.model(5)
    users = np.array([1, 2, 40])
    kw = dict(max_nodes_per_hop=100, batch_size=128)
    eng = rc.InferenceEngine(m, A, **kw)
    want = eng.recommend(users, 10, retrieve=80)
    wu = eng.recommend_users([3, 4], 5)
    eng.predict_draws(users, users, 4)                 # a run over draws in between
    got = eng.recommend(users, 10, retrieve=80, draws=None, beta=0.0, draw_seed=5)
    gu = eng.recommend_users([3, 4], 5, draws=None)
    eng.close()
    assert all(torch.equal(a, b) for a, b in zip(want, got))
    assert all(torch.equal(a, b) for a, b in zip(wu, gu))
    top_i, top_s = rc.recommend(m, A, users, 10, retrieve=80, **kw)
    assert torch.equal(top_i, want[0]) and torch.equal(top_s, want[1])
    # Thompson sampling at S = 1: the key is the one draw
    d = rc.predict_draws(m, A, [1], [5], 1, **kw)
    assert torch.equal(d.mean, d.value[:, 0]) and (d.std == 0).all()


# ---- 5. lifecycle ------------------------------------------------------------------------------------------------------
def test_engine_across_updates_and_sync_free_steps():
    A = support.adj("ml_100k")
    m = support.model(5)
    m.kernel_plan = 2
    g = RatingGraph(A, reserve_nnz=2000)
    kw = dict(max_nodes_per_hop=100, batch_size=64)
    eng = rc.InferenceEngine(m, g, **kw)
    u, v = _random_pairs(A, 60, seed=8)
    before = eng.predict_draws(u, v, 8, draw_seed=1)
    rng = np.random.default_rng(9)
    du = rng.integers(0, A.shape[0], 200)
    dv = rng.integers(0, A.shape[1], 200)
    dx = rng.integers(0, 6, 200)
    g.update(du, dv, dx)
    A2 = _apply_scipy(A, du, dv, dx, A.shape)
    kept = eng.predict_draws(u, v, 8, draw_seed=1)
    kept_r = eng.recommend(u[:5], 10, retrieve=60, draws=8, beta=1.0, draw_seed=1)
    fresh = rc.predict_draws(m, A2, u, v, 8, draw_seed=1, **kw)
    fresh_r = rc.recommend(m, A2, u[:5], 10, retrieve=60, draws=8, beta=1.0, draw_seed=1, **kw)
    for f in kept._fields:
        assert torch.equal(getattr(kept, f), getattr(fresh, f)), f
    assert torch.equal(kept_r[0], fresh_r[0]) and torch.equal(kept_r[1], fresh_r[1])
    assert not torch.equal(before.value, kept.value)
    # steady state: after the eager warm-up and the capture of both slots, no step synchronises with the host
    uu, vv = _random_pairs(A, 400, seed=10)
    for ranking in (False, True):
        outs = []
        for _ in range(2):
            if ranking:
                eng.start_recommend(uu[:40], 10, draws=4, beta=1.0)
            else:
                eng.start_draws(uu, vv, 8)
            for _ in range(4):
                assert eng.step()
            assert len(eng.graphs) == 2
            torch.cuda.set_sync_debug_mode("error")
            try:
                while eng.step():
                    pass
            finally:
                torch.cuda.set_sync_debug_mode("default")
            outs.append(eng.finish())
            assert int(eng.extractor.err.item()) == 0
        for a, b in zip(outs[0], outs[1]):
            assert torch.equal(a, b)
    eng.close()
