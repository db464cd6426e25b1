"""RecommendationCache on the GPU (igmc_b200/recommend.py, csrc/recommend_cache.cu):

* igmc_rescore_plan, igmc_cache_invalidate and igmc_cache_settle byte for byte against their host twins
  (tests/test_recommend_cache_host.py), the chunked bitmap regime, an empty and a duplicated edit list and guard
  entries included;
* a chain of updates - one rating, 10 and 100 ratings, deletes that empty a row, a cached user's own row, new users
  on cached users' items, a batch that forces the depth fallback, a degree increase and the growth of the item count
  - after each of which lists() equals a fresh recommend on the updated graph bit for bit and rescored_pairs the
  twin's count; on plans 2 / 4 / 0 (R = 13) / L2, rgcn="pyg-2", DGCNN_RS, three checkpoints, a shared list with and
  without exclusion, B = 50 / 256 with graphs on and off, k = 1 / 10 with depth k and 50;
* a parameter change rebuilds in full, an outside graph.update raises, a steady-state update makes no more host
  synchronisations than documented."""
import ctypes as C
import os
import tempfile
import warnings

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.util_functions import RatingGraph, _stream_ptr
from tests import test_gpu_recommend as tr
from tests.test_recommend_cache_host import _slot_case

pytestmark = pytest.mark.gpu


def _dev(a, dt=torch.int32):
    return torch.as_tensor(np.asarray(a)).to(dt).cuda()


@pytest.mark.parametrize("bound", [0, 4000])
@pytest.mark.parametrize("shared,exclude", [(False, True), (True, True), (True, False)])
def test_rescore_plan_kernel_matches_twin(bound, shared, exclude):
    lib = _lib.load()
    rng = np.random.default_rng(3)
    A = tr._r13()["adj_train"]
    g = RatingGraph(A)
    h = g.host
    U, ni = 70, g.num_items
    users = rng.integers(g.num_users, size=U)
    users[5] = users[6]                                                     # a user in two slots
    cand = np.unique(rng.integers(ni, size=90)) if shared else None
    nbytes, chunk = C.c_int64(0), C.c_int(0)
    assert lib.igmc_rescore_plan_ws_bytes(U, ni, bound, C.byref(nbytes), C.byref(chunk)) == 0
    assert (chunk.value < U) == (bound > 0)                                 # the chunked regime
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")
    for eu, ev in (([], []), ([users[0]], [3]), (rng.integers(g.num_users, size=30), rng.integers(ni, size=30)),
                   ([7, 7, 7], [11, 11, 11])):                              # empty, own row, random, duplicated
        eu, ev = np.asarray(eu, np.int64), np.asarray(ev, np.int64)
        want_off, want_items, want_full, want_total = rc.rescore_plan_host(h["row_ptr"], h["col_idx"], ni, users,
                                                                           eu, ev, cand, exclude)
        cap = len(want_items) + 8
        out = torch.full((cap,), -7, dtype=torch.int32, device="cuda")      # guard entries past the plan
        user_off = torch.full((U + 2,), -7, dtype=torch.int64, device="cuda")
        full = torch.full((U + 1,), 9, dtype=torch.uint8, device="cuda")
        totals, err = torch.zeros(2, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32,
                                                                                     device="cuda")
        cd = None if cand is None else _dev(cand)
        assert lib.igmc_rescore_plan(C.byref(g._c), _dev(users).data_ptr(), U, _dev(eu if len(eu) else [0]).data_ptr(),
                                     _dev(ev if len(ev) else [0]).data_ptr(), len(eu), _lib.ptr(cd),
                                     0 if cand is None else len(cand), int(exclude), ws.data_ptr(), ws.numel(),
                                     user_off.data_ptr(), out.data_ptr(), cap, full.data_ptr(), totals.data_ptr(),
                                     err.data_ptr(), _stream_ptr()) == 0
        assert int(err.item()) == 0
        assert np.array_equal(user_off[:U + 1].cpu().numpy(), want_off) and int(user_off[U + 1]) == -7
        assert np.array_equal(out[:len(want_items)].cpu().numpy(), want_items)
        assert (out[len(want_items):] == -7).all()
        assert np.array_equal(full[:U].cpu().numpy(), want_full) and int(full[U]) == 9
        assert totals.tolist() == [int(want_off[-1]), want_total]


@pytest.mark.parametrize("D,k", [(1, 1), (6, 3), (10, 10), (50, 10)])
def test_invalidate_and_settle_kernels_match_twins(D, k):
    lib = _lib.load()
    rng = np.random.default_rng(D + k)
    U, ni = 300, 60
    cases = [_slot_case(rng, ni, D, k) for _ in range(U)]
    top_s, top_i = np.stack([c[2] for c in cases]), np.stack([c[3] for c in cases])
    complete = np.array([c[4] for c in cases], np.uint8)
    full = np.array([len(c[5]) == len(c[0]) for c in cases], np.uint8)
    user_off = np.concatenate([[0], np.cumsum([len(c[5]) for c in cases])]).astype(np.int64)
    resc = np.concatenate([c[5] for c in cases] + [np.zeros(1)]).astype(np.int32)
    ws_, wi, wts, wti = rc.cache_invalidate_host(user_off, resc, full, complete, top_s, top_i)
    ds, di = _dev(np.r_[top_s.reshape(-1), 5.0], torch.float32), _dev(np.r_[top_i.reshape(-1), 77], torch.int64)
    ts, ti = torch.full((U + 1,), 3.0, device="cuda"), torch.full((U + 1,), 77, dtype=torch.int64, device="cuda")
    dcomp = _dev(np.r_[complete, 9], torch.uint8)
    assert lib.igmc_cache_invalidate(U, D, _dev(user_off, torch.int64).data_ptr(), _dev(resc).data_ptr(),
                                     _dev(full, torch.uint8).data_ptr(), dcomp.data_ptr(), ds.data_ptr(),
                                     di.data_ptr(), ts.data_ptr(), ti.data_ptr(), _stream_ptr()) == 0
    assert np.array_equal(ds[:-1].cpu().numpy().view(np.uint32), ws_.reshape(-1).view(np.uint32))
    assert np.array_equal(di[:-1].cpu().numpy(), wi.reshape(-1)) and float(ds[-1]) == 5.0 and int(di[-1]) == 77
    assert np.array_equal(ts[:U].cpu().numpy().view(np.uint32), wts.view(np.uint32)) and float(ts[U]) == 3.0
    assert np.array_equal(ti[:U].cpu().numpy(), wti) and int(ti[U]) == 77
    # the merge, then settle on the merged lists
    for j, c in enumerate(cases):
        ws_[j], wi[j] = rc.topk_merge_host(ws_[j], wi[j], c[1][c[5]], c[5])
    gs, gi, gcomp, gredo = rc.cache_settle_host(wts, wti, ws_, wi, k)
    ds, di = _dev(np.r_[ws_.reshape(-1), 5.0], torch.float32), _dev(np.r_[wi.reshape(-1), 77], torch.int64)
    redo, cnt = torch.full((U + 1,), -7, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32,
                                                                                        device="cuda")
    assert lib.igmc_cache_settle(U, D, k, _dev(wts, torch.float32).data_ptr(), _dev(wti, torch.int64).data_ptr(),
                                 ds.data_ptr(), di.data_ptr(), dcomp.data_ptr(), redo.data_ptr(), cnt.data_ptr(),
                                 _stream_ptr()) == 0
    assert np.array_equal(ds[:-1].cpu().numpy().view(np.uint32), gs.reshape(-1).view(np.uint32))
    assert np.array_equal(di[:-1].cpu().numpy(), gi.reshape(-1)) and int(di[-1]) == 77
    assert np.array_equal(dcomp[:U].cpu().numpy(), gcomp) and int(dcomp[U]) == 9
    n = int(cnt.item())
    assert n == len(gredo) and np.array_equal(redo[:n].cpu().numpy(), gredo) and (redo[n:] == -7).all()
    assert 0 < n < U                                                        # both outcomes occur


# ---- end to end -----------------------------------------------------------------------------------------------------
def _chain(g, users, rng, top_items):
    """the update batches of the chain, each (name, users, items, values) built on the graph as it stands"""
    def rand(n, lo=0):
        return rng.integers(g.num_users, size=n), rng.integers(g.num_items, size=n), rng.integers(lo, 6, size=n)

    def row(u):
        h = g.host
        return h["col_idx"][h["row_ptr"][u]:h["row_ptr"][u + 1]]
    yield ("one",) + rand(1, lo=1)
    yield ("ten",) + rand(10)
    yield ("hundred",) + rand(100)
    r = row(int(users[3]))
    yield "empty_row", np.full(len(r), int(users[3])), r, np.zeros(len(r), np.int64)
    yield "own_row", np.full(3, int(users[0])), rng.integers(g.num_items, size=3), np.array([2, 5, 1])
    new, its = g.num_users, [int(x) for x in row(int(users[1]))[:2]] or [0]
    yield "new_users", np.array([new, new + 1, new + 1][:len(its) + 1]), np.array((its * 2)[:len(its) + 1]), \
        np.array([4, 2, 5][:len(its) + 1])
    # every rater of the first slot's top items changes its rating: the lists lose entries below the threshold
    h, cu, cv = g.host, [], []
    for v in [x for x in top_items if x >= 0][:6]:
        raters = h["row_idx"][h["col_ptr"][v]:h["col_ptr"][v + 1]][:8]
        cu += list(raters)
        cv += [v] * len(raters)
    yield "fallback", np.array(cu, np.int64), np.array(cv, np.int64), rng.integers(1, 6, size=len(cu))
    # the longest row and the longest column both grow: with max_nodes_per_hop=None n_cap moves
    h = g.host
    top_u, top_v = int(np.argmax(np.diff(h["row_ptr"]))), int(np.argmax(np.diff(h["col_ptr"])))
    free_v = np.setdiff1d(np.arange(g.num_items), row(top_u))[:2]
    free_u = np.setdiff1d(np.arange(g.num_users), h["row_idx"][h["col_ptr"][top_v]:h["col_ptr"][top_v + 1]])[:2]
    yield "degree", np.r_[np.full(len(free_v), top_u), free_u], np.r_[free_v, np.full(len(free_u), top_v)], \
        np.full(len(free_v) + len(free_u), 3)
    yield "items", np.array([int(users[2])]), np.array([g.num_items]), np.array([4])


CONFIGS = {
    "plan2_b50_nograph_k1_d50": dict(plan=2, mnph=20, B=50, graphs=False, k=1, depth=50),
    "plan4_k10_d10": dict(plan=4, mnph=20, k=10, depth=10),
    "plan0_r13": dict(plan=0, r13=True, mnph=40, k=10, depth=50),
    "l2_uncapped_shared": dict(plan=_lib.plan_l2(1), mnph=None, k=10, depth=50, items="excl"),
    "auto_shared_noexcl": dict(mnph=20, k=10, depth=10, items="all"),
    "pyg2_k1_d1": dict(rgcn="pyg-2", mnph=20, k=1, depth=1),
    "dgcnn": dict(dgcnn=True, mnph=20, k=10, depth=10),
    "ckpt3": dict(ckpt=3, mnph=20, k=10, depth=50),
}


def _setup(cfg):
    if cfg.get("r13"):
        A, R = tr._r13()["adj_train"], 13
    else:
        d = tr._ds("ml_100k")
        A, R = d["adj_train"], 5
    m = tr._model(R, rgcn=cfg.get("rgcn", "pyg-1.4"), dgcnn=cfg.get("dgcnn", False))
    if "plan" in cfg:
        m.kernel_plan = cfg["plan"]
    g = RatingGraph(A, reserve_nnz=20000, reserve_users=8, reserve_items=4)
    rng = np.random.default_rng(11)
    users = np.unique(rng.integers(A.shape[0], size=40))
    items = None
    if cfg.get("items"):
        items = np.unique(rng.integers(A.shape[1], size=600))
    return m, g, users, items


def _run_chain(cfg, tmp):
    m, g, users, items = _setup(cfg)
    paths = None
    if cfg.get("ckpt"):
        paths = []
        for c in range(cfg["ckpt"]):
            torch.manual_seed(100 + c)
            m2 = tr._model(m.num_relations)
            paths.append(os.path.join(tmp, "ck%d.pth" % c))
            torch.save(m2.state_dict(), paths[-1])
    kw = dict(items=items, exclude_rated=cfg.get("items") != "all", max_nodes_per_hop=cfg["mnph"],
              batch_size=cfg.get("B", 256), checkpoints=paths)
    cache = rc.RecommendationCache(m, g, users, cfg["k"], depth=cfg["depth"], use_graph=cfg.get("graphs", True), **kw)
    rng = np.random.default_rng(5)
    seen = {}
    try:
        for name, eu, ev, ex in _chain(g, users, rng, cache._top_i[0].tolist()):
            shape, version = g.shape, g.version
            out = cache.update(eu, ev, ex)
            got_i, got_s = cache.lists()
            want_i, want_s = rc.recommend(m, g, users, cfg["k"], **kw)
            assert torch.equal(got_i, want_i), (name, out)
            assert torch.equal(got_s.view(torch.int32), want_s.view(torch.int32)), (name, out)
            seen[name] = out
            if not out["full"] and g.version != version:
                h = g.host
                off = rc.rescore_plan_host(h["row_ptr"], h["col_idx"], g.num_items, users, eu, ev, items,
                                           cfg.get("items") != "all")[0]
                assert out["rescored_pairs"] == int(off[-1]), name
    finally:
        cache.close()
    return seen


@pytest.mark.parametrize("name", list(CONFIGS))
def test_chain_matches_fresh_recommend(name):
    cfg = CONFIGS[name]
    with tempfile.TemporaryDirectory() as tmp:
        seen = _run_chain(cfg, tmp)
    assert seen["items"]["full"]                                           # the item count grew
    assert not seen["one"]["full"] and not seen["ten"]["full"]
    assert seen["empty_row"]["removed"] > 0
    if cfg["mnph"] is None:
        assert seen["degree"]["full"]                                      # n_cap moved
    if cfg["depth"] == cfg["k"]:
        assert sum(o["rebuilt_users"] for o in seen.values()) > 0          # the depth fallback ran


def test_parameter_change_outside_update_and_sync_count():
    m, g, users, items = _setup(dict(mnph=20))
    cache = rc.RecommendationCache(m, g, users, 10, depth=20, max_nodes_per_hop=20)
    try:
        rng = np.random.default_rng(2)
        eu, ev = rng.integers(g.num_users, size=3), rng.integers(g.num_items, size=3)
        cache.update(eu, ev, [1, 2, 3])                                    # warm: shapes and plans
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                out = cache.update(rng.integers(g.num_users, size=3), rng.integers(g.num_items, size=3), [2, 3, 4])
            finally:
                torch.cuda.set_sync_debug_mode("default")
        syncs = [x for x in w if "called a synchronizing" in str(x.message)]
        assert not out["full"] and out["rebuilt_users"] == 0 and out["rescored_pairs"] > 0
        assert len(syncs) <= 4, [str(x.message) for x in syncs]
        with torch.no_grad():
            m.flat_params.mul_(1.01)
        out = cache.update([int(users[0])], [0], [0])
        assert out["full"]
        want = rc.recommend(m, g, users, 10, max_nodes_per_hop=20)
        got = cache.lists()
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
        g.update([0], [1], [3])
        with pytest.raises(RuntimeError, match="refresh"):
            cache.lists()
        with pytest.raises(RuntimeError, match="refresh"):
            cache.update([0], [2], [3])
        cache.refresh()
        want = rc.recommend(m, g, users, 10, max_nodes_per_hop=20)
        assert torch.equal(cache.lists()[0], want[0])
    finally:
        cache.close()


def test_argument_checks():
    m, g, users, _ = _setup(dict(mnph=20))
    with pytest.raises(NotImplementedError):
        rc.RecommendationCache(m, g, users, 10, h=2)
    with pytest.raises(NotImplementedError):
        rc.RecommendationCache(m, g, users, 10, draws=4)
    with pytest.raises(NotImplementedError):
        rc.RecommendationCache(m, g, users, 10, retrieve=20)
    with pytest.raises(ValueError):
        rc.RecommendationCache(m, g, users, 10, depth=5)
    with pytest.raises(ValueError):
        rc.RecommendationCache(m, g, users, 0)
    with pytest.raises(NotImplementedError):
        rc.RecommendationCache(m, g, users, 300)
