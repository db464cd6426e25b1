"""Every group, diversity and cached-list entry point called through _lib on every case of
tests/group_diverse_cache_cases.py: outputs pre-filled with sentinels and guard entries past them that must stay
untouched, floats compared bit for bit (NaN matching any NaN) with the brute-force enumerations of the header's
contracts, the error word read after every case and the return code of every argument check.  igmc_rescore_plan runs
each case at several chunk sizes, each giving the same plan.  recommend_groups, recommend_diverse and
RecommendationCache.update then run once each on a graph of 9 000 items and 1 100 cached slots against their host
compositions."""
import ctypes as C

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.data import build_adj, synth_ratings
from igmc_b200.util_functions import RatingGraph
from tests import group_diverse_cache_cases as gc
from tests import support
from tests.ranking_cases import same_f32

pytestmark = pytest.mark.gpu

S32, SF, S8 = -77, -7.5, 0xAB
GUARD = 16
CASES = gc.all_cases()


def _of(kernel):
    return [c for c in CASES if c["kernel"] == kernel]


_ALIVE = []   # every input a test uploads: a temporary passed as data_ptr() would return its memory to the allocator


@pytest.fixture(autouse=True)
def _release_inputs():
    yield
    torch.cuda.synchronize()
    _ALIVE.clear()


def _alive(a, dtype=torch.int32):
    """a host array on the device (an empty one as one zero), kept alive for the rest of the session"""
    t = support.dev(support.nonempty(a), dtype)
    _ALIVE.append(t)
    return t


def _err():
    return torch.zeros(1, dtype=torch.int32, device="cuda")


class _Graph:
    """a device CSR (with columns when asked) kept alive with its tensors"""
    def __init__(self, rp, ci, num_users, num_items, cols=False):
        self.keep = [_alive(rp), _alive(ci)]
        cp = None
        if cols:
            cp_h, ri = gc.columns(rp, ci, num_items)
            self.keep += [_alive(cp_h), _alive(ri)]
            cp = self.keep[2].data_ptr()
        self.c = _lib.CSR(self.keep[0].data_ptr(), self.keep[1].data_ptr(), None, cp,
                          self.keep[3].data_ptr() if cols else None, num_users, num_items)


# ---- groups.cu ------------------------------------------------------------------------------------------------------------
def _group_rows(case):
    rp, ci = gc.graph_of(case)
    g = _Graph(rp, ci, case["num_users"], int(ci.max()) + 1)
    members, cap = case["members"], case["cap"]
    G, M = members.shape
    row_ptr, col = support.filled(G + 1, S32), support.filled(cap, S32)
    ws, err, dm = torch.empty(2 * G + 1 + cap, dtype=torch.int32, device="cuda"), _err(), _alive(members)
    code = _lib.load().igmc_group_rows(C.byref(g.c), dm.data_ptr(), G, M, row_ptr.data_ptr(), col.data_ptr(), cap,
                                       ws.data_ptr(), err.data_ptr(), None)
    torch.cuda.synchronize()
    return code, int(err.item()), row_ptr.cpu().numpy(), col.cpu().numpy(), (rp, ci)


@pytest.mark.parametrize("case", _of("group_rows"), ids=support.pid)
def test_group_rows(case):
    code, err, got_rp, got_ci, (rp, ci) = _group_rows(case)
    want_rp, want_ci, want_err = gc.group_rows_reference(case, rp, ci)
    G, cap = len(case["members"]), case["cap"]
    assert code == 0 and err == want_err
    assert np.array_equal(got_rp[:G + 1], want_rp) and (got_rp[G + 1:] == S32).all()
    n = int(want_rp[-1])
    assert np.array_equal(got_ci[:n], want_ci) and (got_ci[max(cap, n):] == S32).all()


def test_group_rows_argument_checks():
    rp, ci = gc.group_graph()
    g = _Graph(rp, ci, gc.GROUP_NU, gc.GROUP_NI)
    z = torch.zeros(64, dtype=torch.int32, device="cuda")
    lib, p = _lib.load(), z.data_ptr()
    for G, M, cap, col in ((0, 1, 4, p), (1, 0, 4, p), (1, 65, 4, p), (1, 2, -1, p), (1, 2, 4, None)):
        assert lib.igmc_group_rows(C.byref(g.c), p, G, M, p, col, cap, p, p, None) == -1
    assert lib.igmc_group_rows(C.byref(g.c), p, 1, 2, p + 64, None, 0, p + 128, p + 252, None) == 0   # no col_idx
    torch.cuda.synchronize()


def _group_pairs(case):
    B = case["B"]
    members = case["members"]
    out = {k: support.filled(B, S32, dt) for k, dt in (("u", torch.int32), ("v", torch.int32), ("pid", torch.int64),
                                               ("tag", torch.int64))}
    keep = [_alive(members), _alive(case["unit_g"]), _alive(case["unit_v"]), _alive(case["unit_tag"], torch.int64)]
    err = _err()
    code = _lib.load().igmc_group_pairs(keep[0].data_ptr(), len(members), members.shape[1], case["num_users"],
                                        case["num_items"], keep[1].data_ptr(), keep[2].data_ptr(), keep[3].data_ptr(),
                                        B, out["u"].data_ptr(), out["v"].data_ptr(), out["pid"].data_ptr(),
                                        out["tag"].data_ptr(), err.data_ptr(), None)
    torch.cuda.synchronize()
    return code, int(err.item()), [out[k].cpu().numpy() for k in ("u", "v", "pid", "tag")]


@pytest.mark.parametrize("case", _of("group_pairs"), ids=support.pid)
def test_group_pairs(case):
    code, err, got = _group_pairs(case)
    want, want_err = gc.group_pairs_reference(case)
    assert code == 0 and err == want_err
    B = case["B"]
    for g, w in zip(got, want):
        assert np.array_equal(g[:B], w) and (g[B:] == S32).all()


def test_group_pairs_argument_checks():
    lib, x = _lib.load(), torch.zeros(64, dtype=torch.int64, device="cuda")
    p = x.data_ptr()
    for G, M, nu, ni, B in ((0, 1, 3, 3, 8), (1, 0, 3, 3, 8), (1, 65, 3, 3, 100), (1, 4, 3, 3, 3), (1, 1, 0, 3, 8),
                            (1, 1, 3, 0, 8)):
        assert lib.igmc_group_pairs(p, G, M, nu, ni, p, p, p, B, p, p, p, p, p, None) == -1
    assert lib.igmc_group_pairs(p, 1, 1, 3, 3, None, p, p, 8, p, p, p, p, p, None) == -1


@pytest.mark.parametrize("form", ["key", "scatter"])
@pytest.mark.parametrize("agg", ["mean", "min", "max"])
@pytest.mark.parametrize("case", _of("group_stats"), ids=support.pid)
def test_group_stats(case, agg, form):
    K, B, M, tag = case["K"], case["B"], case["M"], case["tag"]
    Gu = B // M
    T = int(tag.max()) + 1
    key, score, ms = (support.filled(n, SF, torch.float32) for n in (Gu, T, T * M))
    outs = (key.data_ptr(), None, None) if form == "key" else (None, score.data_ptr(), ms.data_ptr())
    preds = _alive(np.asarray(case["preds"], np.float32).reshape(K, B), torch.float32)
    assert _lib.load().igmc_group_stats(preds.data_ptr(), K, B, M, _lib.GROUP_AGGREGATES.index(agg),
                                        _alive(tag, torch.int64).data_ptr(), *outs, None) == 0
    torch.cuda.synchronize()
    want = gc.group_stats_reference(case, agg)
    nan = float("nan")
    if form == "key":
        got = key.cpu().numpy()
        assert same_f32(got[:Gu], [k for k, _, _ in want]) and (got[Gu:] == SF).all()
    else:
        ws, wm = np.full(T, SF, np.float32), np.full((T, M), SF, np.float32)
        for k, xs, t in want:
            if t >= 0:
                ws[t], wm[t] = k, [nan if v is None else v for v in xs]
        got_s, got_m = score.cpu().numpy(), ms.cpu().numpy()
        assert same_f32(got_s[:T], ws) and (got_s[T:] == SF).all()
        assert same_f32(got_m[:T * M], wm.reshape(-1)) and (got_m[T * M:] == SF).all()


def test_group_stats_argument_checks():
    lib, x = _lib.load(), torch.zeros(64, dtype=torch.float32, device="cuda")
    p = x.data_ptr()
    for K, B, M, agg, key, sc, ms in ((0, 8, 2, 0, p, None, None), (1, 8, 0, 0, p, None, None),
                                      (1, 8, 65, 0, p, None, None), (1, 3, 4, 0, p, None, None),
                                      (1, 8, 2, 3, p, None, None), (1, 8, 2, -1, p, None, None),
                                      (1, 8, 2, 0, None, p, None), (1, 8, 2, 0, None, None, p)):
        assert lib.igmc_group_stats(p, K, B, M, agg, p, key, sc, ms, None) == -1


# ---- diverse.cu -----------------------------------------------------------------------------------------------------------
def _union(items, ni):
    d = _alive(items, torch.int64)
    bitmap = support.filled((ni + 31) // 32, S32)
    mp, lst, nu, err = support.filled(ni, S32), support.filled(ni, S32), support.filled(1, S32), _err()
    code = _lib.load().igmc_item_union(d.data_ptr(), len(items), ni, bitmap.data_ptr(), mp.data_ptr(), lst.data_ptr(),
                                       nu.data_ptr(), err.data_ptr(), None)
    torch.cuda.synchronize()
    return code, int(err.item()), bitmap, mp, lst, nu


@pytest.mark.parametrize("case", _of("item_union"), ids=support.pid)
def test_item_union(case):
    ni = case["num_items"]
    code, err, bitmap, mp, lst, nu = _union(case["items"], ni)
    want_mp, want_lst, want_err = gc.item_union_reference(case)
    assert code == 0 and err == want_err
    n = len(want_lst)
    nu, mp, lst = nu.cpu().numpy(), mp.cpu().numpy(), lst.cpu().numpy()
    assert nu[0] == n and (nu[1:] == S32).all()
    assert np.array_equal(mp[:ni], want_mp) and (mp[ni:] == S32).all()
    assert np.array_equal(lst[:n], want_lst) and (lst[n:] == S32).all()
    W = (ni + 31) // 32
    assert (bitmap[W:].cpu().numpy() == S32).all()                        # the memset stops at the bitmap's end


def test_item_union_argument_checks():
    lib, x = _lib.load(), torch.zeros(64, dtype=torch.int64, device="cuda")
    p = x.data_ptr()
    for n, ni, items in ((-1, 8, p), (1, 0, p), (2, 8, None)):
        assert lib.igmc_item_union(items, n, ni, p, p, p, p, p, None) == -1
    assert lib.igmc_item_union(None, 0, 8, p, p, p, p, p, None) == 0
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def count_graph():
    rp, ci = gc.count_graph()
    return _Graph(rp, ci, gc.COUNT_NU, gc.COUNT_NI)


@pytest.mark.parametrize("case", _of("cocount"), ids=support.pid)
def test_cocount(case, count_graph):
    u = np.asarray(case["union"], np.int64)
    Nu = len(u)
    mp = np.full(gc.COUNT_NI, -1, np.int32)
    mp[u] = np.arange(Nu)
    need = Nu * (Nu - 1) // 2
    table = support.filled(need, S32)
    code = _lib.load().igmc_cocount(C.byref(count_graph.c), _alive(mp).data_ptr(), Nu, table.data_ptr(), case["cap"],
                                    None)
    torch.cuda.synchronize()
    got = table.cpu().numpy()
    if need > case["cap"]:
        assert code == -2 and (got == S32).all()
        return
    assert code == 0
    rp, ci = gc.count_graph()
    want = rc.cocount_host(rp, ci, gc.COUNT_NU, gc.COUNT_NI, u)              # the brute force's twin (CPU tests)
    assert np.array_equal(got[:need].view(np.uint32), want) and (got[need:] == S32).all()


def test_cocount_argument_checks(count_graph):
    lib, x = _lib.load(), torch.zeros(64, dtype=torch.int32, device="cuda")
    p = x.data_ptr()
    assert lib.igmc_cocount(C.byref(count_graph.c), p, -1, p, 10, None) == -1
    assert lib.igmc_cocount(C.byref(count_graph.c), p, gc.COUNT_NI + 1, p, 2 ** 40, None) == -1
    assert lib.igmc_cocount(C.byref(count_graph.c), None, 3, p, 3, None) == -1
    assert lib.igmc_cocount(C.byref(count_graph.c), p, 3, None, 3, None) == -1
    assert lib.igmc_cocount(C.byref(count_graph.c), p, 3, p, 2, None) == -2


def test_huge_table():
    """Nu = 65 537: table indices past 2^31 (8.6 GB of counts), read back by the cosine and the selection"""
    need = gc.HUGE_NU * (gc.HUGE_NU - 1) // 2
    free, _ = torch.cuda.mem_get_info()
    if free < need * 4 + (2 << 30):
        pytest.skip("the 8.6 GB co-count table does not fit the free device memory (%d bytes free)" % free)
    ni = gc.HUGE_NU
    rp, ci = gc.csr([np.asarray(r) for r in gc.HUGE_ROWS])
    g = _Graph(rp, ci, len(gc.HUGE_ROWS), ni, cols=True)
    mp = _alive(np.arange(ni))
    table = torch.full((need + GUARD,), S32, dtype=torch.int32, device="cuda")
    try:
        assert _lib.load().igmc_cocount(C.byref(g.c), mp.data_ptr(), ni, table.data_ptr(), need, None) == 0
        nz, cos = gc.huge_reference()
        idx = torch.as_tensor(sorted(nz), dtype=torch.int64, device="cuda")
        assert table[idx].cpu().tolist() == [nz[i] for i in sorted(nz)]
        assert int(table[:need].sum(dtype=torch.int64)) == sum(nz.values())    # nothing else counted
        assert (table[need:].cpu().numpy() == S32).all()
        items = _alive(gc.HUGE_ITEMS, torch.int64)
        Q = len(gc.HUGE_ITEMS)
        out, err = support.filled(Q * Q, SF, torch.float32), _err()
        assert _lib.load().igmc_item_cosine(C.byref(g.c), items.data_ptr(), Q, mp.data_ptr(), ni, table.data_ptr(),
                                            out.data_ptr(), err.data_ptr(), None) == 0
        torch.cuda.synchronize()
        assert int(err.item()) == 0
        got = out.cpu().numpy()
        assert same_f32(got[:Q * Q], cos.reshape(-1)) and (got[Q * Q:] == SF).all()
        # the greedy selection reads the same entries: pool = the items, scores equal, penalty 1
        pool = np.array([gc.HUGE_ITEMS[:6]], np.int64)
        sc = np.ones((1, 6), np.float32)
        oi, os_, ok = support.filled(6, S32, torch.int64), support.filled(6, SF, torch.float32), \
            support.filled(6, SF, torch.float32)
        assert _lib.load().igmc_diverse_select(C.byref(g.c), _alive(pool, torch.int64).data_ptr(),
                                               _alive(sc, torch.float32).data_ptr(), 1, 6, 6, 1.0, mp.data_ptr(), ni,
                                               table.data_ptr(), oi.data_ptr(), os_.data_ptr(), ok.data_ptr(),
                                               err.data_ptr(), None) == 0
        torch.cuda.synchronize()
        want = _select_with(pool, sc, 6, 1.0, lambda a, b: cos[gc.HUGE_ITEMS.index(a), gc.HUGE_ITEMS.index(b)])
        assert np.array_equal(oi.cpu().numpy()[:6], want[0]) and same_f32(ok.cpu().numpy()[:6], want[1])
    finally:
        del table
        torch.cuda.empty_cache()


def _select_with(pool, scores, k, penalty, sim):
    """the greedy loop of the header over one query with a given sim(a, b): (items, keys)"""
    P = pool.shape[1]
    live, m = [True] * P, [np.float32(0)] * P
    oi, ok = np.full(k, -1, np.int64), np.full(k, -np.inf, np.float32)
    pen = np.float32(penalty)
    for s in range(k):
        keys = [np.float32(scores[0, j] - np.float32(pen * m[j])) for j in range(P)]
        best = -1
        for j in range(P):
            if live[j] and (best < 0 or gc.ranks_before(float(keys[j]), j, float(keys[best]), best)):
                best = j
        oi[s], ok[s], live[best] = pool[0, best], keys[best], False
        for j in range(P):
            if live[j]:
                x = np.float32(sim(int(pool[0, j]), int(pool[0, best])))
                m[j] = x if x > m[j] else m[j]
    return oi, ok


@pytest.fixture(scope="module")
def select_graph():
    rp, ci = gc.select_graph()
    return _Graph(rp, ci, gc.SEL_NU, gc.SEL_NI, cols=True)


def _device_union(g, items, ni, nu_users):
    """map, list and table of the union of items built by the kernels under test (checked above)"""
    code, err, _, mp, lst, nu = _union(np.asarray(items, np.int64).reshape(-1), ni)
    Nu = int(nu[0])
    table = support.filled(Nu * (Nu - 1) // 2, S32)
    assert _lib.load().igmc_cocount(C.byref(g.c), mp.data_ptr(), Nu, table.data_ptr(), Nu * (Nu - 1) // 2, None) == 0
    return mp, Nu, table


@pytest.mark.parametrize("case", _of("select"), ids=support.pid)
def test_diverse_select(case, select_graph):
    pi, ps, k = case["pool_item"], case["pool_score"], case["k"]
    Q, P = pi.shape
    mp, Nu, table = _device_union(select_graph, pi, gc.SEL_NI, gc.SEL_NU)
    oi, os_, ok = support.filled(Q * k, S32, torch.int64), support.filled(Q * k, SF, torch.float32), \
        support.filled(Q * k, SF, torch.float32)
    err = _err()
    code = _lib.load().igmc_diverse_select(C.byref(select_graph.c), _alive(pi, torch.int64).data_ptr(),
                                           _alive(ps, torch.float32).data_ptr(), Q, P, k, case["penalty"],
                                           mp.data_ptr(), Nu, table.data_ptr(), oi.data_ptr(), os_.data_ptr(),
                                           ok.data_ptr(), err.data_ptr(), None)
    torch.cuda.synchronize()
    wi, ws, wk, werr = gc.select_reference(case)
    assert code == 0 and int(err.item()) == werr
    n = Q * k
    oi, os_, ok = oi.cpu().numpy(), os_.cpu().numpy(), ok.cpu().numpy()
    assert np.array_equal(oi[:n], wi.reshape(-1)) and (oi[n:] == S32).all()
    assert same_f32(os_[:n], ws.reshape(-1)) and (os_[n:] == SF).all()
    assert same_f32(ok[:n], wk.reshape(-1)) and (ok[n:] == SF).all()


def test_diverse_select_argument_checks(select_graph):
    lib, x = _lib.load(), torch.zeros(64, dtype=torch.int64, device="cuda")
    p = x.data_ptr()
    for Q, P, k, pen in ((1, 3, 4, 1.0), (1, 257, 2, 1.0), (1, 0, 1, 1.0), (1, 3, 0, 1.0), (-1, 3, 2, 1.0),
                         (1, 3, 2, -1.0), (1, 3, 2, float("inf")), (1, 3, 2, float("nan"))):
        assert lib.igmc_diverse_select(C.byref(select_graph.c), p, p, Q, P, k, pen, p, 3, p, p, p, p, None,
                                       None) == -1
    assert lib.igmc_diverse_select(C.byref(select_graph.c), p, p, 1, 3, 2, 1.0, p, 3, None, p, p, p, None, None) == -1
    assert lib.igmc_diverse_select(C.byref(select_graph.c), None, None, 0, 3, 2, 1.0, None, 0, None, None, None, None,
                                   None, None) == 0


@pytest.mark.parametrize("case", _of("cosine"), ids=support.pid)
def test_item_cosine(case, select_graph):
    items = case["items"]
    Q = len(items)
    mp, Nu, table = _device_union(select_graph, items, gc.SEL_NI, gc.SEL_NU)
    out, err = support.filled(Q * Q, SF, torch.float32), _err()
    assert _lib.load().igmc_item_cosine(C.byref(select_graph.c), _alive(items, torch.int64).data_ptr(), Q,
                                        mp.data_ptr(), Nu, table.data_ptr(), out.data_ptr(), err.data_ptr(), None) == 0
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert int(err.item()) == 0
    assert same_f32(got[:Q * Q], gc.cosine_reference(case).reshape(-1)) and (got[Q * Q:] == SF).all()


def test_item_cosine_flags_ids_outside_the_union(select_graph):
    _, ci = gc.select_graph()
    a, b, c = np.unique(ci)[:3].tolist()
    mp, Nu, table = _device_union(select_graph, [a, c], gc.SEL_NI, gc.SEL_NU)
    items = np.array([a, b, gc.SEL_NI, -1, c], np.int64)                   # b: not in the union
    out, err = support.filled(25, SF, torch.float32), _err()
    lib = _lib.load()
    assert lib.igmc_item_cosine(C.byref(select_graph.c), _alive(items, torch.int64).data_ptr(), 5, mp.data_ptr(), Nu,
                                table.data_ptr(), out.data_ptr(), err.data_ptr(), None) == 0
    torch.cuda.synchronize()
    got = out.cpu().numpy()[:25].reshape(5, 5)
    assert int(err.item()) == gc.ERR and (got[1:4] == 0).all() and (got[:, 1:4] == 0).all()
    assert got[0, 0] == 1 and got[4, 4] == 1
    p = out.data_ptr()
    assert lib.igmc_item_cosine(C.byref(select_graph.c), p, -1, p, 1, p, p, p, None) == -1
    assert lib.igmc_item_cosine(C.byref(select_graph.c), p, 3, p, 3, None, p, p, None) == -1


@pytest.mark.parametrize("case", _of("ws_bytes"), ids=support.pid)
def test_diverse_ws_bytes(case):
    nbytes, chunk = C.c_int64(-1), C.c_int(-1)
    assert _lib.load().igmc_diverse_ws_bytes(*case["args"], C.byref(nbytes), C.byref(chunk)) == 0
    assert (nbytes.value, chunk.value) == gc.ws_reference(case)
    assert _lib.load().igmc_diverse_ws_bytes(*case["args"], None, None) == -1
    q, pool, ni, bound = case["args"]
    for bad in ((0, pool, ni), (q, 0, ni), (q, pool, 0)):
        assert _lib.load().igmc_diverse_ws_bytes(*bad, bound, C.byref(nbytes), None) == -1


# ---- recommend_cache.cu ---------------------------------------------------------------------------------------------------
def _rescore(case, g, chunk, out_cap):
    U, ni = len(case["users"]), case["num_items"]
    ws = torch.empty(gc.plan_ws_bytes(ni, chunk), dtype=torch.uint8, device="cuda")
    user_off, out = support.filled(U + 1, S32, torch.int64), support.filled(max(out_cap, 0), S32)
    full, totals, err = support.filled(U, S8, torch.uint8), support.filled(2, S32, torch.int64), _err()
    cand = case["cand"]
    cd = None if cand is None else _alive(cand)
    eu, ev = _alive(case["edit_u"]), _alive(case["edit_v"])
    code = _lib.load().igmc_rescore_plan(C.byref(g.c), _alive(case["users"]).data_ptr(), U, eu.data_ptr(),
                                         ev.data_ptr(), len(case["edit_u"]), _lib.ptr(cd),
                                         0 if cand is None else len(cand), case["exclude"], ws.data_ptr(), ws.numel(),
                                         user_off.data_ptr(), out.data_ptr(), out_cap, full.data_ptr(),
                                         totals.data_ptr(), err.data_ptr(), None)
    torch.cuda.synchronize()
    return code, int(err.item()), [t.cpu().numpy() for t in (user_off, out, full, totals)]


@pytest.mark.parametrize("case", _of("rescore"), ids=support.pid)
def test_rescore_plan_every_chunk_size(case):
    rp, ci = gc.cache_graph(case["num_items"])
    g = _Graph(rp, ci, gc.CACHE_NU, case["num_items"])
    off, items, full, totals, want_err = gc.rescore_reference(case)
    U, n = len(case["users"]), len(items)
    caps = [n] + ([n - 1] if n > 0 and "out_cap=total-1" in case["claims"] else [])
    for chunk in case["chunks"]:
        for cap in caps:
            code, err, (g_off, g_out, g_full, g_tot) = _rescore(case, g, chunk, cap)
            what = (chunk, cap)
            assert code == 0, what
            assert err == (want_err or (gc.ERR if cap < n else 0)), what
            assert np.array_equal(g_off[:U + 1], off) and (g_off[U + 1:] == S32).all(), what
            assert np.array_equal(g_out[:min(cap, n)], items[:cap]) and (g_out[cap:] == S32).all(), what
            assert np.array_equal(g_full[:U], full) and (g_full[U:] == S8).all(), what
            assert tuple(g_tot[:2]) == totals and (g_tot[2:] == S32).all(), what


def test_rescore_plan_argument_checks():
    rp, ci = gc.cache_graph(33)
    g = _Graph(rp, ci, gc.CACHE_NU, 33)
    lib, x = _lib.load(), torch.zeros(4096, dtype=torch.int64, device="cuda")
    p = x.data_ptr()
    ws = gc.plan_ws_bytes(33, 1)
    assert lib.igmc_rescore_plan(C.byref(g.c), p, 2, p, p, 1, None, 0, 1, p, ws - 1, p, p, 8, p, p, p, None) == -2
    for U, E, cand, nc, cap, ub in ((-1, 1, None, 0, 8, p), (2, -1, None, 0, 8, p), (2, 1, p, 0, 8, p),
                                    (2, 1, None, -1, 8, p), (2, 1, None, 0, -1, p), (2, 1, None, 0, 8, None)):
        assert lib.igmc_rescore_plan(C.byref(g.c), ub, U, p, p, E, cand, nc, 1, p, ws, p, p, cap, p, p, p, None) == -1
    assert lib.igmc_rescore_plan(C.byref(g.c), p, 2, p, p, 1, None, 0, 1, p, ws, p, None, 8, p, p, p, None) == -1
    nbytes, chunk = C.c_int64(0), C.c_int(0)
    assert lib.igmc_rescore_plan_ws_bytes(3000, 32769, gc.plan_ws_bytes(32769, 1025), C.byref(nbytes),
                                          C.byref(chunk)) == 0
    assert chunk.value == 1025 and nbytes.value == gc.plan_ws_bytes(32769, 1025)
    assert lib.igmc_rescore_plan_ws_bytes(3000, 0, 0, C.byref(nbytes), None) == -1
    torch.cuda.synchronize()


@pytest.mark.parametrize("case", _of("invalidate"), ids=support.pid)
def test_cache_invalidate(case):
    U, D = case["top_i"].shape
    ts, ti = _alive(np.r_[case["top_s"].reshape(-1), [SF] * GUARD], torch.float32), \
        _alive(np.r_[case["top_i"].reshape(-1), [S32] * GUARD], torch.int64)
    thr_s, thr_i = support.filled(U, SF, torch.float32), support.filled(U, S32, torch.int64)
    assert _lib.load().igmc_cache_invalidate(U, D, _alive(case["user_off"], torch.int64).data_ptr(),
                                             _alive(case["resc"]).data_ptr(),
                                             _alive(case["full"], torch.uint8).data_ptr(),
                                             _alive(case["complete"], torch.uint8).data_ptr(), ts.data_ptr(),
                                             ti.data_ptr(), thr_s.data_ptr(), thr_i.data_ptr(), None) == 0
    torch.cuda.synchronize()
    ws, wi, wts, wti = gc.invalidate_reference(case)
    for got, want, sent in ((ts, ws, SF), (ti, wi, S32), (thr_s, wts, SF), (thr_i, wti, S32)):
        got, want = got.cpu().numpy(), want.reshape(-1)
        n = len(want)
        assert (same_f32(got[:n], want) if want.dtype == np.float32 else np.array_equal(got[:n], want))
        assert (got[n:] == sent).all()


@pytest.mark.parametrize("case", _of("settle"), ids=support.pid)
def test_cache_settle(case):
    U, D = case["top_i"].shape
    ts, ti = _alive(np.r_[case["top_s"].reshape(-1), [SF] * GUARD], torch.float32), \
        _alive(np.r_[case["top_i"].reshape(-1), [S32] * GUARD], torch.int64)
    complete, redo, cnt = support.filled(U, S8, torch.uint8), support.filled(U, S32), support.filled(1, S32)
    assert _lib.load().igmc_cache_settle(U, D, case["k"], _alive(case["thr_s"], torch.float32).data_ptr(),
                                         _alive(case["thr_i"], torch.int64).data_ptr(), ts.data_ptr(), ti.data_ptr(),
                                         complete.data_ptr(), redo.data_ptr(), cnt.data_ptr(), None) == 0
    torch.cuda.synchronize()
    ws, wi, wc, wr = gc.settle_reference(case)
    ts, ti, complete, redo, cnt = (t.cpu().numpy() for t in (ts, ti, complete, redo, cnt))
    n = U * D
    assert same_f32(ts[:n], ws.reshape(-1)) and (ts[n:] == SF).all()
    assert np.array_equal(ti[:n], wi.reshape(-1)) and (ti[n:] == S32).all()
    assert np.array_equal(complete[:U], wc) and (complete[U:] == S8).all()
    r = len(wr)
    assert cnt[0] == r and (cnt[1:] == S32).all()
    assert np.array_equal(redo[:r], wr) and (redo[r:] == S32).all()


def test_invalidate_and_settle_argument_checks():
    lib, x = _lib.load(), torch.zeros(64, dtype=torch.int64, device="cuda")
    p = x.data_ptr()
    for U, D in ((-1, 4), (2, 0), (2, 257)):
        assert lib.igmc_cache_invalidate(U, D, p, p, p, p, p, p, p, p, None) == -1
    assert lib.igmc_cache_invalidate(2, 4, None, p, p, p, p, p, p, p, None) == -1
    for U, D, k in ((-1, 4, 2), (2, 0, 1), (2, 257, 2), (2, 4, 0), (2, 4, 5)):
        assert lib.igmc_cache_settle(U, D, k, p, p, p, p, p, p, p, None) == -1
    assert lib.igmc_cache_settle(2, 4, 2, p, p, p, p, p, p, None, None) == -1
    assert lib.igmc_cache_settle(2, 4, 2, None, p, p, p, p, p, p, None) == -1


# ---- end to end on a graph of 9 000 items ---------------------------------------------------------------------------------
E2E_NU, E2E_NI = 1100, 9000


@pytest.fixture(scope="module")
def e2e():
    from igmc_b200.models import IGMC
    u, v, lab = synth_ratings(E2E_NU, E2E_NI, 30000, 5, seed=6)
    A = build_adj(u, v, lab, E2E_NU, E2E_NI)
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    rng = np.random.default_rng(8)
    items = np.unique(np.r_[rng.choice(E2E_NI, 50, replace=False), 8192, 8193, 8999, 8998])
    return A, m, items


def test_recommend_groups_e2e(e2e):
    """300 groups (past one chunk of the group scans) over a shared list reaching past item 8 192"""
    A, m, items = e2e
    g = RatingGraph(A)
    rng = np.random.default_rng(9)
    deg = np.diff(g.host["row_ptr"])[:g.num_users]
    pool = np.flatnonzero(deg > 0)
    groups = [[int(x) for x in rng.choice(pool, int(rng.integers(1, 5)), replace=False)] for _ in range(300)]
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=50, batch_size=256)
    try:
        members = rc._group_members(groups, g.num_users, 64)
        us = np.unique(members[members >= 0]).astype(np.int64)
        tab = eng.predict_pairs(np.repeat(us, len(items)), np.tile(items, len(us))).cpu().numpy().reshape(len(us), -1)

        def scorer(uu, vv):
            return tab[np.searchsorted(us, np.asarray(uu, np.int64)), np.searchsorted(items, np.asarray(vv, np.int64))]
        hp = g.host
        for agg in ("mean", "min"):
            ti, ts = eng.recommend_groups(groups, 5, agg, items)
            wi, ws = rc.recommend_groups_host(hp["row_ptr"], hp["col_idx"], g.num_items, members, 5, agg, scorer,
                                              items)
            assert np.array_equal(ti.cpu().numpy(), wi) and same_f32(ts.cpu().numpy(), ws)
    finally:
        eng.close()


def test_recommend_diverse_e2e(e2e):
    """pools over a shared list with items past 8 192: the union scan's second chunk"""
    A, m, items = e2e
    g = RatingGraph(A)
    users = np.arange(0, 60, 5, dtype=np.int64)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=50, batch_size=256)
    try:
        got = eng.recommend_diverse(users, 8, 1.5, 40, items=items)
        hp = g.host

        def pooler(us, p):
            ti, ts = eng.recommend(us, p, items=items)
            return ti.cpu().numpy(), ts.cpu().numpy()
        want = rc.recommend_diverse_host(hp["row_ptr"], hp["col_idx"], hp["col_ptr"], g.num_users, g.num_items, users,
                                         8, 1.5, pooler, 40)
        assert (pooler(users, 40)[0] >= 8192).any()
        assert np.array_equal(got.items.cpu().numpy(), want[0])
        assert same_f32(got.scores.cpu().numpy(), want[1]) and same_f32(got.keys.cpu().numpy(), want[2])
    finally:
        eng.close()


def test_recommendation_cache_e2e(e2e):
    """1 100 cached slots (past one chunk of k_cache_settle and k_rp_scan) over a catalogue of 9 000 items"""
    A, m, items = e2e
    g = RatingGraph(A, reserve_nnz=100)
    users = np.arange(E2E_NU, dtype=np.int64)
    kw = dict(items=items, max_nodes_per_hop=50, batch_size=256)
    cache = rc.RecommendationCache(m, g, users, 5, depth=10, **kw)
    try:
        rng = np.random.default_rng(10)
        eu, ev = rng.integers(0, E2E_NU, 12), np.r_[rng.choice(items, 10), 8192, 8999]
        out = cache.update(eu, ev, rng.integers(1, 6, 12))
        assert not out["full"] and out["rescored_pairs"] > 0
        got_i, got_s = cache.lists()
        want_i, want_s = rc.recommend(m, g, users, 5, **kw)
        assert torch.equal(got_i, want_i) and torch.equal(got_s.view(torch.int32), want_s.view(torch.int32))
    finally:
        cache.close()
