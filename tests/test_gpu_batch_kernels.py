"""igmc_batch_ptrs and igmc_batch_prepare called directly on foreign batches, against the brute-force references of
tests/foreign_batch_cases.py written from the header's contract.

Every output is sentinel-filled and sized past what the kernel may write; the guard must stay untouched.  The error
word is read after every call.  ``symmetric = 1`` must build the same in-lists and leave the out-lists untouched.
igmc_batch_prepare is never launched on the offsets of an igmc_batch_ptrs call that flagged an error (they are
undefined then)."""
import ctypes as C

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200.util_functions import _stream_ptr
from tests import foreign_batch_cases as fb
from tests import support

pytestmark = pytest.mark.gpu

GUARD = 64
S32 = -777
ERR_SMEM_NODES, ERR_BAD_BATCH = 4, 5     # IGMC_ERR_* (csrc/common.cuh)
R = 5
SMEM_NCAP_MAX = 200 * 1024 // 8 - 1      # 2 (n_cap + 1) ints of shared memory within 200 KB


def _take_err(err):
    code = int(err.item())
    err.zero_()
    return code


def _ptrs(batch, src, N, E, B, err):
    batch_d, src_d = support.dev_np(batch if N else [0], np.int64), support.dev_np(src if E else [0], np.int64)
    node_ptr, edge_ptr = support.filled(B + 1, S32, torch.int32, GUARD), support.filled(B + 1, S32, torch.int32, GUARD)
    _lib.check(_lib.load().igmc_batch_ptrs(batch_d.data_ptr() if N else None, src_d.data_ptr(), N, E, B,
                                           node_ptr.data_ptr(), edge_ptr.data_ptr(), err.data_ptr(), _stream_ptr()),
               "igmc_batch_ptrs")
    return node_ptr.cpu().numpy(), edge_ptr.cpu().numpy(), _take_err(err)


def _prepare(ei, et, node_ptr, edge_ptr, B, n_cap, symmetric, err, stride_pad=0):
    """(return code, {in/out: (ptr, adj, eid) with guards}, error code); edge_index as a [2, E + stride_pad] buffer"""
    ei = np.asarray(ei, np.int64).reshape(2, -1)
    N, E = int(node_ptr[B]), ei.shape[1]
    buf = np.full((2, E + stride_pad), -5, np.int64)
    buf[:, :E] = ei
    ei_d, et_d = support.dev_np(buf.reshape(-1), np.int64), support.dev_np(np.append(et, 0), np.int64)
    np_d, ep_d = support.dev_np(node_ptr[:B + 1], np.int32), support.dev_np(edge_ptr[:B + 1], np.int32)
    t = {k: support.filled(N + 1 if k.endswith("ptr") else E, S32, torch.int32, GUARD)
         for k in ("in_ptr", "in_adj", "in_eid", "out_ptr", "out_adj", "out_eid")}
    tmp = torch.zeros(E + 1, dtype=torch.int64, device="cuda")
    A = _lib.Adj(*(t[k].data_ptr() for k in ("in_ptr", "in_adj", "in_eid", "out_ptr", "out_adj", "out_eid")),
                 tmp.data_ptr(), int(symmetric))
    rc = _lib.load().igmc_batch_prepare(ei_d.data_ptr(), E + stride_pad, et_d.data_ptr(), np_d.data_ptr(),
                                        ep_d.data_ptr(), B, n_cap, C.byref(A), err.data_ptr(), _stream_ptr())
    torch.cuda.synchronize()
    got = {side: tuple(t["%s_%s" % (side, k)].cpu().numpy() for k in ("ptr", "adj", "eid")) for side in ("in", "out")}
    return rc, got, _take_err(err)


def _untouched(a):
    return bool(np.all(a == S32))


def _check_valid(ob, err, n_cap=None, stride_pad=0):
    B, bt = int(ob["num_graphs"]), np.asarray(ob["batch"], np.int64)
    ei, et = np.asarray(ob["edge_index"], np.int64).reshape(2, -1), np.asarray(ob["edge_type"], np.int64)
    N, E = len(bt), ei.shape[1]
    node_ptr, edge_ptr, code = _ptrs(bt, ei[0], N, E, B, err)
    want_np, want_ep = fb.ptrs_reference(bt, ei[0], B)
    assert code == 0
    assert np.array_equal(node_ptr[:B + 1], want_np) and _untouched(node_ptr[B + 1:])
    assert np.array_equal(edge_ptr[:B + 1], want_ep) and _untouched(edge_ptr[B + 1:])
    if n_cap is None:
        n_cap = max(int(np.diff(want_np).max(initial=0)), 2)
    want = fb.lists_reference(ei, et, want_np)
    for symmetric in (0, 1):
        rc, got, code = _prepare(ei, et, node_ptr, edge_ptr, B, n_cap, symmetric, err, stride_pad)
        assert rc == 0 and code == 0, (rc, code)
        for side in ("in",) if symmetric else ("in", "out"):
            for k, (g, w) in enumerate(zip(got[side], want[side])):
                assert np.array_equal(g[:len(w)], w), (side, k, symmetric)
                assert _untouched(g[len(w):]), (side, k, symmetric)
        if symmetric:
            assert all(_untouched(a) for a in got["out"])


def _empty_graph(F):
    return (np.zeros((0, F), np.float32), np.zeros((2, 0), np.int64), np.zeros(0, np.int64), 0.0)


def _with_empty(ob, where):
    """``ob`` with node-less graphs at the (final) positions ``where``"""
    parts = fb.split(ob)
    for at in sorted(where):
        parts.insert(at, _empty_graph(np.asarray(ob["x"]).shape[1]))
    return fb.collate(parts)


def _hub_graph(deg=300, seed=0):
    """one graph of deg + 2 nodes: node 0 receives an edge of a random type from every other node, plus a ring"""
    rng = np.random.default_rng(seed)
    n = deg + 2
    x = np.zeros((n, 4), np.float32)
    x[0, 0] = x[1, 1] = 1
    x[2:, 2] = 1
    src = np.concatenate([np.arange(1, n), np.arange(n)])
    dst = np.concatenate([np.zeros(n - 1, np.int64), (np.arange(n) + 1) % n])
    o = rng.permutation(len(src))
    return fb.collate([(x, np.stack([src, dst])[:, o], rng.integers(0, R, len(src)), 1.0)])


@pytest.fixture(scope="module")
def small():
    return fb.small(R)


@pytest.fixture
def err():
    yield torch.zeros(1, dtype=torch.int32, device="cuda")


VALID = ["permuted", "multigraph", "multigraph_B1", "skewed", "edgeless_middle", "empty_first_middle_last",
         "all_empty", "hub_in300", "types_0_255", "stride_gt_E", "n_eq_ncap", "ncap_smem_max"]


@pytest.mark.parametrize("case", VALID)
def test_valid(case, small, err):
    kw = {}
    if case == "permuted":
        ob = fb.permuted(small, 1)
    elif case == "multigraph":
        ob = fb.multigraph(small, R, 2)
    elif case == "multigraph_B1":
        ob = fb.multigraph(small, R, 3, graphs=[0])
    elif case == "skewed":
        ob = fb.skewed(small, R, 5, 4, senders=3, receivers=2, fan=2)[0]
    elif case == "edgeless_middle":
        ob = fb.with_edgeless(small, 8, 5)
    elif case == "empty_first_middle_last":
        ob = _with_empty(fb.permuted(small, 1), [0, 9, 18])
        sizes = np.bincount(ob["batch"], minlength=ob["num_graphs"])
        assert ob["num_graphs"] == 19 and sizes[0] == sizes[9] == sizes[18] == 0
    elif case == "all_empty":
        ob = fb.collate([_empty_graph(4)] * 3)
        assert len(ob["batch"]) == 0 and ob["edge_index"].shape[1] == 0
    elif case == "hub_in300":
        ob = _hub_graph()                      # rank_sort_list: a 300-entry list takes more than one lane pass
    elif case == "types_0_255":
        ob = fb.multigraph(small, R, 2)
        ob["edge_type"] = np.where(np.arange(len(ob["edge_type"])) % 3 == 0, 255, ob["edge_type"] % 1)
    elif case == "stride_gt_E":
        ob, kw = fb.multigraph(small, R, 2), dict(stride_pad=37)
    elif case == "n_eq_ncap":
        ob = fb.multigraph(small, R, 2)
        kw = dict(n_cap=int(np.bincount(ob["batch"]).max()))
    else:
        ob, kw = fb.permuted(small, 1), dict(n_cap=SMEM_NCAP_MAX)
    _check_valid(ob, err, **kw)


def test_ncap_over_smem_limit(small, err):
    ob = fb.permuted(small, 1)
    bt, ei = np.asarray(ob["batch"]), np.asarray(ob["edge_index"])
    node_ptr, edge_ptr, code = _ptrs(bt, ei[0], len(bt), ei.shape[1], ob["num_graphs"], err)
    assert code == 0
    rc, got, code = _prepare(ei, ob["edge_type"], node_ptr, edge_ptr, ob["num_graphs"], SMEM_NCAP_MAX + 1, 0, err)
    assert rc == -3 and code == 0
    assert all(_untouched(a) for side in got.values() for a in side)


def _ptrs_invalid(case, ob):
    bt, ei = np.asarray(ob["batch"]).copy(), np.asarray(ob["edge_index"]).copy()
    B = int(ob["num_graphs"])
    nptr = np.concatenate([[0], np.cumsum(np.bincount(bt, minlength=B))])
    if case == "batch_decreasing":
        bt[nptr[3] + 1] = 1
    elif case == "batch_id_ge_B":
        bt[nptr[B - 1]:] = B
    elif case == "leading_minus_one":
        bt[:nptr[1]] = -1                     # graph 0's nodes (its targets included) belong to no graph
        keep = ei[0] >= nptr[1]
        ei = ei[:, keep]                      # and have no edges: nothing else would flag them
    elif case == "edge_src_out_of_range":
        ei[0, ei.shape[1] // 2] = len(bt)
    elif case == "edge_src_negative":
        ei[0, 0] = -1
    elif case == "edges_not_grouped":
        e0 = np.nonzero(bt[ei[0]] == 2)[0][0]
        ei[:, [0, e0]] = ei[:, [e0, 0]]
    return bt, ei


PTRS_INVALID = ["batch_decreasing", "batch_id_ge_B", "leading_minus_one", "edge_src_out_of_range",
                "edge_src_negative", "edges_not_grouped"]


@pytest.mark.parametrize("case", PTRS_INVALID)
def test_ptrs_invalid(case, small, err):
    ob = fb.permuted(small, 1)
    bt, ei = _ptrs_invalid(case, ob)
    _, _, code = _ptrs(bt, ei[0], len(bt), ei.shape[1], ob["num_graphs"], err)
    assert code == ERR_BAD_BATCH, code


PREPARE_INVALID = ["dst_in_other_graph", "type_minus_one", "type_256", "n_over_ncap"]


@pytest.mark.parametrize("case", PREPARE_INVALID)
def test_prepare_invalid(case, small, err):
    ob = fb.multigraph(small, R, 2)
    bt, ei, et = np.asarray(ob["batch"]), np.asarray(ob["edge_index"]).copy(), np.asarray(ob["edge_type"]).copy()
    B = int(ob["num_graphs"])
    node_ptr, edge_ptr, code = _ptrs(bt, ei[0], len(bt), ei.shape[1], B, err)
    assert code == 0
    n_cap, want = int(np.bincount(bt).max()), ERR_BAD_BATCH
    bad = int(edge_ptr[4])                    # the first edge of graph 4
    if case == "dst_in_other_graph":
        ei[1, bad] = node_ptr[5]
    elif case == "type_minus_one":
        et[bad] = -1
    elif case == "type_256":
        et[bad] = 256
    else:
        n_cap, want = n_cap - 1, ERR_SMEM_NODES
    for symmetric in (0, 1):
        rc, got, code = _prepare(ei, et, node_ptr, edge_ptr, B, n_cap, symmetric, err)
        assert rc == 0 and code == want, (symmetric, code)
        if case.startswith("type"):
            # the bad entry joins no list: every other graph's lists and pointers are the reference's, graph 4's are
            # the reference's without that edge (its last slot left unwritten), and the terminal pointer is E
            ref = fb.lists_reference(ei, np.where(np.arange(len(et)) == bad, 0, et), node_ptr[:B + 1])
            keep = np.arange(len(et)) != bad
            cut = fb.lists_reference(ei[:, keep], et[keep], node_ptr[:B + 1])
            lo, hi, N = int(edge_ptr[4]), int(edge_ptr[5]), int(node_ptr[B])
            n4 = np.arange(int(node_ptr[4]), int(node_ptr[5]))
            for side in ("in",) if symmetric else ("in", "out"):
                ptr, adj, eid = got[side]
                others = np.setdiff1d(np.arange(N + 1), n4)
                assert np.array_equal(ptr[others], ref[side][0][others]), side
                assert np.array_equal(ptr[n4], cut[side][0][n4]), side
                assert ptr[N] == len(et) and _untouched(ptr[N + 1:])
                outside = np.r_[0:lo, hi:int(edge_ptr[B])]
                assert np.array_equal(adj[outside], ref[side][1][outside])
                assert np.array_equal(eid[outside], ref[side][2][outside])
                cut_eid = cut[side][2][lo:hi - 1]
                assert np.array_equal(adj[lo:hi - 1], cut[side][1][lo:hi - 1])
                assert np.array_equal(eid[lo:hi - 1], cut_eid + (cut_eid >= bad))
                assert adj[hi - 1] == S32 and eid[hi - 1] == S32
