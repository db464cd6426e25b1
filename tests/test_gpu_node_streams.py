"""The node explanation kernels called directly on batches built here, against brute-force enumeration written from
the header's contract (tests/node_stream_cases.py), not against the host twins.

* igmc_explain_node_count: num_nodes at each tag, untouched elsewhere;
* igmc_node_occlusion_mask: edge_keep edge by edge (0 exactly on the directed edges of the node's ratings), the node's
  global id, label and rating count at its position; a position outside the graph sets the error word, drops nothing
  and records nothing;
* igmc_node_grad_scatter over K = 1 and 3 checkpoints: bit for bit the float32 sum in in-list order (int32 view);
  records at k = 0 only; a graph whose node count is not the base pass's sets the error word and writes nothing.
Every output is sentinel-filled and sized past what the kernel may write; the guard is checked."""
import ctypes as C

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200.util_functions import _stream_ptr
from tests import node_stream_cases as ns
from tests import support

pytestmark = pytest.mark.gpu

GUARD = 64
S32 = -777
FSENT = 0x7f80dead
ERR_CANDIDATES = 7     # IGMC_ERR_CANDIDATES (csrc/common.cuh)


def _take_err(err):
    code = int(err.item())
    err.zero_()
    return code


def _batch_out(bt):
    E = int(bt["edge_ptr"][-1])
    ecap = E + 16
    ei = np.zeros((2, ecap), np.int64)
    ei[0, :E], ei[1, :E] = bt["src"], bt["dst"]
    t = dict(node_ptr=support.dev_np(bt["node_ptr"], np.int32), edge_ptr=support.dev_np(bt["edge_ptr"], np.int32),
             edge_index=support.dev_np(ei.reshape(-1), np.int64), node_label=support.dev_np(bt["node_label"], np.uint8),
             node_gid=support.dev_np(bt["node_gid"], np.int32), adj_in_ptr=support.dev_np(bt["in_ptr"], np.int32),
             adj_eid=support.dev_np(np.concatenate([bt["in_eid"], [0]]), np.int32))
    O = _lib.BatchOut()
    O.edge_cap = ecap
    for k, v in t.items():
        setattr(O, k, v.data_ptr())
    return O, t


@pytest.fixture
def err():
    yield torch.zeros(1, dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("name", list(ns.SHAPES))
def test_node_count(name, err):
    shapes, h = ns.SHAPES[name]
    bt = ns.make_batch(11, shapes, h)
    B = len(shapes)
    tag = np.arange(B)[::-1] * 2            # pair 2 * (B - 1 - g); the odd pairs are untouched
    tag[0] = -1
    out = support.filled(2 * B, S32, torch.int32, GUARD)
    node_ptr, tag_d = support.dev_np(bt["node_ptr"], np.int32), support.dev_np(tag, np.int64)  # alive until it has run
    _lib.check(_lib.load().igmc_explain_node_count(node_ptr.data_ptr(), tag_d.data_ptr(), B, out.data_ptr(),
                                                   _stream_ptr()),
               "igmc_explain_node_count")
    want = np.full(2 * B + GUARD, S32)
    for g in range(1, B):
        want[tag[g]] = len(ns.positions(bt, g))
    assert np.array_equal(out.cpu().numpy(), want), name


@pytest.mark.parametrize("name", list(ns.SHAPES))
@pytest.mark.parametrize("where", ["first", "last", "chunk", "invalid"])
def test_node_occlusion_mask(name, where, err):
    shapes, h = ns.SHAPES[name]
    bt = ns.make_batch(12, shapes, h)
    B = len(shapes)
    lib = _lib.load()
    O, keep_t = _batch_out(bt)
    E = int(bt["edge_ptr"][-1])
    npos = [len(ns.positions(bt, g)) for g in range(B)]
    pick = dict(first=lambda n: 0, last=lambda n: n - 1, chunk=lambda n: min(ns.MASK_THREADS, n - 1),
                invalid=lambda n: n)
    j = np.array([pick[where](n) if n else 0 for n in npos])
    tag = 3 * np.arange(B) + 1                # positions 1, 4, 7, ...: the rest of T stays untouched
    if B > 1:
        tag[1] = -1                            # a padding graph: nothing dropped, nothing recorded
    T = 3 * B + 1
    keep = support.filled(E, 7, torch.uint8, GUARD)
    rec = [support.filled(T, S32, torch.int32, GUARD) for _ in range(3)]
    tag_d, j_d = support.dev_np(tag, np.int64), support.dev_np(j, np.int32)
    _lib.check(lib.igmc_node_occlusion_mask(C.byref(O), B, tag_d.data_ptr(), j_d.data_ptr(), keep.data_ptr(),
                                            rec[0].data_ptr(), rec[1].data_ptr(), rec[2].data_ptr(), err.data_ptr(),
                                            _stream_ptr()), "igmc_node_occlusion_mask")
    want_keep = np.ones(E, np.uint8)
    want_rec = np.full((3, T), S32)
    bad = False
    for g in range(B):
        if tag[g] < 0:
            continue
        drop, r = ns.mask_brute(bt, g, int(j[g]))
        if r is None:
            bad = True
            continue
        want_keep[drop] = 0
        want_rec[:, tag[g]] = r
    assert _take_err(err) == (ERR_CANDIDATES if bad else 0), (name, where)
    got = keep.cpu().numpy()
    assert np.array_equal(got[:E], want_keep) and (got[E:] == 7).all(), (name, where)
    for g in range(B):                         # edge by edge: 0 exactly on the node's ratings' two directed copies
        e = np.arange(bt["edge_ptr"][g], bt["edge_ptr"][g + 1])
        m = len(e) // 2
        assert np.array_equal(got[e[:m]], got[e[m:]])
    for k in range(3):
        assert np.array_equal(rec[k].cpu().numpy()[:T], want_rec[k]), (name, where, k)
        assert (rec[k].cpu().numpy()[T:] == S32).all()


@pytest.mark.parametrize("name", list(ns.SHAPES))
@pytest.mark.parametrize("K", [1, 3])
def test_node_grad_scatter(name, K, err):
    shapes, h = ns.SHAPES[name]
    bt = ns.make_batch(13, shapes, h)
    B = len(shapes)
    lib = _lib.load()
    O, keep_t = _batch_out(bt)
    E = int(bt["edge_ptr"][-1])
    npos = np.array([len(ns.positions(bt, g)) for g in range(B)])
    tag = np.random.default_rng(3).permutation(B)
    counts = np.zeros(B, np.int64)
    counts[tag] = npos
    if B > 1:
        tag[-1] = -1                          # a padding graph writes nothing
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    T = int(off[-1])
    rng = np.random.default_rng(4)
    grads = [rng.standard_normal(E + 1).astype(np.float32) for _ in range(K)]
    if E:
        grads[0][rng.integers(0, E, 3)] = [np.inf, -0.0, 1e30]
    out = support.filled(T, 0.0, torch.float32, GUARD)
    out.view(torch.int32).fill_(FSENT)
    rec = [support.filled(T, S32, torch.int32, GUARD) for _ in range(3)]
    want = np.full(T, FSENT, np.int32).view(np.float32)
    want_rec = np.full((3, T), S32)
    tag_d, off_d = support.dev_np(tag, np.int64), support.dev_np(off, np.int64)
    for k in range(K):
        g_dev = support.dev_np(grads[k], np.float32)
        _lib.check(lib.igmc_node_grad_scatter(C.byref(O), B, tag_d.data_ptr(), g_dev.data_ptr(), off_d.data_ptr(), k,
                                              K, out.data_ptr(), rec[0].data_ptr(), rec[1].data_ptr(),
                                              rec[2].data_ptr(), err.data_ptr(), _stream_ptr()),
                   "igmc_node_grad_scatter")
        assert _take_err(err) == 0
        for g in range(B):
            if tag[g] < 0:
                continue
            v, recs = ns.grad_brute(bt, g, grads[k])
            o = int(off[tag[g]])
            seg = slice(o, o + len(v))
            cur = v if k == 0 else (want[seg] + v).astype(np.float32)
            if k == K - 1 and K > 1:
                cur = (cur / np.float32(K)).astype(np.float32)
            want[seg] = cur
            if k == 0:
                want_rec[:, seg] = np.asarray(recs, np.int64).T.reshape(3, -1)
        got = out.cpu().numpy()
        assert np.array_equal(got.view(np.int32)[:T], want.view(np.int32)), (name, K, k)
        assert (got.view(np.int32)[T:] == FSENT).all()
        for i in range(3):
            assert np.array_equal(rec[i].cpu().numpy()[:T], want_rec[i] if k == 0 else np.full(T, S32)), (name, k, i)
            assert (rec[i].cpu().numpy()[T:] == S32).all()
            rec[i].fill_(S32)


def test_node_grad_scatter_rejects_a_foreign_count(err):
    shapes, h = ns.SHAPES["one rating and many"]
    bt = ns.make_batch(14, shapes, h)
    B = len(shapes)
    O, keep_t = _batch_out(bt)
    npos = np.array([len(ns.positions(bt, g)) for g in range(B)])
    npos[0] += 1                                   # the base pass counted another subgraph for pair 0
    off = np.concatenate([[0], np.cumsum(npos)]).astype(np.int64)
    T = int(off[-1])
    out = support.filled(T, 0.0, torch.float32, GUARD)
    out.view(torch.int32).fill_(FSENT)
    rec = [support.filled(T, S32, torch.int32, GUARD) for _ in range(3)]
    g = support.dev_np(np.ones(int(bt["edge_ptr"][-1]) + 1), np.float32)
    tag_d, off_d = support.dev_np(np.arange(B), np.int64), support.dev_np(off, np.int64)
    _lib.check(_lib.load().igmc_node_grad_scatter(C.byref(O), B, tag_d.data_ptr(), g.data_ptr(), off_d.data_ptr(), 0,
                                                  1, out.data_ptr(),
                                                  rec[0].data_ptr(), rec[1].data_ptr(), rec[2].data_ptr(),
                                                  err.data_ptr(), _stream_ptr()), "igmc_node_grad_scatter")
    assert _take_err(err) == ERR_CANDIDATES
    got = out.cpu().numpy().view(np.int32)
    assert (got[:off[1]] == FSENT).all() and (got[off[1]:T] != FSENT).all()
