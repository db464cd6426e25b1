"""Run structure of the staged list images of the relation-space kernels (csrc/rgcn_rs.cu, stage_lists).

The gather writes every type run of a segment with one plain store, so it relies on what igmc_stage_lists encodes:
the last entry of every type run within a segment carries the RUN_END bit (bit 21), and a segment's seg_row holds the
types present in it above bit 16.  Each image built here is decoded on the host and checked against the batch's
(type, neighbour)-sorted in-lists: flags, masks and the neighbours the masked offsets decode to."""
import numpy as np
import pytest
import torch

from igmc_b200.data import build_adj, make_synthetic_dataset, synth_ratings
from tests import support
from tests.helpers import IMG_HDR, XCH, XR, own_cap_of

pytestmark = pytest.mark.gpu

ENT_OFF, RUN_END = 0x1FFFFF, 1 << 21


def _batch(A, pairs, R, mnph, B=None, seed=3):
    from igmc_b200.util_functions import MyDynamicDataset
    pu, pv, pl = [np.asarray(x, np.int64) for x in pairs]
    d = MyDynamicDataset(None, A, (pu, pv), pl, 1, 1.0, mnph, None, None, np.arange(1, R + 1, dtype=np.float32),
                         seed=seed)
    idx = np.arange(len(pu)) if B is None else np.random.default_rng(0).choice(len(pu), B, replace=False)
    return d.extract_batch(idx)


def _check_images(m, b, training):
    """decode every row of the batch's forward (and backward) list image; returns {name: staged flag per row}"""
    m._step = 7
    st = m.stage_batch(b, training, m.make_dropout(training))
    assert st is not None, "not a relation-space plan"
    torch.cuda.synchronize()
    b.check()
    p = b._priv
    n_cap = p["n_cap"]
    node_ptr = p["node_ptr"].cpu().numpy()
    _, t = b.adjacency()   # extractor batches: the batch kernel's own (symmetric) adjacency buffers
    in_ptr = (t["in_ptr"] if "in_ptr" in t else t["adj_in_ptr"]).cpu().numpy()
    in_adj = (t["in_adj"] if "in_adj" in t else t["adj_in"]).cpu().numpy().view(np.uint32)
    dropped = training and m.adj_dropout > 0
    staged_rows = {}
    for name, (img, tt) in st.items():
        cl = img.cluster
        oc = own_cap_of(n_cap, cl)
        tcap = oc + XR * XCH
        tabs, ents = tt["tab"].cpu().numpy(), tt["ent"].cpu().numpy().view(np.uint32)
        staged_rows[name] = tabs[:, 2].copy()
        for blk in range(b.num_graphs * cl):
            tab, ent = tabs[blk], ents[blk]
            total, nseg, staged, n_own = (int(x) for x in tab[:IMG_HDR])
            g, rank = divmod(blk, cl)
            nb, n = int(node_ptr[g]), int(node_ptr[g + 1] - node_ptr[g])
            lo = min(n, rank * own_cap_of(n, cl))
            assert n_own == min(n, lo + own_cap_of(n, cl)) - lo
            base = IMG_HDR
            lptr = tab[base:base + n_own + 1]
            seg0 = base + 3 * (oc + 4)
            seg_p0 = tab[seg0:seg0 + nseg]
            seg_p1 = tab[seg0 + tcap:seg0 + tcap + nseg]
            seg_row = tab[seg0 + 2 * tcap:seg0 + 2 * tcap + nseg]
            if not staged:
                assert np.all(seg_row >> 16 == 0), (name, blk)
                continue
            e = ent[:total]
            assert np.all((e >> 22) & 3 == 0), (name, blk)
            off = e & ENT_OFF
            nbr = off >> 5
            assert np.all(off & 31 == (nbr & 7) << 2), (name, blk)
            # the masked offsets decode to the node's (type, neighbour) in-list: all of it without edge dropout, a
            # subsequence (the kept entries, in order) with it
            for i in range(n_own):
                glob = in_adj[in_ptr[nb + lo + i]:in_ptr[nb + lo + i + 1]]
                want = list(zip((glob >> 16).tolist(), (glob & 0xFFFF).tolist()))
                got = list(zip((e[lptr[i]:lptr[i + 1]] >> 24).tolist(), nbr[lptr[i]:lptr[i + 1]].tolist()))
                if not dropped:
                    assert got == want, (name, blk, i)
                else:
                    it = iter(want)
                    assert all(x in it for x in got), (name, blk, i)
            covered = np.zeros(total, np.int32)
            for s in range(nseg):
                p0, p1 = int(seg_p0[s]), int(seg_p1[s])
                covered[p0:p1] += 1
                ty = (e[p0:p1] >> 24).astype(np.int64)
                flag = (e[p0:p1] & RUN_END) != 0
                want_flag = np.append(ty[1:] != ty[:-1], True) if p1 > p0 else np.zeros(0, bool)
                assert np.array_equal(flag, want_flag), (name, blk, s)
                assert flag.sum() == len(set(ty.tolist())), (name, blk, s)   # every type is one run
                assert int(seg_row[s]) >> 16 == int(np.bitwise_or.reduce(1 << ty, initial=0)), (name, blk, s)
            assert np.all(covered == 1), (name, blk)
    return staged_rows


def test_run_flags_ml_1m():
    """ml_1m*, batch 50, mnph 100: the flagship workload's images, train step with and without edge dropout"""
    ds = make_synthetic_dataset("ml_1m", seed=0)
    b = _batch(ds["adj_train"], ds["train"], 5, 100, B=50)
    for p in (0.0, 0.2):
        staged = _check_images(support.model(5, adj_dropout=p), b, True)
        assert staged["fwd"].all() and staged["bwd"].all()


def test_run_flags_ml_100k_dropout():
    """ml_100k*, mnph 200, edge dropout 0.2: compacted kept lists"""
    ds = make_synthetic_dataset("ml_100k", seed=0)
    b = _batch(ds["adj_train"], ds["train"], 5, 200, B=50)
    staged = _check_images(support.model(5, adj_dropout=0.2), b, True)
    assert staged["fwd"].any()


def test_run_flags_twelve_relations():
    """R = 12 (the largest type mask), synthetic ratings, train step and eval images"""
    u, v, lab = synth_ratings(400, 300, 9000, num_classes=12, seed=5)
    A = build_adj(u, v, lab, 400, 300)
    b = _batch(A, (u, v, lab), 12, 60, B=40)
    m = support.model(12, adj_dropout=0.2)
    _check_images(m, b, True)
    _check_images(m, b, False)


def test_unstaged_lists_carry_no_masks():
    """a dense 101 x 101 block at plan 2 (n_cap 202): the backward's lists exceed its capacity and are not staged
    (the kernel then reads the global lists); their segment rows carry no type mask, the staged forward's do"""
    rng = np.random.default_rng(3)
    bu, bv = np.nonzero(rng.random((101, 101)) < 1.1)
    bl = rng.integers(0, 5, len(bu))
    su, sv, sl = synth_ratings(200, 200, 3000, num_classes=5, seed=4)
    u, v, lab = np.concatenate([bu, su + 101]), np.concatenate([bv, sv + 101]), np.concatenate([bl, sl])
    A = build_adj(u, v, lab, 301, 301)
    blk = np.nonzero((u < 101) & (v < 101))[0]
    bg = np.nonzero(u >= 101)[0]
    pick = np.array([blk[17], bg[0], blk[5000], bg[1]])
    b = _batch(A, (u[pick], v[pick], lab[pick]), 5, 100)
    assert b._priv["n_cap"] == 202
    m = support.model(5, adj_dropout=0.2)
    m.kernel_plan = 2
    staged = _check_images(m, b, True)
    assert np.any((staged["fwd"] == 1) & (staged["bwd"] == 0)), "no CTA with staged forward and global backward lists"
