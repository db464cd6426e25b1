"""The foreign-batch builders (tests/foreign_batch_cases.py) build what they claim, their brute-force references of
igmc_batch_ptrs / igmc_batch_prepare agree with an independent formulation on every builder, and
``Batch.from_data_list`` collates per-graph ``Data`` objects into the arrays ``from_arrays`` receives.  No GPU."""
import functools

import numpy as np
import pytest
import torch

from tests import foreign_batch_cases as fb

R = 5


@functools.lru_cache(maxsize=None)
def _small():
    return fb.small(R)


@functools.lru_cache(maxsize=None)
def _ml_100k():
    return fb.ml_100k()


@functools.lru_cache(maxsize=None)
def _ml_100k_mnph100():
    return fb.ml_100k(B=16, mnph=100)


def _builders():
    return {
        "permuted": lambda: fb.permuted(_small(), 1),
        "multigraph": lambda: fb.multigraph(_small(), R, 2),
        "multigraph_B1": lambda: fb.multigraph(_small(), R, 3, graphs=[0]),
        "skewed": lambda: fb.skewed(_small(), R, graph=5, seed=4, senders=3, receivers=2, fan=2)[0],
        "staging_split": lambda: fb.staging_split(_ml_100k_mnph100(), _small(), R)[0],
        "edgeless_middle": lambda: fb.with_edgeless(_small(), 8, 5),
        "ml_100k_permuted": lambda: fb.permuted(_ml_100k(), 6),
    }


BUILDERS = list(_builders())


def _lexsort_lists(ob):
    """the lists by one numpy lexsort over (key node, type, local neighbour, edge id)"""
    ei, et, bt = np.asarray(ob["edge_index"]), np.asarray(ob["edge_type"]), np.asarray(ob["batch"])
    N, E = len(bt), ei.shape[1]
    nptr = np.concatenate([[0], np.cumsum(np.bincount(bt, minlength=int(ob["num_graphs"])))])
    out = {}
    for name, key, nbr in (("in", ei[1], ei[0]), ("out", ei[0], ei[1])):
        local = nbr - nptr[bt[nbr]]
        order = np.lexsort((np.arange(E), local, et, key))
        ptr = np.concatenate([[0], np.cumsum(np.bincount(key, minlength=N))]).astype(np.int32)
        adj = (local[order] | (et[order] << 16)).astype(np.int64).astype(np.uint32).view(np.int32)
        out[name] = (ptr, adj, order.astype(np.int32))
    return out


@pytest.mark.parametrize("name", BUILDERS)
def test_builder_claims(name):
    ob = _builders()[name]()
    B, x, bt = ob["num_graphs"], np.asarray(ob["x"]), np.asarray(ob["batch"])
    ei, et = np.asarray(ob["edge_index"]), np.asarray(ob["edge_type"])
    assert fb.grouped(ob) and np.all(np.diff(bt) >= 0) and len(ob["y"]) == B
    assert np.all(x.sum(1) == 1) and et.min(initial=0) >= 0 and et.max(initial=0) < R
    tu, ti = fb.targets(ob)
    nptr = np.concatenate([[0], np.cumsum(np.bincount(bt, minlength=B))])
    for g in range(B):      # one target of each kind, the two last nodes of their graph
        assert len(tu[g]) == 1 and len(ti[g]) == 1
        assert tu[g][0] == nptr[g + 1] - 2 and ti[g][0] == nptr[g + 1] - 1
    loops = int(np.sum(ei[0] == ei[1]))
    same, mixed = fb.parallel_pairs(ob)
    if name.startswith("multigraph"):
        assert loops >= sum((n + 2) // 3 for n in np.diff(nptr)) and same > 0 and mixed > 0
        pairs = set(zip(ei[0].tolist(), ei[1].tolist()))
        assert any((d, s) not in pairs for s, d in pairs), "no rating left with one direction"
    else:
        assert loops == 0
    if name == "edgeless_middle":
        sizes = np.diff(nptr)
        ecount = np.bincount(bt[ei[0]], minlength=B)
        assert sizes[8] == 2 and ecount[8] == 0 and B == 17
    if name == "multigraph_B1":
        assert B == 1
    if name == "ml_100k_permuted":
        assert np.diff(nptr).max() == 402
    if name == "skewed":
        _, S, T = fb.skewed(_small(), R, graph=5, seed=4, senders=3, receivers=2, fan=2)
        _check_hubs(ob, nptr, 5, S, T, 2)
    if name == "staging_split":
        _, hubs = fb.staging_split(_ml_100k_mnph100(), _small(), R)
        for g, kw in fb.SPLIT_SHAPES:
            _check_hubs(ob, nptr, g, *hubs[g], kw["fan"])


def _check_hubs(ob, nptr, g, S, T, fan):
    """senders first in graph g with an out-edge to every non-sender and no in-edge; receivers just before the two
    targets with ``fan`` in-edges from every node that is neither a sender nor a receiver, one from every sender, and
    no out-edge"""
    ei = np.asarray(ob["edge_index"])
    lo, hi = nptr[g], nptr[g + 1]
    H, K = len(S), len(T)
    assert np.array_equal(S, np.arange(lo, lo + H)) and np.array_equal(T, np.arange(hi - 2 - K, hi - 2))
    for s in S:
        assert np.sum(ei[1] == s) == 0
        assert sorted(ei[1][ei[0] == s].tolist()) == list(range(lo + H, hi))
    plain = [v for v in range(lo, hi) if v not in set(S.tolist()) | set(T.tolist())]
    for t in T:
        assert np.sum(ei[0] == t) == 0
        assert sorted(ei[0][ei[1] == t].tolist()) == sorted(S.tolist() + plain * fan)


@pytest.mark.parametrize("name", BUILDERS)
def test_references_agree(name):
    ob = _builders()[name]()
    B, bt, ei = ob["num_graphs"], np.asarray(ob["batch"]), np.asarray(ob["edge_index"])
    node_ptr, edge_ptr = fb.ptrs_reference(bt, ei[0], B)
    assert np.array_equal(node_ptr, np.searchsorted(bt, np.arange(B + 1), "left"))
    assert np.array_equal(edge_ptr, np.searchsorted(bt[ei[0]], np.arange(B + 1), "left"))
    got, want = fb.lists_reference(ei, ob["edge_type"], node_ptr), _lexsort_lists(ob)
    for side in ("in", "out"):
        for a, b in zip(got[side], want[side]):
            assert np.array_equal(a, b), side


def test_from_data_list_collates_like_from_arrays(monkeypatch):
    """per-graph Data objects through Batch.from_data_list: the arrays handed to from_arrays are the case's"""
    from igmc_b200.util_functions import Batch, Data
    ob = fb.multigraph(_small(), R, 7)
    seen = {}

    def capture(x, edge_index, edge_type, batch, y, num_graphs=None, device=None):
        seen.update(x=x, edge_index=edge_index, edge_type=edge_type, batch=batch, y=y, num_graphs=num_graphs)
        return "batch"

    monkeypatch.setattr(Batch, "from_arrays", staticmethod(capture))
    data = [Data(x=torch.from_numpy(x), edge_index=torch.from_numpy(np.ascontiguousarray(ei)),
                 edge_type=torch.from_numpy(et), y=torch.tensor([y], dtype=torch.float32))
            for x, ei, et, y in fb.split(ob)]
    assert Batch.from_data_list(data) == "batch"
    for k in ("x", "edge_index", "edge_type", "batch", "y"):
        assert np.array_equal(seen[k].numpy(), np.asarray(ob[k])), k
    assert seen["num_graphs"] == ob["num_graphs"]


def test_staging_split_enters_both_regimes():
    """host-only pin of the staging_split shape (plan queries, no GPU): on plan 2 of an R = 5 model, a CTA of graph 0
    keeps its in-entries within the forward's list capacity while even 70 % of its out-entries (the backward's, after
    the step's 20 % edge dropout) exceed the backward's; a CTA of graph 4 has 70 % of its in-entries past the
    forward's capacity and all of its out-entries within the backward's.  If list capacities are retuned and this
    fails, tests/test_gpu_foreign_batch_bounds.py's staging-split case has stopped covering the split: re-pick
    SPLIT_SHAPES."""
    import ctypes
    from igmc_b200 import _lib
    from igmc_b200.models import IGMC
    from tests.helpers import own_counts
    ob, _ = fb.staging_split(_ml_100k_mnph100(), _small(), R)
    sizes = np.bincount(np.asarray(ob["batch"]))
    n_cap = int(sizes.max())
    assert n_cap <= 256                         # no list hint: the capacities below are the plan's
    m = IGMC(4, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True)
    caps = []
    for bw in (0, 1):
        img = _lib.Stage()
        assert _lib.load().igmc_stage_plan(ctypes.byref(m._cmodel), n_cap, fb.SPLIT_PLAN, bw, ctypes.byref(img)) == 0
        caps.append(img.lcap)
    fcap, bcap = caps
    ins, outs = fb.cta_entries(ob, 0, own_counts(int(sizes[0]), fb.SPLIT_PLAN))
    assert any(i <= fcap and 0.7 * o > bcap for i, o in zip(ins, outs)), (ins, outs, caps)
    ins, outs = fb.cta_entries(ob, 4, own_counts(int(sizes[4]), fb.SPLIT_PLAN))
    assert any(0.7 * i > fcap and o <= bcap for i, o in zip(ins, outs)), (ins, outs, caps)


def test_static_store_refuses_edge_types_outside_a_byte():
    """StaticStore.from_arrays keeps one byte per edge type: a type outside 0..255 is refused on the host"""
    from igmc_b200.util_functions import StaticStore
    x = torch.zeros(2, 4)
    x[0, 0] = x[1, 1] = 1
    ei = torch.tensor([[0, 1], [1, 0]])
    for bad in (-1, 256):
        with pytest.raises(ValueError, match="edge types must lie in 0..255"):
            StaticStore.from_arrays("cpu", 4, x, ei, torch.tensor([bad, bad]), torch.ones(1),
                                    torch.tensor([0, 2]), torch.tensor([0, 2]))
