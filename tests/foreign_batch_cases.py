"""Foreign (PyG-collated) batches of shapes the subgraph extractor never builds, and brute-force references of the
batch kernels' contract (include/igmc_b200.h: igmc_batch_ptrs, igmc_batch_prepare).

Every batch the extractor writes has its target user and item at local nodes 0 and 1, each rating as two mirrored
directed edges ``[u|v ; v|u]``, no self-loop, no parallel edge and canonical edge order.  ``IGMC.forward`` on any
collated batch (``Batch.from_arrays`` / ``from_data_list``) promises nothing of the kind, so the builders here start
from extracted subgraphs (the oracle's ``extract_batch``) and take each property away, keeping what the reference's
readout needs: exactly one label-0 and one label-1 node per graph.

* ``permuted``: nodes permuted within every graph, the two targets last (owned by the last CTA of a cluster plan);
  edges renumbered and shuffled within their graph, still grouped by graph;
* ``multigraph``: before the permutation, one direction of 25 % of the ratings removed, 20 % of the edges
  duplicated (half with their own type, half with another) and a self-loop of a random type on every third node;
* ``skewed``: one graph gains sender hubs (out-edges to every other node, no in-edge), owned by its first CTA, and
  receiver hubs (parallel in-edges from every other node, no out-edge), owned by its last; ``staging_split`` sizes
  them so that one CTA's out-lists and another's in-lists leave the list buffers of a cluster plan;
* ``with_edgeless``: a 2-node graph without edges (the targets only) inserted between the others.

The fp64 oracle of the model on self-loops and parallel edges is pinned against naive loops over random multigraphs
in tests/test_relation_mean.py; this module only builds the batches and the batch-structure references."""
import numpy as np

LABEL_USER, LABEL_ITEM = 0, 1


# ---- per-graph split and collate --------------------------------------------------------------------------------
def split(ob):
    """[(x, local edge_index [2, e], edge_type [e], y)] of a collated batch dict (edges grouped by graph)"""
    x, ei, et = np.asarray(ob["x"]), np.asarray(ob["edge_index"]), np.asarray(ob["edge_type"])
    bt, y = np.asarray(ob["batch"]), np.asarray(ob["y"]).reshape(-1)
    B = int(ob["num_graphs"])
    nptr = np.concatenate([[0], np.cumsum(np.bincount(bt, minlength=B))])
    ge = bt[ei[0]] if ei.shape[1] else np.zeros(0, np.int64)
    out = []
    for g in range(B):
        sel = np.nonzero(ge == g)[0]
        out.append((x[nptr[g]:nptr[g + 1]].copy(), ei[:, sel] - nptr[g], et[sel].copy(), float(y[g])))
    return out


def collate(graphs):
    """the batch dict of per-graph (x, local edge_index, edge_type, y): PyG's offset-concat"""
    xs, eis, ets, bs, ys = [], [], [], [], []
    off = 0
    for g, (x, ei, et, y) in enumerate(graphs):
        xs.append(x)
        eis.append(np.asarray(ei, np.int64).reshape(2, -1) + off)
        ets.append(np.asarray(et, np.int64))
        bs.append(np.full(len(x), g, np.int64))
        ys.append(y)
        off += len(x)
    return dict(x=np.concatenate(xs, 0).astype(np.float32), edge_index=np.concatenate(eis, 1),
                edge_type=np.concatenate(ets), batch=np.concatenate(bs), y=np.asarray(ys, np.float32),
                num_graphs=len(graphs))


def _targets_last(x, rng):
    """new position -> old node: the non-target nodes shuffled, then the target user, then the target item"""
    lab = np.argmax(x, 1)
    tu, ti = np.nonzero(lab == LABEL_USER)[0], np.nonzero(lab == LABEL_ITEM)[0]
    assert len(tu) == 1 and len(ti) == 1
    rest = np.nonzero((lab != LABEL_USER) & (lab != LABEL_ITEM))[0]
    return np.concatenate([rng.permutation(rest), tu, ti])


def _permute_graph(x, ei, et, y, rng):
    order = _targets_last(x, rng)
    new_of_old = np.empty(len(order), np.int64)
    new_of_old[order] = np.arange(len(order))
    shuffle = rng.permutation(ei.shape[1])
    return x[order], new_of_old[ei[:, shuffle]], et[shuffle], y


def permuted(ob, seed=0):
    rng = np.random.default_rng(seed)
    return collate([_permute_graph(*g, rng) for g in split(ob)])


def _multi_graph(x, ei, et, y, R, rng):
    """one graph of the extractor's layout [u|v ; v|u] made a multigraph (see the module docstring)"""
    e = ei.shape[1]
    m = e // 2
    keep = np.ones(e, bool)
    drop = rng.choice(m, m // 4, replace=False)                      # 25 % of the ratings lose one direction
    keep[drop + m * rng.integers(0, 2, len(drop))] = False
    ei, et = ei[:, keep], et[keep]
    dup = rng.choice(ei.shape[1], ei.shape[1] // 5, replace=False)   # 20 % of the edges twice
    other = (et[dup] + rng.integers(1, R, len(dup))) % R if R > 1 else et[dup]
    dtype = np.where(np.arange(len(dup)) % 2 == 0, et[dup], other)   # half the same type, half another
    loops = np.arange(0, len(x), 3)                                  # a self-loop on every third node
    ei = np.concatenate([ei, ei[:, dup], np.stack([loops, loops])], 1)
    et = np.concatenate([et, dtype, rng.integers(0, R, len(loops))])
    return x, ei, et, y


def multigraph(ob, R, seed=0, graphs=None):
    """``graphs``: keep only these graphs (``[0]``: the B = 1 case)"""
    rng = np.random.default_rng(seed)
    parts = split(ob)
    if graphs is not None:
        parts = [parts[g] for g in graphs]
    return collate([_permute_graph(*_multi_graph(*g, R, rng), rng) for g in parts])


def skewed(ob, R, graph=0, seed=0, senders=1, receivers=1, fan=1, permute=True):
    """permuted, and graph ``graph`` gains hubs of label 3: ``senders`` sender hubs, each with one out-edge to every
    node of the graph that is not a sender and no in-edge, first in the graph's node order (the first CTA of a cluster
    plan owns them), and ``receivers`` receiver hubs, each with ``fan`` parallel in-edges from every node that is
    neither a sender nor a receiver (plus the senders' edges) and no out-edge, just before the two targets (the last
    CTA owns them).  ``permute=False`` leaves the other graphs as they are.  Returns (batch dict, sender ids, receiver
    ids) as batch-wide node ids."""
    rng = np.random.default_rng(seed)
    parts = split(ob)
    x, ei, et, y = parts[graph]
    n, H, K = len(x), int(senders), int(receivers)
    hub = np.zeros((H + K, x.shape[1]), x.dtype)
    hub[:, 3] = 1
    S, T = np.arange(n, n + H), np.arange(n + H, n + H + K)
    base, rec = np.arange(n), np.append(np.arange(n), T)
    new = [np.stack([np.full(len(rec), s), rec]) for s in S]
    new += [np.stack([np.tile(base, fan), np.full(fan * n, t)]) for t in T]
    ei = np.concatenate([ei] + new, 1)
    et = np.concatenate([et, rng.integers(0, R, sum(e.shape[1] for e in new))])
    if permute:
        parts = [_permute_graph(*g, rng) for g in parts]
    lab = np.argmax(x, 1)
    rest = np.nonzero((lab != LABEL_USER) & (lab != LABEL_ITEM))[0]
    order = np.concatenate([S, rng.permutation(rest), T, np.nonzero(lab == LABEL_USER)[0],
                            np.nonzero(lab == LABEL_ITEM)[0]])
    new_of_old = np.empty(len(order), np.int64)
    new_of_old[order] = np.arange(len(order))
    shuffle = rng.permutation(ei.shape[1])
    parts[graph] = (np.concatenate([x, hub])[order], new_of_old[ei[:, shuffle]], et[shuffle], y)
    off = sum(len(p[0]) for p in parts[:graph])
    return collate(parts), off + new_of_old[S], off + new_of_old[T]


# Two graphs whose hubs split list staging between the forward (in-lists) and the backward (out-lists) on plan 2 of
# an R = 5 model (n_cap 233, no list hint below 257 nodes; pinned on the host by tests/test_foreign_batch_cases.py):
# graph 0, a 202-node ml_100k* subgraph + 30 senders + 1 receiver, has a first CTA whose out-entries exceed the
# backward's list capacity while its in-entries stay within the forward's; graph 4, a small subgraph + 170 receivers
# fed three times by every other node, has a last CTA that owns receivers and the targets only: in-entries past the
# forward's capacity, out-entries within the backward's.
SPLIT_PLAN = 2
SPLIT_SHAPES = ((0, dict(senders=30, receivers=1, fan=1)), (4, dict(senders=0, receivers=170, fan=3)))


def staging_split(big, small_ob, R):
    """graphs 0-3 of ``big`` (ml_100k* at mnph 100, the largest graph first) and 0-3 of ``small_ob``, with the hubs of
    SPLIT_SHAPES.  Returns (batch dict, {graph: (sender ids, receiver ids)})."""
    pb = split(big)
    pb.sort(key=lambda g: -len(g[0]))
    ob = collate(pb[:4] + split(small_ob)[:4])
    hubs = {}
    for k, (g, kw) in enumerate(SPLIT_SHAPES):
        ob, S, T = skewed(ob, R, graph=g, seed=4 + g, permute=k == 0, **kw)
        hubs[g] = (S, T)
    return ob, hubs


def cta_entries(ob, g, own):
    """(in-entries, out-entries) of every CTA of graph ``g`` whose CTAs own the contiguous node counts ``own``"""
    bt, ei = np.asarray(ob["batch"]), np.asarray(ob["edge_index"])
    lo = int(np.searchsorted(bt, g))
    b = lo + np.cumsum([0] + list(own))
    ins = [int(np.sum((ei[1] >= b[r]) & (ei[1] < b[r + 1]))) for r in range(len(own))]
    outs = [int(np.sum((ei[0] >= b[r]) & (ei[0] < b[r + 1]))) for r in range(len(own))]
    return ins, outs


def with_edgeless(ob, at, seed=0):
    """permuted, with a graph of the two target nodes and no edge inserted before graph ``at``"""
    rng = np.random.default_rng(seed)
    parts = [_permute_graph(*g, rng) for g in split(ob)]
    x = np.zeros((2, np.asarray(ob["x"]).shape[1]), np.float32)
    x[0, LABEL_USER] = x[1, LABEL_ITEM] = 1
    parts.insert(at, (x, np.zeros((2, 0), np.int64), np.zeros(0, np.int64), 3.0))
    return collate(parts)


# ---- brute-force references of the header's contract ------------------------------------------------------------
def ptrs_reference(batch, edge_src, B):
    """igmc_batch_ptrs: node_ptr[b] = first node with batch id >= b, edge_ptr[b] = first edge whose source lies in a
    graph >= b (both [B + 1], ending at N and E)"""
    batch, edge_src = list(map(int, batch)), list(map(int, edge_src))
    node_ptr = [sum(1 for c in batch if c < b) for b in range(B + 1)]
    edge_ptr = [sum(1 for s in edge_src if batch[s] < b) for b in range(B + 1)]
    return np.asarray(node_ptr, np.int32), np.asarray(edge_ptr, np.int32)


def lists_reference(edge_index, edge_type, node_ptr):
    """igmc_batch_prepare: per node its in-list (edges into it) and out-list (edges out of it), entries
    (type, local neighbour, batch-wide edge id) sorted lexicographically, packed as nbr | type << 16; absolute list
    offsets with the terminal ptr[N] = E.  Returns {"in": (ptr, adj, eid), "out": (ptr, adj, eid)}."""
    src, dst = [list(map(int, r)) for r in np.asarray(edge_index).reshape(2, -1)]
    et = list(map(int, edge_type))
    N, E = int(node_ptr[-1]), len(et)
    graph_of = {}
    for g in range(len(node_ptr) - 1):
        for v in range(int(node_ptr[g]), int(node_ptr[g + 1])):
            graph_of[v] = int(node_ptr[g])
    out = {}
    for name, key, nbr in (("in", dst, src), ("out", src, dst)):
        lists = [[] for _ in range(N)]
        for e in range(E):
            lists[key[e]].append((et[e], nbr[e] - graph_of[key[e]], e))
        ptr, adj, eid = [], [], []
        for v in range(N):
            ptr.append(len(adj))
            ent = sorted(lists[v])
            adj += [n | t << 16 for t, n, _ in ent]
            eid += [e for _, _, e in ent]
        ptr.append(len(adj))
        out[name] = (np.asarray(ptr, np.int32), np.asarray(adj, np.int64).astype(np.uint32).view(np.int32),
                     np.asarray(eid, np.int32))
    return out


# ---- properties the builders claim --------------------------------------------------------------------------------
def targets(ob):
    """(target user, target item) batch-wide node id per graph"""
    lab = np.argmax(np.asarray(ob["x"]), 1)
    bt = np.asarray(ob["batch"])
    B = int(ob["num_graphs"])
    tu = [np.nonzero((bt == g) & (lab == LABEL_USER))[0] for g in range(B)]
    ti = [np.nonzero((bt == g) & (lab == LABEL_ITEM))[0] for g in range(B)]
    return tu, ti


def parallel_pairs(ob):
    """(directed pairs that occur more than once with one type, with more than one type)"""
    ei, et = np.asarray(ob["edge_index"]), np.asarray(ob["edge_type"])
    seen = {}
    for s, d, t in zip(ei[0].tolist(), ei[1].tolist(), et.tolist()):
        seen.setdefault((s, d), []).append(t)
    same = sum(1 for ts in seen.values() if len(ts) > len(set(ts)))
    mixed = sum(1 for ts in seen.values() if len(set(ts)) > 1)
    return same, mixed


def grouped(ob):
    """edges grouped by graph (sources' graphs non-decreasing) and each edge inside its source's graph"""
    ei, bt = np.asarray(ob["edge_index"]), np.asarray(ob["batch"])
    if not ei.shape[1]:
        return True
    gs, gd = bt[ei[0]], bt[ei[1]]
    return bool(np.all(np.diff(gs) >= 0) and np.all(gs == gd))


# ---- base batches (extracted subgraphs, numpy oracle) -------------------------------------------------------------
def small(R=5, B=16):
    """the oracle batch of tests/test_gpu_model.py: 16 subgraphs of a synthetic 120 x 90 matrix, mnph 30"""
    from tests.test_gpu_model import _oracle_batch
    return _oracle_batch(R=R, B=B)[3]


def ml_100k(B=16, mnph=200):
    """ml_100k* subgraphs at mnph 200: up to 402 nodes"""
    from igmc_b200.data import make_synthetic_dataset
    from oracle import extract_np
    ds = make_synthetic_dataset("ml_100k", seed=0)
    tu, tv, tl = ds["train"]
    idx = np.arange(B)
    cv = np.arange(1, 6, dtype=np.float32)
    return extract_np.extract_batch(extract_np.RatingCSR(ds["adj_train"]), tu[idx], tv[idx], tl[idx], cv, 1, 1.0,
                                    mnph, seed=3, pair_ids=idx)
