"""Batches for the node explanation kernels (csrc/explain.cu: igmc_explain_node_count, igmc_node_occlusion_mask,
igmc_node_grad_scatter) and their brute-force enumeration, written from the header's contract.

A batch is a list of subgraphs in the extractor's layout: per graph its users (target first) then its items (target
first), node_label 0 / 1 on the targets and 2d / 2d + 1 on a user / item at distance d <= h, edge_index
[u|v ; v|u] with batch node ids, and per node the in-list of its in-edges sorted by (type, neighbour).  Graphs cover a
subgraph with only its targets, nodes with one rating and with many, an isolated non-target node, h = 2 labels and a
graph of more than one chunk (MASK_THREADS) of nodes."""
import numpy as np

MASK_THREADS = 256     # csrc/explain.cu: `constexpr int MASK_THREADS`, the chunk of foreach_position


def _graph(rng, nu, ni, density, h, R, isolated=False):
    """one subgraph: (labels [n], gids [n], ratings [(user, item, type)] with graph-local node ids)"""
    lab = np.empty(nu + ni, np.int64)
    lab[0], lab[nu] = 0, 1
    lab[1:nu] = 2 * rng.integers(1, h + 1, nu - 1)
    lab[nu + 1:] = 2 * rng.integers(1, h + 1, ni - 1) + 1
    gid = np.concatenate([rng.choice(10 ** 6, nu, replace=False), rng.choice(10 ** 6, ni, replace=False)])
    ratings = []
    for a in range(nu):
        for b in range(ni):
            if (a, b) == (0, 0) or (isolated and (a == nu - 1 or b == ni - 1)):
                continue
            # every non-target node keeps a rating to a target so that it belongs to the subgraph
            if rng.random() < density or (a == 0 and b > 0) or (b == 0 and a > 0):
                ratings.append((a, nu + b, int(rng.integers(0, R))))
    return lab, gid, ratings


def make_batch(seed, shapes, h=1, R=5):
    """``shapes``: per graph (users, items, density, isolated).  Returns numpy arrays node_ptr, edge_ptr, src, dst,
    edge_type, node_label, node_gid, in_ptr, in_eid and the per-graph ratings counts"""
    rng = np.random.default_rng(seed)
    node_ptr, edge_ptr = [0], [0]
    src, dst, et, lab, gid = [], [], [], [], []
    for nu, ni, dens, iso in shapes:
        l, g, rs = _graph(rng, nu, ni, dens, h, R, iso)
        rng.shuffle(rs)
        n0 = node_ptr[-1]
        u = [n0 + a for a, _, _ in rs]
        v = [n0 + b for _, b, _ in rs]
        t = [r for _, _, r in rs]
        src += u + v
        dst += v + u
        et += t + t
        lab.append(l)
        gid.append(g)
        node_ptr.append(n0 + len(l))
        edge_ptr.append(edge_ptr[-1] + 2 * len(rs))
    src, dst, et = (np.asarray(a, np.int64) for a in (src, dst, et))
    N = node_ptr[-1]
    in_ptr = np.zeros(N + 1, np.int64)
    in_eid = []
    for n in range(N):
        e = np.flatnonzero(dst == n)
        e = e[np.lexsort((src[e], et[e]))]          # by (type, neighbour)
        in_eid += e.tolist()
        in_ptr[n + 1] = len(in_eid)
    return dict(node_ptr=np.asarray(node_ptr, np.int64), edge_ptr=np.asarray(edge_ptr, np.int64), src=src, dst=dst,
                edge_type=et, node_label=np.concatenate(lab).astype(np.uint8), node_gid=np.concatenate(gid),
                in_ptr=in_ptr, in_eid=np.asarray(in_eid, np.int64))


SHAPES = {
    # name: (per graph (users, items, density, isolated), h)
    "one rating and many": ([(4, 5, 0.0, False), (6, 3, 0.7, False), (1, 1, 0.0, False), (3, 8, 0.3, False)], 1),
    "only targets": ([(1, 1, 0.0, False), (1, 1, 0.0, False)], 1),
    "isolated node": ([(4, 4, 0.5, True), (2, 3, 0.5, False)], 1),
    "h=2 labels": ([(5, 7, 0.3, False), (7, 4, 0.4, False)], 2),
    "chunk boundaries": ([(150, 160, 0.01, False), (3, 2, 0.5, False), (1, 300, 0.0, False)], 1),
}


def positions(bt, g):
    """the batch node ids of graph g's positions: its nodes with node_label >= 2, in order"""
    return [n for n in range(bt["node_ptr"][g], bt["node_ptr"][g + 1]) if bt["node_label"][n] >= 2]


def mask_brute(bt, g, j):
    """(the directed edges of graph g that the mask drops, the node's (gid, label, ratings)) for position j, or
    (empty, None) for a j outside the graph's positions"""
    pos = positions(bt, g)
    if not 0 <= j < len(pos):
        return [], None
    p = pos[j]
    drop = [e for e in range(bt["edge_ptr"][g], bt["edge_ptr"][g + 1]) if bt["src"][e] == p or bt["dst"][e] == p]
    ratings = sum(1 for e in range(bt["edge_ptr"][g], bt["edge_ptr"][g + 1]) if bt["src"][e] == p)
    return drop, (int(bt["node_gid"][p]), int(bt["node_label"][p]), ratings)


def grad_brute(bt, g, edge_grad):
    """per position of graph g: the float32 sum, in the node's in-list order, of each rating's user -> item edge
    gradient plus its item -> user edge gradient (the first rating's value as it is), and the node's record"""
    e0, m = int(bt["edge_ptr"][g]), int(bt["edge_ptr"][g + 1] - bt["edge_ptr"][g]) // 2
    vals, recs = [], []
    for p in positions(bt, g):
        lst = bt["in_eid"][bt["in_ptr"][p]:bt["in_ptr"][p + 1]]
        v = np.float32(0)
        for t, e in enumerate(lst):
            a = e if e < e0 + m else e - m          # the user -> item copy
            assert bt["src"][a] == bt["dst"][a + m] and bt["dst"][a] == bt["src"][a + m]
            r = np.float32(np.float32(edge_grad[a]) + np.float32(edge_grad[a + m]))
            v = r if t == 0 else np.float32(v + r)
        vals.append(v)
        recs.append((int(bt["node_gid"][p]), int(bt["node_label"][p]), len(lst)))
    return np.asarray(vals, np.float32), recs
