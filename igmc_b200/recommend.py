"""Score unrated (user, item) pairs and recommend the top-k items per user on the fused kernels.

IGMC is inductive: it scores any (user, item) pair from the pair's enclosing subgraph.  The reference only reduces
predictions to an RMSE over a labelled dataset (train_eval.py:182-245); ranking the items a user has not rated means
building a dataset of every candidate pair and looping over it in Python.  Here:

* ``predict_pairs(model, graph, users, items)`` -> fp32 scores of the explicit pairs ``(users[i], items[i])``;
* ``recommend(model, graph, users, k)`` -> per query user the ``k`` best candidate items and their scores (candidates:
  ``items``, per-user lists ``items[U, width]``, the retriever's ``retrieve=M`` items or every item, without the
  user's rated items when ``exclude_rated``), ranked by score descending, then item ascending; a NaN score ranks
  last; missing slots hold item -1 and score -inf;
* ``corated_items(graph, users, m)`` -> per query user the ``m`` items with the most bridges (3-paths u - i - u' - v,
  ``igmc_corated_items``): the cheap first stage that proposes each user's candidates for the model to rank;
* ``explain_pairs(model, graph, users, items, m)`` -> per pair its score and, for every rating in its enclosing
  subgraph, the score change from removing that rating (csrc/explain.cu): a base pass of the pairs, then an occlusion
  pass over (pair, rating) positions whose batches carry an edge mask into a training-mode forward without dropout;
* ``attribute_pairs(model, graph, users, items, m)`` -> the same layout with, per rating, the score's gradient with
  respect to a weight on that rating (igmc_edge_grad): the same base pass, then one gradient pass over the P pairs, each
  an L2-plan eval forward and one backward whose list walk writes every edge's term;
* ``InferenceEngine``: the pipelined, graph-replayed loop behind all of them.  Per step the side stream produces the next
  batch's candidate pairs (``igmc_candidate_pairs``, from a device cursor) and extracts it while the main stream runs
  the eval forward of the current batch (once per checkpoint) and merges its scores into the running per-user top-k
  lists (``igmc_topk_merge``) or scatters them to their pair index (``igmc_score_scatter``).  The step is one CUDA graph
  per batch slot, captured after an eager warm-up; between steps there is no host copy and no host synchronisation.

Every pair samples its subgraph with ``pair_id = u * num_items + v``: its subgraph, and so its score, does not depend on
the API that scored it, the batch it fell into or the candidate list.  The host twins below restate the kernels'
integer arithmetic for the CPU tests (tests/test_recommend_host.py).
"""
import collections
import contextlib
import ctypes as C

import numpy as np
import torch

from . import _lib
from .train_eval import replay_step
from .util_functions import RatingGraph, SubgraphExtractor, _stream_ptr

__all__ = ["predict_pairs", "recommend", "corated_items", "explain_pairs", "Explanation", "attribute_pairs",
           "Attribution", "InferenceEngine"]


# ---- input validation (host) ----------------------------------------------------------------------------------------
def _host_ids(a, name, hi):
    """ids as a host int64 vector (device tensors: one copy to the host), each in [0, hi) or IndexError"""
    if torch.is_tensor(a):
        a = a.detach().cpu().numpy()
    a = np.asarray(a).reshape(-1)
    if a.size == 0:
        return np.zeros(0, np.int64)
    if not np.issubdtype(a.dtype, np.integer):
        raise TypeError("%s must be integer ids, not %s" % (name, a.dtype))
    a = a.astype(np.int64)
    lo, top = int(a.min()), int(a.max())
    if lo < 0 or top >= hi:
        raise IndexError("%s: id %d out of range [0, %d)" % (name, lo if lo < 0 else top, hi))
    return a


def _is_rows(items):
    """a 2-D ``items`` names per-user candidate lists"""
    return items is not None and (items.dim() == 2 if torch.is_tensor(items) else np.ndim(items) == 2)


def _user_rows(items, U, num_items, dev):
    """per-user candidate rows [U, width] as an int32 device tensor.  Host arrays are checked here (IndexError for an
    id outside [-1, num_items)); integer device tensors are used as they are and checked by the kernel.  ValueError
    when the row count is not U."""
    if not torch.is_tensor(items):
        items = np.asarray(items)
    if items.shape[0] != U:
        raise ValueError("items has %d rows, one per query user is %d" % (items.shape[0], U))
    if torch.is_tensor(items) and items.device.type == "cuda":
        if items.is_floating_point() or items.is_complex() or items.dtype == torch.bool:
            raise TypeError("items must be integer ids, not %s" % items.dtype)
        return items.to(device=dev, dtype=torch.int32).contiguous()
    a = np.asarray(items.cpu().numpy() if torch.is_tensor(items) else items)
    if a.size and not np.issubdtype(a.dtype, np.integer):
        raise TypeError("items must be integer ids, not %s" % a.dtype)
    a = a.astype(np.int64)
    if a.size and (a.min() < -1 or a.max() >= num_items):
        bad = int(a.min()) if a.min() < -1 else int(a.max())
        raise IndexError("items: id %d out of range [-1, %d)" % (bad, num_items))
    return torch.from_numpy(a.astype(np.int32)).to(dev)


def _check_m(m, num_items):
    m = int(m)
    if m < 1 or m > num_items:
        raise ValueError("the number of retrieved items must lie in [1, %d], not %d" % (num_items, m))
    return m


def _corated(lib, g, users, m, exclude_rated, err, ws):
    """igmc_corated_items for the int32 device tensor ``users`` on graph ``g``: (items, paths) [U, m] int32.  ``ws``: a
    dict whose "ws" tensor is grown to the workspace the shape needs"""
    U, dev = int(users.numel()), g.device
    nbytes = C.c_int64(0)
    _lib.check(lib.igmc_corated_ws_bytes(g.num_users, g.num_items, U, m, C.byref(nbytes)), "igmc_corated_ws_bytes")
    if ws.get("ws") is None or ws["ws"].numel() < nbytes.value:
        ws["ws"] = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    items = torch.empty(U, m, dtype=torch.int32, device=dev)
    paths = torch.empty(U, m, dtype=torch.int32, device=dev)
    _lib.check(lib.igmc_corated_items(C.byref(g._c), users.data_ptr(), U, m, int(bool(exclude_rated)),
                                      ws["ws"].data_ptr(), ws["ws"].numel(), items.data_ptr(), paths.data_ptr(),
                                      err.data_ptr(), _stream_ptr()), "igmc_corated_items")
    return items, paths


def _check_k(k):
    k = int(k)
    if k < 1:
        raise ValueError("k must be >= 1, not %d" % k)
    if k > _lib.TOPK_MAX:
        raise NotImplementedError("the top-k merge kernel keeps at most k = %d items per user" % _lib.TOPK_MAX)
    return k


def _check_top(m, name):
    """None, or a count in [1, IGMC_TOPK_MAX] of entries to keep per pair"""
    if m is None:
        return None
    m = int(m)
    if m < 1:
        raise ValueError("%s must be >= 1, not %d" % (name, m))
    if m > _lib.TOPK_MAX:
        raise NotImplementedError("an explanation keeps at most %s = %d ratings per pair" % (name, _lib.TOPK_MAX))
    return m


# The result of explain_pairs, device tensors: score [P] fp32 (= predict_pairs), num_edges [P] int32 (the ratings of
# each pair's subgraph), offsets [P+1] int64 (their exclusive prefix) and, per rating, user / item / rating int32 and
# delta fp32 (score without the rating - score): flat [offsets[P]] with pair p at [offsets[p], offsets[p+1]), or
# [P, m] padded with -1 / -1 / -1 / 0.
Explanation = collections.namedtuple("Explanation", "score num_edges offsets user item rating delta")

# The result of attribute_pairs: Explanation's layout and order with grad (d score / d m_e, the rating's weight m_e at
# m = 1) in place of delta.  -grad is the first-order estimate of explain_pairs' delta.
Attribution = collections.namedtuple("Attribution", "score num_edges offsets user item rating grad")


# ---- host twins of the candidate and merge kernels (csrc/recommend.cu) ----------------------------------------------
def candidate_plan_host(row_ptr, col_idx, num_items, users, cand=None, exclude_rated=True):
    """twin of igmc_candidate_plan: (user_off [U+1], rated_off [U+1] or None, rated_pos or None)"""
    users = np.asarray(users, np.int64)
    U = len(users)
    deg = np.asarray(row_ptr[users + 1] - row_ptr[users], np.int64) if U else np.zeros(0, np.int64)
    lists = cand is not None and exclude_rated
    rated_pos = []
    if cand is None:
        cnt = num_items - deg if exclude_rated else np.full(U, num_items, np.int64)
    elif not exclude_rated:
        cnt = np.full(U, len(cand), np.int64)
    else:
        cand = np.asarray(cand, np.int64)
        hits = np.zeros(U, np.int64)
        for j, u in enumerate(users):
            row = np.asarray(col_idx[row_ptr[u]:row_ptr[u + 1]], np.int64)
            p = np.searchsorted(cand, row)
            found = (p < len(cand)) & (cand[np.minimum(p, max(len(cand) - 1, 0))] == row) if len(cand) else \
                np.zeros(len(row), bool)
            rated_pos.append(p[found])
            hits[j] = int(found.sum())
        cnt = len(cand) - hits
    user_off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    if not lists:
        return user_off, None, None
    rated_off = np.concatenate([[0], np.cumsum([len(r) for r in rated_pos])]).astype(np.int64)
    return user_off, rated_off, (np.concatenate(rated_pos) if rated_pos else np.zeros(0, np.int64)).astype(np.int64)


def candidate_pairs_host(row_ptr, col_idx, num_items, users, cand, exclude_rated, plan, pos, B):
    """twin of igmc_candidate_pairs for global positions [pos, pos + B): (links_u, links_v, pair_id, tag)"""
    user_off, rated_off, rated_pos = plan
    P = int(user_off[-1])
    out = np.zeros((4, B), np.int64)
    for i in range(B):
        g = pos + i
        real = g < P
        if not real:
            g = P - 1
        j = int(np.searchsorted(user_off, g, side="right")) - 1      # the last j with user_off[j] <= g
        j = min(j, len(users) - 1)
        c = g - int(user_off[j])
        u = int(users[j])
        p = c
        if exclude_rated:
            r = rated_pos[rated_off[j]:rated_off[j + 1]] if cand is not None else col_idx[row_ptr[u]:row_ptr[u + 1]]
            r = np.asarray(r, np.int64)
            p = c + int(np.count_nonzero(r - np.arange(len(r)) <= c))
        v = int(cand[p]) if cand is not None else p
        out[:, i] = (u, v, u * num_items + v, j if real else -1)
    return out


def _before(a_s, a_i, b_s, b_i):
    """the ranking order of igmc_topk_merge: score descending, item ascending, NaN last, empty slots (item < 0) after
    everything"""
    if a_i < 0:
        return False
    if b_i < 0:
        return True
    an, bn = np.isnan(a_s), np.isnan(b_s)
    if an or bn:
        return a_i < b_i if (an and bn) else bool(bn)
    return a_s > b_s or (a_s == b_s and a_i < b_i)


def topk_merge_host(top_s, top_i, seg_s, seg_i):
    """twin of one CTA of igmc_topk_merge: the running list (k, ranked) merged with one segment of new candidates by
    rank counting; returns the new (scores, items)"""
    k = len(top_s)
    S = list(np.asarray(top_s, np.float32)) + list(np.asarray(seg_s, np.float32))
    It = list(np.asarray(top_i, np.int64)) + list(np.asarray(seg_i, np.int64))
    out_s, out_i = np.array(top_s, np.float32), np.array(top_i, np.int64)
    for e in range(len(S)):
        if e < k:
            r = e
        else:
            r = sum(1 for o in range(k) if _before(S[o], It[o], S[e], It[e]))
        r += sum(1 for x in range(k, len(S)) if x != e and _before(S[x], It[x], S[e], It[e]))
        if r < k:
            out_s[r], out_i[r] = S[e], It[e]
    return out_s, out_i


def corated_host(row_ptr, col_idx, num_users, num_items, users, m, exclude_rated=True):
    """twin of igmc_corated_items: per query user the ``m`` items with the most bridges, paths[v] = sum over u' != u
    of |N(u) & N(u')| * [u' rated v] (B B^T B without the u' = u term), ordered by paths descending then item
    ascending, items without a bridge dropped; (items [U, m], paths [U, m]) int32 padded with -1 / 0"""
    import scipy.sparse as ssp
    users = np.asarray(users, np.int64).reshape(-1)
    rp = np.asarray(row_ptr, np.int64)
    nnz = int(rp[num_users])
    Bm = ssp.csr_matrix((np.ones(nnz, np.int64), np.asarray(col_idx[:nnz], np.int64), rp[:num_users + 1]),
                        shape=(num_users, num_items))
    Bu = Bm[users]                                           # [U, ni]
    W = (Bu @ Bm.T).toarray()                                # |N(u) & N(u')|
    W[np.arange(len(users)), users] = 0                      # u' != u
    P = W @ Bm                                               # [U, ni] (dense @ sparse: dense)
    P = np.asarray(P, np.int64)
    if exclude_rated:
        P[Bu.toarray() > 0] = 0
    items = np.full((len(users), m), -1, np.int32)
    paths = np.zeros((len(users), m), np.int32)
    for j in range(len(users)):
        o = np.argsort(-P[j], kind="stable")[:m]            # paths descending, then item ascending
        o = o[P[j][o] > 0]
        items[j, :len(o)], paths[j, :len(o)] = o, P[j][o]
    return items, paths


def candidate_lists_host(row_ptr, col_idx, num_items, users, rows, exclude_rated=True):
    """twin of igmc_candidate_lists: (user_off [U+1] int64, lists) - per query slot its row sorted, deduplicated, -1
    slots dropped and (exclude_rated) the user's rated items removed"""
    users = np.asarray(users, np.int64).reshape(-1)
    rows = np.asarray(rows, np.int64).reshape(len(users), -1)
    out = []
    for j, u in enumerate(users):
        r = np.unique(rows[j])
        r = r[(r >= 0) & (r < num_items)]
        if exclude_rated:
            r = r[~np.isin(r, np.asarray(col_idx[row_ptr[u]:row_ptr[u + 1]], np.int64))]
        out.append(r)
    user_off = np.concatenate([[0], np.cumsum([len(r) for r in out])]).astype(np.int64)
    return user_off, (np.concatenate(out) if out else np.zeros(0, np.int64)).astype(np.int32)


def rank_host(scores, items, k):
    """brute-force ranking: the first ``k`` of ``items`` by (score descending, item ascending, NaN last), padded
    with (-1, -inf)"""
    scores, items = np.asarray(scores, np.float32), np.asarray(items, np.int64)
    o = np.argsort(items, kind="stable")
    o = o[np.argsort(-scores[o], kind="stable")]          # numpy sorts NaN last
    top_i = np.full(k, -1, np.int64)
    top_s = np.full(k, -np.inf, np.float32)
    n = min(k, len(o))
    top_i[:n], top_s[:n] = items[o[:n]], scores[o[:n]]
    return top_s, top_i


# ---- host twins of the explanation kernels (csrc/explain.cu) --------------------------------------------------------
def explain_offsets_host(num_edges):
    """twin of igmc_explain_offsets: the exclusive int64 prefix [P+1] of the per-pair rating counts"""
    return np.concatenate([[0], np.cumsum(np.asarray(num_edges, np.int64))]).astype(np.int64)


def occlusion_pairs_host(offsets, pair_u, pair_v, num_items, pos, B):
    """twin of igmc_occlusion_pairs for positions [pos, pos + B): (links_u, links_v, pair_id, tag, edge_j)"""
    offsets = np.asarray(offsets, np.int64)
    P, T = len(offsets) - 1, int(offsets[-1])
    out = np.zeros((5, B), np.int64)
    for i in range(B):
        c = pos + i
        real = c < T
        if not real:
            c = T - 1
        q = min(int(np.searchsorted(offsets, c, side="right")) - 1, P - 1)     # the last q with offsets[q] <= c
        u, v = int(pair_u[q]), int(pair_v[q])
        out[:, i] = (u, v, u * num_items + v, c if real else -1, c - offsets[q])
    return out


def occlusion_mask_host(edge_ptr, tag, edge_j):
    """twin of igmc_occlusion_mask's edge_keep [edge_ptr[B]]: graph g with tag >= 0 drops its directed edges
    edge_ptr[g] + j and edge_ptr[g] + E_g/2 + j"""
    edge_ptr = np.asarray(edge_ptr, np.int64)
    keep = np.ones(int(edge_ptr[-1]), np.uint8)
    for g in range(len(edge_ptr) - 1):
        m = int(edge_ptr[g + 1] - edge_ptr[g]) // 2
        if tag[g] >= 0 and 0 <= edge_j[g] < m:
            keep[edge_ptr[g] + edge_j[g]] = keep[edge_ptr[g] + m + edge_j[g]] = 0
    return keep


def explain_order_host(score, occluded, offsets, m=None):
    """twin of igmc_occlusion_order's permutation: (delta [T] fp32, order) where order is, per pair q, the positions of
    its segment by |delta| descending, NaN after every number, ties by j - flat [T] (m None) or [P, m] padded with -1.
    ``score`` None: delta = occluded (attribution gradients)"""
    occluded = np.asarray(occluded, np.float32)
    offsets = np.asarray(offsets, np.int64)
    P = len(offsets) - 1
    q = np.repeat(np.arange(P), np.diff(offsets))
    delta = occluded.copy() if score is None else (occluded - np.asarray(score, np.float32)[q]).astype(np.float32)
    order = []
    for p in range(P):
        seg = np.arange(offsets[p], offsets[p + 1])
        a = np.abs(delta[seg])
        o = np.lexsort((seg, np.where(np.isnan(a), np.inf, -a), np.isnan(a)))    # NaN last, |delta| desc, then j
        order.append(seg[o])
    if m is None:
        return delta, (np.concatenate(order) if order else np.zeros(0, np.int64)).astype(np.int64)
    top = np.full((P, m), -1, np.int64)
    for p, o in enumerate(order):
        top[p, :min(m, len(o))] = o[:m]
    return delta, top


def edge_grad_scatter_host(edge_ptr, tag, edge_grad, offsets, out, k=0, K=1):
    """twin of igmc_edge_grad_scatter's values for checkpoint ``k`` of ``K``: graph g with tag q >= 0 writes rating j's
    edge_grad[e0 + j] + edge_grad[e0 + E_g/2 + j] to out[offsets[q] + j] (k = 0), or adds it (k > 0), then divides by
    K (k = K - 1); fp32 throughout.  ``out`` [T] is updated in place and returned"""
    edge_ptr, offsets = np.asarray(edge_ptr, np.int64), np.asarray(offsets, np.int64)
    edge_grad = np.asarray(edge_grad, np.float32)
    for g in range(len(edge_ptr) - 1):
        q = int(tag[g])
        if q < 0:
            continue
        e0, m = int(edge_ptr[g]), int(edge_ptr[g + 1] - edge_ptr[g]) // 2
        v = edge_grad[e0:e0 + m] + edge_grad[e0 + m:e0 + 2 * m]
        o = int(offsets[q])
        if k > 0:
            v = out[o:o + m] + v
        if k == K - 1:
            v = v / np.float32(K)
        out[o:o + m] = v
    return out


# ---- the engine -----------------------------------------------------------------------------------------------------
class InferenceEngine(object):
    """Pipelined, graph-replayed scoring of candidate pairs (module docstring).  ``checkpoints``: state_dict files of
    ``model``'s class, each scored and averaged (fp32 sum in checkpoint order / K); None scores ``model``'s own
    parameters as they are when a run starts.

        eng = InferenceEngine(model, graph, batch_size=256)
        eng.start_recommend(users, k)          # or start_pairs(users, items) / start_explain / start_attribute(users, items, m)
        while eng.step():
            pass
        top_items, top_scores = eng.finish()   # (predict: scores; explain: an Explanation; attribute: an Attribution)

    An engine serves across updates of its ``RatingGraph`` (``graph.update``) between runs; an update during a run
    makes its next ``step`` raise RuntimeError.
    """

    def __init__(self, model, graph, h=1, sample_ratio=1.0, max_nodes_per_hop=None, batch_size=256,
                 checkpoints=None, sample_seed=0, use_graph=True):
        dev = model.flat_params.device
        if dev.type != "cuda":
            raise RuntimeError("igmc_b200 inference needs the model on a CUDA device (there is no CPU path)")
        if model.num_features != 2 * int(h) + 2:
            raise ValueError("the model takes %d node features, hop %d extraction gives %d"
                             % (model.num_features, int(h), 2 * int(h) + 2))
        self.B = int(batch_size)
        if self.B < 1:
            raise ValueError("batch_size must be >= 1")
        self.lib = _lib.load()
        self.model, self.dev, self.use_graph = model, dev, bool(use_graph)
        self.graph = graph if isinstance(graph, RatingGraph) else RatingGraph(graph, dev)
        if self.graph.device is None or self.graph.device != dev:
            self.graph.to(dev)
        R = model.num_relations
        self.extractor = SubgraphExtractor(self.graph, [0], [0], [0], np.arange(1, R + 1, dtype=np.float32), h,
                                           sample_ratio, max_nodes_per_hop, max_batch=self.B, seed=sample_seed)
        self.drop = model.make_dropout(False)        # eval: no edge dropout, no hidden dropout
        if checkpoints:
            own = model.flat_params.clone()
            self.params = []
            for path in checkpoints:
                model.load_state_dict(torch.load(path, map_location=dev))
                self.params.append(model.flat_params.clone())
            with torch.no_grad():
                model.flat_params.copy_(own)
            model._prepped = False
        else:
            self.params = [model.flat_params]
        self.K = len(self.params)
        self.wprep = [torch.zeros_like(model._wprep_buf()) for _ in range(self.K)]
        i32, i64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.int64, device=dev)
        self.cursor = torch.zeros(1, **i64)
        # per batch slot: the candidate pairs igmc_extract_batch reads (idx = NULL) and their query slot / pair index
        self.slots = [dict(u=torch.zeros(self.B, **i32), v=torch.zeros(self.B, **i32), pid=torch.zeros(self.B, **i64),
                           tag=torch.zeros(self.B, **i64)) for _ in range(2)]
        self.preds = torch.zeros(self.K, self.B, dtype=torch.float32, device=dev)
        self.side = torch.cuda.Stream(dev)
        self.run = None
        self._retrieve_ws = {}       # the retriever's workspace when its histograms do not fit in shared memory
        self._grad_plans = {}        # the model's plan cache while a gradient pass forces the L2 plan

    # ---- one run: plan, prime, steps, finish --------------------------------------------------------------------
    def start_recommend(self, users, k, items=None, exclude_rated=True, retrieve=None):
        """plan a ranking run (one host sync: the candidate total).  ``items``: one candidate list for every user, or
        a 2-D [U, width] array of per-user lists (-1 = empty slot); ``retrieve=M``: each user's M items with the most
        bridges (``corated_items``) are its candidates.  Returns the number of candidate pairs."""
        k = _check_k(k)
        g = self.graph
        if retrieve is not None and items is not None:
            raise ValueError("retrieve= chooses the candidates itself: pass it without items=")
        per_user = retrieve is not None or _is_rows(items)
        m = None if retrieve is None else _check_m(retrieve, g.num_items)
        users = _host_ids(users, "users", g.num_users)
        cand = None if items is None or per_user else np.unique(_host_ids(items, "items", g.num_items))
        U, dev = len(users), self.dev
        rows = _user_rows(items, U, g.num_items, dev) if per_user and m is None else None
        run = dict(kind="recommend", U=U, k=k, version=g.version,
                   top_s=torch.full((U, k), -float("inf"), dtype=torch.float32, device=dev),
                   top_i=torch.full((U, k), -1, dtype=torch.int64, device=dev))
        self.run = run
        if U == 0 or (cand is not None and len(cand) == 0) or (rows is not None and rows.shape[1] == 0):
            run["P"] = 0
            return 0
        i64 = dict(dtype=torch.int64, device=dev)
        run["users"] = torch.from_numpy(users.astype(np.int32)).to(dev)
        if per_user:
            return self._plan_lists(run, rows, m, exclude_rated)
        run["cand"] = None if cand is None else torch.from_numpy(cand.astype(np.int32)).to(dev)
        run["user_off"] = torch.zeros(U + 1, **i64)
        lists = cand is not None and bool(exclude_rated)
        if lists:
            rp = g.host["row_ptr"]
            run["rated_off"] = torch.zeros(U + 1, **i64)
            run["rated_pos"] = torch.zeros(max(int((rp[users + 1] - rp[users]).sum()), 1), dtype=torch.int32,
                                           device=dev)
        Cd = _lib.Candidates()
        Cd.users, Cd.cand = run["users"].data_ptr(), _lib.ptr(run["cand"])
        Cd.user_off = run["user_off"].data_ptr()
        Cd.rated_off, Cd.rated_pos = _lib.ptr(run.get("rated_off")), _lib.ptr(run.get("rated_pos"))
        Cd.num_query, Cd.num_cand = U, 0 if cand is None else len(cand)
        Cd.exclude_rated = int(bool(exclude_rated))
        _lib.check(self.lib.igmc_candidate_plan(C.byref(g._c), C.byref(Cd), self.extractor.err.data_ptr(),
                                                _stream_ptr()), "igmc_candidate_plan")
        Cd.num_pairs = run["P"] = int(run["user_off"][U].item())
        run["Cd"] = Cd
        if run["P"] > 0:
            self._prime()
        return run["P"]

    def _plan_lists(self, run, rows, m, exclude_rated):
        """the plan of a run over per-user candidate rows (``rows``, or the retriever's top ``m`` per user):
        igmc_candidate_lists compacts them into run["lists"] and user_off"""
        g, U, dev = self.graph, run["U"], self.dev
        err = self.extractor.err
        if rows is None:
            rows, _ =_corated(self.lib, g, run["users"], m, exclude_rated, err, self._retrieve_ws)
        width = int(rows.shape[1])
        run["rows"] = rows
        run["lists"] = torch.empty(max(U * width, 1), dtype=torch.int32, device=dev)
        run["user_off"] = torch.zeros(U + 1, dtype=torch.int64, device=dev)
        nbytes = C.c_int64(0)
        _lib.check(self.lib.igmc_candidate_lists_ws_bytes(U, width, C.byref(nbytes)), "igmc_candidate_lists_ws_bytes")
        run["lists_ws"] = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
        Cd = _lib.Candidates()
        Cd.users, Cd.user_off = run["users"].data_ptr(), run["user_off"].data_ptr()
        Cd.num_query, Cd.exclude_rated = U, int(bool(exclude_rated))
        _lib.check(self.lib.igmc_candidate_lists(C.byref(g._c), C.byref(Cd), rows.data_ptr(), width,
                                                 run["lists"].data_ptr(), run["lists_ws"].data_ptr(),
                                                 run["lists_ws"].numel(), err.data_ptr(), _stream_ptr()),
                   "igmc_candidate_lists")
        Cd.cand, Cd.per_user = run["lists"].data_ptr(), 1
        Cd.num_pairs = run["P"] = int(run["user_off"][U].item())
        run["Cd"] = Cd
        if run["P"] > 0:
            self._prime()
        return run["P"]

    def start_pairs(self, users, items):
        """plan a run over the explicit pairs (users[i], items[i]).  Returns their number."""
        return self._start_explicit("pairs", users, items)

    def start_explain(self, users, items, m=None):
        """plan an explanation run over the explicit pairs (users[i], items[i]) (``explain_pairs``): the base pass
        scores them and counts their subgraphs' ratings; once it is done, ``step`` reads the total (the run's one host
        sync) and goes on with the occlusion pass.  ``m``: keep each pair's first m ratings.  Returns the number of
        pairs."""
        m = _check_top(m, "m")
        return self._start_explicit("explain", users, items, m=m, phase="base")

    def start_attribute(self, users, items, m=None):
        """plan an attribution run over the explicit pairs (users[i], items[i]) (``attribute_pairs``): the base pass of
        ``start_explain``, then (after the run's one host sync, the rating total) a gradient pass over the same pairs.
        ``m``: keep each pair's first m ratings.  Returns the number of pairs."""
        m = _check_top(m, "m")
        return self._start_explicit("attribute", users, items, m=m, phase="base")

    def _start_explicit(self, kind, users, items, **extra):
        g = self.graph
        users = _host_ids(users, "users", g.num_users)
        items = _host_ids(items, "items", g.num_items)
        if len(users) != len(items):
            raise ValueError("users and items must have the same length (%d vs %d)" % (len(users), len(items)))
        P, dev = len(users), self.dev
        run = dict(kind=kind, P=P, version=g.version, scores=torch.empty(P, dtype=torch.float32, device=dev), **extra)
        self.run = run
        if kind in ("explain", "attribute"):
            run["num_edges"] = torch.zeros(P, dtype=torch.int32, device=dev)
            run["offsets"] = torch.zeros(P + 1, dtype=torch.int64, device=dev)
            for s in self.slots:
                if kind == "explain" and "j" not in s:
                    s["j"] = torch.zeros(self.B, dtype=torch.int32, device=dev)
        if P == 0:
            return 0
        run["pu"] = torch.from_numpy(users.astype(np.int32)).to(dev)
        run["pv"] = torch.from_numpy(items.astype(np.int32)).to(dev)
        Cd = _lib.Candidates()
        Cd.pair_u, Cd.pair_v, Cd.num_pairs = run["pu"].data_ptr(), run["pv"].data_ptr(), P
        run["Cd"] = Cd
        self._prime()
        return P

    def _rating_total(self, phase):
        """after the base pass of an explanation or attribution run: the offsets of the pairs' ratings, their total T
        (the run's one host sync) and the output buffers [T] (run["occ"]: occluded scores or gradients).  Returns T."""
        run, dev = self.run, self.dev
        _lib.check(self.lib.igmc_explain_offsets(run["num_edges"].data_ptr(), run["P"], run["offsets"].data_ptr(),
                                                 _stream_ptr()), "igmc_explain_offsets")
        T = run["T"] = int(run["offsets"][run["P"]].item())
        run["phase"] = phase
        run["occ"] = torch.empty(T, dtype=torch.float32, device=dev)
        for k in ("user", "item", "rating"):
            run[k] = torch.empty(T, dtype=torch.int32, device=dev)
        if T == 0:
            run["steps"] = run["done"] = 0
        if T >= (1 << 31) - 1:
            raise NotImplementedError("an explanation run covers fewer than 2^31 - 1 ratings, not %d" % T)
        return T

    def _start_occlusion(self):
        """the occlusion pass of an explanation run primed.  Returns True when it has positions."""
        T = self._rating_total("occlude")
        if T == 0:
            return False
        run, dev = self.run, self.dev
        ecap = self.extractor._out_caps(self.B)[1]
        for s in self.slots:
            if s.get("keep") is None or s["keep"].numel() < ecap:
                s["keep"] = torch.ones(ecap, dtype=torch.uint8, device=dev)
            # a training-mode forward with both dropout rates 0: the eval forward of the kept edges
            d = self.model.make_dropout(False)[0]
            d.edge_keep = s["keep"].data_ptr()
            s["drop"] = (d, [s["keep"]])
        self._prime(T)
        return True

    def _start_gradient(self):
        """the gradient pass of an attribution run primed: the P pairs again, on the L2 plan with as many CTAs per
        subgraph as ``l2_cluster`` gives this batch shape, whatever plan the model chose for the base pass.  Returns
        True when there are ratings."""
        from .models import l2_cluster
        n_cap = self.batches[0]._priv["n_cap"]
        if self._rating_total("grad") == 0:
            return False
        run, m, dev = self.run, self.model, self.dev
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        run["plan"] = _lib.plan_l2(l2_cluster(n_cap, self.B, sms))
        ncap, ecap = self.extractor._out_caps(self.B)[:2]
        L, f32 = len(m.convs), dict(dtype=torch.float32, device=dev)
        ext = m._cmodel.readout != 0
        # d score / d lin2 output of every graph: multiply_by for IGMC, 1 for DGCNN_RS (its lin2 output is the score)
        run["gws"] = dict(seed=torch.full((self.B,), 1.0 if ext else float(m._cmodel.multiply_by), **f32),
                          scratch=torch.empty(2, ncap, _lib.HIDDEN, **f32), edge_grad=torch.empty(ecap, **f32),
                          dstate=torch.empty(ncap, _lib.HIDDEN * L, **f32) if ext else None,
                          pgrad=torch.zeros(m._cmodel.param_count, **f32) if ext else None)
        with self._forced_plan():
            self._prime()
        return True

    @contextlib.contextmanager
    def _forced_plan(self):
        """inside the block the model launches the gradient pass's plan (run["plan"], with its own plan cache); the
        model's plan and cache are restored after it"""
        run, m = self.run, self.model
        if run is None or run.get("plan") is None:
            yield
            return
        own = (m.kernel_plan, m._plans)
        m.kernel_plan, m._plans = run["plan"], self._grad_plans
        try:
            yield
        finally:
            m.kernel_plan, m._plans = own

    def _prime(self, total=None):
        """candidate pairs + extraction of the first batch, the model's plan for it (its one host sync, if any) and
        the prepared weights of every parameter set; captured graphs of an earlier run or pass are dropped (they hold
        its buffers, its candidate total and the graph's shape as it was; the extractor follows an updated graph).
        ``total``: the positions of the pass (default: the run's pairs)."""
        run = self.run
        run["steps"] = ((run["P"] if total is None else total) + self.B - 1) // self.B
        run["done"] = 0
        self.graphs, self.eager_done = {}, set()
        self.cursor.zero_()
        self.batches = [None, None]
        self._next(0)
        if _lib.is_rs(self.model._plan(self.batches[0])):
            for j in range(self.K):
                with self._params(j):
                    self.model.prep_weights()

    def _next(self, slot):
        """candidate pairs of the next B positions (device cursor) + their extraction into batch slot ``slot``"""
        s, run, err = self.slots[slot], self.run, self.extractor.err.data_ptr()
        occlude = run.get("phase") == "occlude"
        if occlude:
            _lib.check(self.lib.igmc_occlusion_pairs(C.byref(self.graph._c), run["pu"].data_ptr(),
                                                     run["pv"].data_ptr(), run["offsets"].data_ptr(), run["P"],
                                                     self.cursor.data_ptr(), self.B, s["u"].data_ptr(),
                                                     s["v"].data_ptr(), s["pid"].data_ptr(), s["tag"].data_ptr(),
                                                     s["j"].data_ptr(), err, _stream_ptr()), "igmc_occlusion_pairs")
        else:
            _lib.check(self.lib.igmc_candidate_pairs(C.byref(self.graph._c), C.byref(run["Cd"]),
                                                     self.cursor.data_ptr(), self.B, s["u"].data_ptr(),
                                                     s["v"].data_ptr(), s["pid"].data_ptr(), s["tag"].data_ptr(), err,
                                                     _stream_ptr()), "igmc_candidate_pairs")
        b = self.batches[slot] = self.extractor.extract(pairs=(s["u"], s["v"], None), pair_ids=s["pid"], reuse=True,
                                                        slot=slot)
        if occlude:
            _lib.check(self.lib.igmc_occlusion_mask(C.byref(b._lazy["_c"]), self.B, s["tag"].data_ptr(),
                                                    s["j"].data_ptr(), s["keep"].data_ptr(), run["user"].data_ptr(),
                                                    run["item"].data_ptr(), run["rating"].data_ptr(), err,
                                                    _stream_ptr()), "igmc_occlusion_mask")
        elif run.get("phase") == "base":
            _lib.check(self.lib.igmc_explain_count(b._priv["edge_ptr"].data_ptr(), s["tag"].data_ptr(), self.B,
                                                   run["num_edges"].data_ptr(), _stream_ptr()), "igmc_explain_count")

    @contextlib.contextmanager
    def _params(self, j):
        """the model's kernels read parameter set ``j`` and its prepared weights inside the block (the launch code of
        the model is used as it is; only the buffers it reads are exchanged)"""
        m = self.model
        own = (m.flat_params, m._wprep, m.__dict__.get("_prepped", False))
        m.flat_params, m._wprep, m._prepped = self.params[j], self.wprep[j], True
        try:
            yield
        finally:
            m.flat_params, m._wprep, m._prepped = own

    def _score(self, slot):
        """eval forward of batch ``slot`` with every parameter set, then the merge / scatter of the mean.  An occlusion
        batch runs the training-mode forward with its slot's edge mask and no dropout: the eval forward of each
        subgraph without its masked rating."""
        m, b, s, run = self.model, self.batches[slot], self.slots[slot], self.run
        if run.get("phase") == "grad":
            return self._gradient(slot)
        occlude = run.get("phase") == "occlude"
        training, drop = (True, s["drop"]) if occlude else (False, self.drop)
        preds = None
        for j in range(self.K):
            with self._params(j):
                pred, _ = m._launch_forward(b, training, drop)
            if self.K == 1:
                preds = pred
            else:
                self.preds[j].copy_(pred)
                preds = self.preds
        if run["kind"] == "recommend":
            _lib.check(self.lib.igmc_topk_merge(preds.data_ptr(), self.K, self.B, s["tag"].data_ptr(),
                                                s["v"].data_ptr(), run["k"], run["top_s"].data_ptr(),
                                                run["top_i"].data_ptr(), _stream_ptr()), "igmc_topk_merge")
        else:
            out = run["occ"] if occlude else run["scores"]
            _lib.check(self.lib.igmc_score_scatter(preds.data_ptr(), self.K, self.B, s["tag"].data_ptr(),
                                                   out.data_ptr(), _stream_ptr()), "igmc_score_scatter")

    def _gradient(self, slot):
        """per parameter set: the eval forward of batch ``slot`` on the L2 plan, (DGCNN_RS) the SortPooling backward
        seeded with d score / d lin2 output, igmc_edge_grad and the scatter of each rating's gradient to its position
        (checkpoint k of K: stored, then added, then divided by K)"""
        m, b, s, run = self.model, self.batches[slot], self.slots[slot], self.run
        gw, p, st = run["gws"], b._priv, _stream_ptr()
        adj_c, _ = b.adjacency()
        d = self.drop[0]
        for j in range(self.K):
            with self._params(j):
                _, saved = m._launch_forward(b, False, self.drop)
                ws = saved["ws"]
                S = _lib.Saved.from_buffer_copy(saved["S"])
                S.l2_scratch = gw["scratch"].data_ptr()
                if gw["dstate"] is not None:
                    S.dstate = gw["dstate"].data_ptr()
                    _lib.check(self.lib.igmc_sortpool_backward(C.byref(m._csort), m.flat_params.data_ptr(),
                                                               ws["states"].data_ptr(), p["node_ptr"].data_ptr(),
                                                               self.B, p["n_cap"], C.byref(ws["sp"]["S"]),
                                                               gw["seed"].data_ptr(), gw["dstate"].data_ptr(), 1.0,
                                                               gw["pgrad"].data_ptr(), b._err.data_ptr(), st),
                               "igmc_sortpool_backward")
                _lib.check(self.lib.igmc_edge_grad(C.byref(m._cmodel), m.flat_params.data_ptr(),
                                                   p["node_label"].data_ptr(), p["node_ptr"].data_ptr(),
                                                   p["edge_ptr"].data_ptr(), C.byref(adj_c), self.B, p["n_cap"],
                                                   C.byref(d), C.byref(S), gw["seed"].data_ptr(),
                                                   gw["edge_grad"].data_ptr(), ws["cluster"], b._err.data_ptr(), st),
                           "igmc_edge_grad")
            _lib.check(self.lib.igmc_edge_grad_scatter(C.byref(b._lazy["_c"]), self.B, s["tag"].data_ptr(),
                                                       gw["edge_grad"].data_ptr(), run["offsets"].data_ptr(), j,
                                                       self.K, run["occ"].data_ptr(), run["user"].data_ptr(),
                                                       run["item"].data_ptr(), run["rating"].data_ptr(),
                                                       self.extractor.err.data_ptr(), st), "igmc_edge_grad_scatter")

    def _launch(self, slot):
        main = torch.cuda.current_stream()
        self.side.wait_stream(main)
        with self._forced_plan():
            with torch.cuda.stream(self.side):
                # the next batch is produced and extracted beside this batch's forward (gate: only once the forward's
                # clusters are resident, see TrainEngine._launch_pipe); after the last batch it is all padding
                self.model.gate_wait(self.batches[slot])
                self._next(slot ^ 1)
            self._score(slot)
        main.wait_stream(self.side)

    def step(self):
        """score the current batch while the next one is extracted.  Returns False once every batch is scored."""
        run = self.run
        if run is None or run["P"] == 0 or run["done"] >= run["steps"]:
            return False
        if self.graph.version != run["version"]:
            raise RuntimeError("the rating graph was updated during this run: its candidates and captured steps belong "
                               "to the old graph; start the run again")
        slot = run["done"] & 1
        replay_step(self.graphs, self.eager_done, slot, lambda: self._launch(slot), self.use_graph)
        run["done"] += 1
        if run["done"] < run["steps"]:
            return True
        if run.get("phase") != "base":
            return False
        return self._start_occlusion() if run["kind"] == "explain" else self._start_gradient()

    def finish(self):
        """wait for the run, check the error word (one host sync) and return (top_items [U, k] int64, top_scores
        [U, k] fp32), the scores [P] fp32 or the ``Explanation``, on the device"""
        run = self.run
        while self.step():
            pass
        if run.get("phase") == "base":    # no pairs: the run has no second pass
            self._rating_total("none")
        code = int(self.extractor.err.item())
        if code:
            self.extractor.err.zero_()
        _lib.check_kernel_error(code)
        self.run = None
        if run["kind"] == "recommend":
            return run["top_i"], run["top_s"]
        if run["kind"] in ("explain", "attribute"):
            return self._order(run)
        return run["scores"]

    def _order(self, run):
        """igmc_occlusion_order: every pair's ratings by |delta| (attribution: |grad|) descending (NaN last, ties by
        position), all of them or the first m"""
        P, T, m, dev = run["P"], run["T"], run["m"], self.dev
        shape = (P, m) if m else (T,)
        out = dict(user=torch.empty(shape, dtype=torch.int32, device=dev),
                   item=torch.empty(shape, dtype=torch.int32, device=dev),
                   rating=torch.empty(shape, dtype=torch.int32, device=dev),
                   delta=torch.empty(shape, dtype=torch.float32, device=dev))
        nbytes = C.c_int64(0)
        _lib.check(self.lib.igmc_occlusion_order_ws_bytes(P, T, C.byref(nbytes)), "igmc_occlusion_order_ws_bytes")
        ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
        explain = run["kind"] == "explain"
        _lib.check(self.lib.igmc_occlusion_order(run["scores"].data_ptr() if explain else None, run["occ"].data_ptr(),
                                                 run["offsets"].data_ptr(), P, T, run["user"].data_ptr(),
                                                 run["item"].data_ptr(), run["rating"].data_ptr(), m or 0,
                                                 ws.data_ptr(), ws.numel(), out["user"].data_ptr(),
                                                 out["item"].data_ptr(), out["rating"].data_ptr(),
                                                 out["delta"].data_ptr(), _stream_ptr()), "igmc_occlusion_order")
        return (Explanation if explain else Attribution)(run["scores"], run["num_edges"], run["offsets"], out["user"],
                                                         out["item"], out["rating"], out["delta"])

    def recommend(self, users, k, items=None, exclude_rated=True, retrieve=None):
        self.start_recommend(users, k, items, exclude_rated, retrieve)
        return self.finish()

    def predict_pairs(self, users, items):
        self.start_pairs(users, items)
        return self.finish()

    def explain_pairs(self, users, items, m=None):
        self.start_explain(users, items, m)
        return self.finish()

    def attribute_pairs(self, users, items, m=None):
        self.start_attribute(users, items, m)
        return self.finish()

    def close(self):
        torch.cuda.synchronize()
        self.graphs = {}


# ---- public API -----------------------------------------------------------------------------------------------------
def predict_pairs(model, graph, users, items, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None, batch_size=256,
                  checkpoints=None, sample_seed=0):
    """eval-mode scores [P] (fp32, on the model's device) of the pairs (users[i], items[i]); a pair rated in ``graph``
    is scored on its subgraph without the target edge, as in training.  ``checkpoints``: average of the checkpoints'
    scores (fp32 sum in checkpoint order / K)."""
    nu, ni = graph.shape
    users, items = _host_ids(users, "users", nu), _host_ids(items, "items", ni)
    if len(users) != len(items):
        raise ValueError("users and items must have the same length (%d vs %d)" % (len(users), len(items)))
    if len(users) == 0:
        return torch.zeros(0, dtype=torch.float32, device=model.flat_params.device)
    eng = InferenceEngine(model, graph, h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)
    try:
        return eng.predict_pairs(users, items)
    finally:
        eng.close()


def explain_pairs(model, graph, users, items, m=None, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None, batch_size=256,
                  checkpoints=None, sample_seed=0):
    """why each pair (users[i], items[i]) got its score: for every rating in the pair's enclosing subgraph (a rated
    pair's own rating excluded, as in ``predict_pairs``), delta = the score of that subgraph without the rating (both
    directed edges removed; same nodes, no re-sampling) - the pair's score.  Returns an ``Explanation`` of device
    tensors: score [P] (bit for bit ``predict_pairs``), num_edges [P], offsets [P+1] and per rating user / item /
    rating (its label) / delta, ordered within a pair by |delta| descending, NaN after every number, ties by the
    rating's position in the subgraph's edge_index; flat with pair p at [offsets[p], offsets[p+1]) when ``m`` is None,
    else the first ``m`` per pair [P, m], padded with user / item / rating -1 and delta 0.  ``checkpoints``: every score
    is the fp32 checkpoint mean, as in ``predict_pairs``."""
    nu, ni = graph.shape
    m = _check_top(m, "m")
    users, items = _host_ids(users, "users", nu), _host_ids(items, "items", ni)
    if len(users) != len(items):
        raise ValueError("users and items must have the same length (%d vs %d)" % (len(users), len(items)))
    if len(users) == 0:
        dev = model.flat_params.device
        shape = (0, m) if m else (0,)
        i32 = dict(dtype=torch.int32, device=dev)
        return Explanation(torch.zeros(0, dtype=torch.float32, device=dev), torch.zeros(0, **i32),
                           torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(shape, **i32),
                           torch.zeros(shape, **i32), torch.zeros(shape, **i32),
                           torch.zeros(shape, dtype=torch.float32, device=dev))
    eng = InferenceEngine(model, graph, h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)
    try:
        return eng.explain_pairs(users, items, m)
    finally:
        eng.close()


def attribute_pairs(model, graph, users, items, m=None, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None,
                    batch_size=256, checkpoints=None, sample_seed=0):
    """why each pair (users[i], items[i]) got its score, to first order and in one backward pass per pair: every rating
    e of the pair's enclosing subgraph (a rated pair's own rating excluded) gets a weight m_e on the messages of both
    its directed edges in every layer, the mean normalisers counting the weights (deg(v) = sum of m over v's in-edges;
    ``rgcn="pyg-2"``: |N_r(v)| per relation), so that a 0/1 weight is dropout_adj's mask and m = 1 the model.  grad =
    d score / d m_e at m = 1; -grad estimates ``explain_pairs``' delta.  A node whose mean runs over one in-edge (its
    only one; pyg-2: its only one of that relation) adds nothing at that layer: removing the edge jumps its aggregate
    to 0, and the relaxation has no slope there.  DGCNN_RS: the gradient flows through the SortPooling order of the
    forward.  Returns an ``Attribution`` in ``Explanation``'s layout: score [P] (bit for bit ``predict_pairs``),
    num_edges [P], offsets [P+1], per rating user / item / rating / grad ordered by |grad| descending, NaN last, ties
    by position; the first ``m`` per pair [P, m] padded with -1 / -1 / -1 / 0.  The gradient pass runs the L2 kernel
    plan whatever plan the model uses.  ``checkpoints``: score and grad are fp32 checkpoint means (sum in checkpoint
    order / K)."""
    nu, ni = graph.shape
    m = _check_top(m, "m")
    users, items = _host_ids(users, "users", nu), _host_ids(items, "items", ni)
    if len(users) != len(items):
        raise ValueError("users and items must have the same length (%d vs %d)" % (len(users), len(items)))
    if len(users) == 0:
        dev = model.flat_params.device
        shape = (0, m) if m else (0,)
        i32 = dict(dtype=torch.int32, device=dev)
        return Attribution(torch.zeros(0, dtype=torch.float32, device=dev), torch.zeros(0, **i32),
                           torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(shape, **i32),
                           torch.zeros(shape, **i32), torch.zeros(shape, **i32),
                           torch.zeros(shape, dtype=torch.float32, device=dev))
    eng = InferenceEngine(model, graph, h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)
    try:
        return eng.attribute_pairs(users, items, m)
    finally:
        eng.close()


def recommend(model, graph, users, k, *, items=None, exclude_rated=True, retrieve=None, h=1, sample_ratio=1.0,
              max_nodes_per_hop=None, batch_size=256, checkpoints=None, sample_seed=0):
    """for every query user the ``k`` best candidate items: (top_items [U, k] int64, top_scores [U, k] fp32), on the
    model's device.  Candidates: ``items`` (sorted, deduplicated), a 2-D ``items`` [U, width] of per-user lists (-1 =
    empty slot; each row sorted and deduplicated), the user's ``retrieve`` items with the most bridges
    (``corated_items``), or every item; minus the user's rated items when ``exclude_rated``.  Order: score
    descending, then item ascending; a NaN score ranks last; a user with fewer than ``k`` candidates gets item -1 /
    score -inf in the empty slots.  A pair's score does not depend on the candidates it was ranked among."""
    k = _check_k(k)
    nu, ni = graph.shape
    if retrieve is not None and items is not None:
        raise ValueError("retrieve= chooses the candidates itself: pass it without items=")
    if retrieve is not None:
        _check_m(retrieve, ni)
    users = _host_ids(users, "users", nu)
    if _is_rows(items):
        if torch.is_tensor(items) and items.device.type == "cuda":
            if items.shape[0] != len(users):
                raise ValueError("items has %d rows, one per query user is %d" % (items.shape[0], len(users)))
        else:
            items = _user_rows(items, len(users), ni, torch.device("cpu")).numpy()
    elif items is not None:
        items = _host_ids(items, "items", ni)
    if len(users) == 0:
        dev = model.flat_params.device
        return (torch.zeros(0, k, dtype=torch.int64, device=dev), torch.zeros(0, k, dtype=torch.float32, device=dev))
    eng = InferenceEngine(model, graph, h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)
    try:
        return eng.recommend(users, k, items, exclude_rated, retrieve)
    finally:
        eng.close()


def corated_items(graph, users, m, exclude_rated=True):
    """per query user the ``m`` items with the most bridges to it: (items [U, m], paths [U, m]) int32 on the graph's
    device.  paths[v] counts the 3-paths u - i - u' - v (u' != u): the edges that join u's and v's stars in their
    h = 1 enclosing subgraph, without which the model has no collaborative signal for the pair.  Ordered by paths
    descending, then item ascending; items without a bridge are never returned, the rest of a row is item -1 /
    paths 0; ``exclude_rated`` drops the user's rated items.  Exact integer counts: runs are bit-identical.
    ``graph``: a RatingGraph or a rating matrix (copied to the current CUDA device).  One host synchronisation (the
    error word)."""
    g = graph if isinstance(graph, RatingGraph) else RatingGraph(graph)
    if g.device is None:
        raise RuntimeError("igmc_b200 retrieval runs on a CUDA device (there is no CPU path)")
    m = _check_m(m, g.num_items)
    users = _host_ids(users, "users", g.num_users)
    lib = _lib.load()
    err = torch.zeros(1, dtype=torch.int32, device=g.device)
    items, paths = _corated(lib, g, torch.from_numpy(users.astype(np.int32)).to(g.device), m, exclude_rated, err, {})
    _lib.check_kernel_error(int(err.item()))
    return items, paths
