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
* ``recommend_users(model, graph, items, k)`` and ``corated_users(graph, items, m)`` ask the same from the item's side:
  per query item the ``k`` best users (the audience of a new or promoted item) and the ``m`` users with the most
  bridges to it.  The candidate kernels run on the graph's transposed view (``RatingGraph._ct``) and
  ``igmc_item_query_pairs`` turns their pairs back into (user, item); every score is ``predict_pairs``' score of the
  pair;
* ``explain_pairs(model, graph, users, items, m)`` -> per pair its score and, for every rating in its enclosing
  subgraph, the score change from removing that rating (csrc/explain.cu): a base pass of the pairs, then an occlusion
  pass over (pair, rating) positions whose batches carry an edge mask into a training-mode forward without dropout;
* ``attribute_pairs(model, graph, users, items, m)`` -> the same layout with, per rating, the score's gradient with
  respect to a weight on that rating (igmc_edge_grad): the same base pass, then one gradient pass over the P pairs, each
  an L2-plan eval forward and one backward whose list walk writes every edge's term;
* ``explain_nodes`` / ``attribute_nodes(model, graph, users, items, m)`` -> the same two answers per node of the
  enclosing subgraph (its users and items other than the two targets): the score change from removing every rating of
  the node, and the score's gradient with respect to a gate on all of them.  The passes are the two above with the
  pair's nodes as positions;
* ``pair_gradients(model, graph, users, items, y)`` -> per-example gradients [K, P, param_count] of each pair's squared
  error (or score), ``influence(model, graph, train, test, k)`` -> per test pair the k training pairs of largest and
  smallest TracIn-CP influence, ``self_influence(model, graph, train)`` -> sum_k eta_k ||grad l_i||^2
  (csrc/influence.cu): a per-graph gradient assembly after the training backward, a split-K GEMM of the conv blocks
  plus the readout's rank-1 factors, and a streaming top-k merge;
* ``RatingSessions(graph, users, session, items, values)`` -> users described by ratings passed with the query: per
  session a user id (new ids start from an empty row) and edits to that user's row in ``RatingGraph.update``'s
  encoding, applied only while that user's own pairs are scored; ``predict_sessions``, ``recommend_sessions`` and
  ``corated_items_sessions`` score, rank and retrieve for many sessions in one run and leave the graph unchanged.  A
  session's results are bit for bit those of the graph functions on the graph with that session's edits applied;
* ``predict_draws(model, graph, users, items, draws)`` -> per pair S Monte-Carlo-dropout draws of its score (the
  training-mode forward under the model's own edge and hidden dropout, masks keyed by the pair id and the draw index)
  and their mean and std (csrc/draws.cu); ``recommend``, ``recommend_users`` and ``recommend_sessions`` with
  ``draws=S`` rank by mean + beta * std over S draws (Thompson sampling at S = 1, UCB for beta > 0);
* ``counterfactual(model, graph, users, items, rivals, max_removals)`` -> per query (u, X, Y) the ratings of u whose
  removal together puts X behind the rival Y, found greedily with every candidate scored exactly (csrc/counterfactual.cu):
  a base pass, then per step one pass over every remaining rating of every active query, each trial extracted in
  session mode with the user's row without its removals;
* ``elicit(model, sessions, n, targets)`` -> per session the ``n`` items it should be asked to rate: every answer to
  every question scored exactly (the session's row plus the hypothetical rating, extracted in session mode), ranked by
  the mean over ``targets`` of how far the answers move each target's score (csrc/elicit.cu);
  ``question_impact(model, sessions, session, questions, targets)`` -> that impact and the mean target score under
  each answer for explicit (session, question) units;
* ``RecommendationCache(model, graph, users, k)`` -> ``recommend``'s lists kept exact across ``graph.update``: an update
  rescores only the pairs whose h = 1 enclosing subgraph it can reach (csrc/recommend_cache.cu) and repairs the cached
  lists with them;
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
import os

import numpy as np
import torch

from . import _lib
from .train_eval import replay_step
from .util_functions import RatingGraph, SubgraphExtractor, _cuda_ints, _on_device_i32, _stream_ptr, _update_inputs

__all__ = ["predict_pairs", "recommend", "corated_items", "explain_pairs", "Explanation", "attribute_pairs",
           "Attribution", "pair_gradients", "influence", "self_influence", "Influence", "InferenceEngine",
           "RatingSessions", "predict_sessions", "recommend_sessions", "corated_items_sessions", "recommend_users",
           "corated_users", "explain_nodes", "NodeExplanation", "attribute_nodes", "NodeAttribution", "predict_draws",
           "Draws", "counterfactual", "Counterfactual", "elicit", "question_impact", "QuestionImpact",
           "RecommendationCache"]


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


def _user_rows(items, U, num_items, name="items"):
    """per-user candidate rows [U, width] checked on the host: a host array as int32 (IndexError for an id outside
    [-1, num_items)); an integer CUDA tensor as it is, checked by the kernel.  ValueError when the row count is not
    U.  ``name``: the argument the rows came in (item-side runs: per-item rows of users)."""
    if not torch.is_tensor(items):
        items = np.asarray(items)
    if items.shape[0] != U:
        raise ValueError("%s has %d rows, one per query slot is %d" % (name, items.shape[0], U))
    if _cuda_ints(items, name):
        return items
    a = np.asarray(items.cpu().numpy() if torch.is_tensor(items) else items)
    if a.size and not np.issubdtype(a.dtype, np.integer):
        raise TypeError("%s must be integers, not %s" % (name, a.dtype))
    a = a.astype(np.int64)
    if a.size and (a.min() < -1 or a.max() >= num_items):
        bad = int(a.min()) if a.min() < -1 else int(a.max())
        raise IndexError("%s: id %d out of range [-1, %d)" % (name, bad, num_items))
    return a.astype(np.int32)


def _check_count(n, name, hi, over=NotImplementedError):
    """``n`` as an int in [1, hi]: ValueError below 1, ``over`` above ``hi``"""
    n = int(n)
    if n < 1 or n > hi:
        raise (ValueError if n < 1 else over)("%s must lie in [1, %d], not %d" % (name, hi, n))
    return n


def _check_top(m):
    """None, or the count m in [1, IGMC_TOPK_MAX] of ratings an explanation keeps per pair"""
    return None if m is None else _check_count(m, "m", _lib.TOPK_MAX)


def _ranking_inputs(k, batch_size, items, retrieve, U, num_items, name="items"):
    """(k, m, cand, rows) of a ranking run over U query slots, checked on the host: m = ``retrieve`` (or None), cand
    the sorted distinct items of a 1-D ``items`` (or None), rows a 2-D ``items`` as ``_user_rows`` returns it (or
    None).  Item-side runs pass the candidate users as ``items``, num_users as ``num_items`` and ``name`` = "users"."""
    k = _check_count(k, "k", _lib.TOPK_MAX)
    _check_merge_fits(k, batch_size)
    if retrieve is not None and items is not None:
        raise ValueError("retrieve= chooses the candidates itself: pass it without %s=" % name)
    m = None if retrieve is None else _check_count(retrieve, "retrieve", num_items, ValueError)
    if _is_rows(items):
        return k, m, None, _user_rows(items, U, num_items, name)
    return k, m, None if items is None else np.unique(_host_ids(items, name, num_items)), None


def _corated(lib, shape, entry, args, U, m, exclude_rated, err, ws):
    """the retriever ``entry`` (igmc_corated_items, igmc_corated_sessions or igmc_corated_users, leading arguments
    ``args``) for U query slots on a graph of ``shape`` (num_users, num_items; the item side: the transposed shape):
    (ids, paths) [U, m] int32 on ``err``'s device.  ``ws``: a dict whose "ws" tensor is grown to the workspace the
    shape needs"""
    dev = err.device
    nbytes = C.c_int64(0)
    _lib.check(lib.igmc_corated_ws_bytes(shape[0], shape[1], U, m, C.byref(nbytes)), "igmc_corated_ws_bytes")
    if ws.get("ws") is None or ws["ws"].numel() < nbytes.value:
        ws["ws"] = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
    items = torch.empty(U, m, dtype=torch.int32, device=dev)
    paths = torch.empty(U, m, dtype=torch.int32, device=dev)
    _lib.check(getattr(lib, entry)(*args, m, int(bool(exclude_rated)), ws["ws"].data_ptr(), ws["ws"].numel(),
                                   items.data_ptr(), paths.data_ptr(), err.data_ptr(), _stream_ptr()), entry)
    return items, paths


def _check_merge_fits(k, batch_size):
    """ValueError unless the top-k merge (igmc_topk_merge, igmc_influence_topk) can run k kept entries against batches
    of ``batch_size`` pairs: it holds both in one CTA's shared memory.  A batch size below 1 is the engine's to refuse."""
    if int(batch_size) >= 1 and not _lib.load().igmc_topk_fits(int(k), int(batch_size)):
        raise ValueError("k = %d with batch_size = %d does not fit the top-k merge's shared memory (k + batch_size "
                         "entries in one CTA): lower batch_size or k" % (int(k), int(batch_size)))


INFLUENCE_T_MAX = 1024   # test pairs of one influence run: the test-side store is K * T * (conv block + factors) floats


def _host_y(y, name, n):
    """targets as a host fp32 vector of length ``n``; ValueError when the length differs or a value is not finite"""
    if torch.is_tensor(y):
        y = y.detach().cpu().numpy()
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    if len(y) != n:
        raise ValueError("%s has %d values, one per pair is %d" % (name, len(y), n))
    if not np.all(np.isfinite(y)):
        raise ValueError("%s must be finite" % name)
    return y.astype(np.float32)


def _host_pairs(shape, users, items, y=None, name="", first="users"):
    """(users, items, y or None) checked on the host: ids in range of ``shape``, matching lengths, finite y.  ``name``:
    the argument the pairs came in (train, test), ``first``: what the first array holds"""
    pre = name + " " if name else ""
    nu, ni = shape
    users, items = _host_ids(users, pre + first, nu), _host_ids(items, pre + "items", ni)
    if len(users) != len(items):
        raise ValueError("%s%s and items must have the same length (%d vs %d)" % (pre, first, len(users), len(items)))
    return users, items, (None if y is None else _host_y(y, pre + "y", len(users)))


def _split_pairs(pairs, name, need_y):
    """(users, items) or (users, items, y) -> a 3-tuple; ValueError for another arity or a missing y"""
    pairs = tuple(pairs)
    if len(pairs) not in (2, 3) or (need_y and len(pairs) != 3):
        raise ValueError("%s must be (users, items, y)%s" % (name, "" if need_y else " or (users, items)"))
    return pairs if len(pairs) == 3 else pairs + (None,)


def _check_lrs(lrs, K):
    """eta_k per checkpoint as a list of K floats (None: all 1)"""
    if lrs is None:
        return [1.0] * K
    lrs = [float(x) for x in np.asarray(lrs, dtype=np.float64).reshape(-1)]
    if len(lrs) != K:
        raise ValueError("lrs has %d values, one per checkpoint is %d" % (len(lrs), K))
    if not all(np.isfinite(lrs)):
        raise ValueError("lrs must be finite")
    return lrs


def _check_test_count(T):
    if T > INFLUENCE_T_MAX:
        raise NotImplementedError("an influence run takes at most %d test pairs, not %d: split the test set"
                                  % (INFLUENCE_T_MAX, T))


def _influence_inputs(shape, train, test, k, batch_size, lrs, K):
    """(k, train, test, lrs) of an influence run checked on the host; train and test as ``_host_pairs`` returns them"""
    k = _check_count(k, "k", _lib.TOPK_MAX)
    _check_merge_fits(k, batch_size)
    tr = _host_pairs(shape, *_split_pairs(train, "train", True), name="train")
    te = _host_pairs(shape, *_split_pairs(test, "test", False), name="test")
    _check_test_count(len(te[0]))
    return k, tr, te, _check_lrs(lrs, K)


def _check_per_pair_model(model):
    if model._cmodel.readout != 0:
        raise NotImplementedError("per-pair gradients need the IGMC readout: DGCNN_RS's SortPooling readout gradient "
                                  "is summed over the batch")


# The result of explain_pairs, device tensors: score [P] fp32 (= predict_pairs), num_edges [P] int32 (the ratings of
# each pair's subgraph), offsets [P+1] int64 (their exclusive prefix) and, per rating, user / item / rating int32 and
# delta fp32 (score without the rating - score): flat [offsets[P]] with pair p at [offsets[p], offsets[p+1]), or
# [P, m] padded with -1 / -1 / -1 / 0.
Explanation = collections.namedtuple("Explanation", "score num_edges offsets user item rating delta")

# The result of attribute_pairs: Explanation's layout and order with grad (d score / d m_e, the rating's weight m_e at
# m = 1) in place of delta.  -grad is the first-order estimate of explain_pairs' delta.
Attribution = collections.namedtuple("Attribution", "score num_edges offsets user item rating grad")

# The result of explain_nodes: score [P] fp32 (= predict_pairs), num_nodes [P] int32 (the non-target nodes of each
# pair's subgraph), offsets [P+1] int64 and, per node, node (its global user or item id) / label (its node_label: even
# a user, odd an item, 2h or 2h+1 at distance h) / ratings (its ratings in the subgraph) int32 and delta fp32 (score
# with every rating of the node removed - score): flat or [P, m] padded with -1 / -1 / 0 / 0.
NodeExplanation = collections.namedtuple("NodeExplanation", "score num_nodes offsets node label ratings delta")

# The result of attribute_nodes: NodeExplanation's layout and order with grad (d score / d g_n at g = 1, g_n a gate on
# the weight of each of the node's ratings: the sum of attribute_pairs' grad over them) in place of delta.
NodeAttribution = collections.namedtuple("NodeAttribution", "score num_nodes offsets node label ratings grad")

# the runs that explain a pair by its nodes, and the result of each explanation or attribution run
_NODE_KINDS = ("explain_nodes", "attribute_nodes")
_EXPLAIN_RESULTS = dict(explain=Explanation, attribute=Attribution, explain_nodes=NodeExplanation,
                        attribute_nodes=NodeAttribution)

# The result of influence: per test pair the k training pairs with the largest influence (pro_*, value descending) and
# the k with the smallest (con_*, value ascending), [T, k] device tensors; index = position in the training list
# (int64), value fp32; ties by index ascending, NaN after every number, empty slots index -1 and value -inf / +inf.
Influence = collections.namedtuple("Influence", "pro_index pro_value con_index con_value")


def influence_order_host(values, k):
    """twin of igmc_influence_topk over a whole run: (pro_index, pro_value, con_index, con_value) for one test pair's
    values [N] (index = position), padded with (-1, -inf) / (-1, +inf)"""
    v = np.asarray(values, np.float32)
    idx = np.arange(len(v))
    out = []
    for sign, pad in ((1.0, -np.inf), (-1.0, np.inf)):
        key = np.where(np.isnan(v), np.inf, -sign * v.astype(np.float64))
        o = np.lexsort((idx, key, np.isnan(v)))          # NaN last, key descending, then index
        ti = np.full(k, -1, np.int64)
        tv = np.full(k, pad, np.float32)
        n = min(k, len(o))
        ti[:n], tv[:n] = o[:n], v[o[:n]]
        out += [ti, tv]
    return tuple(out)


def influence_merge_host(top_v, top_i, seg_v, seg_i, sign):
    """twin of one side of one CTA of igmc_influence_topk: the running list (ranked under key sign * value) merged with
    a batch's values (index < 0 skipped) by rank counting; returns the new (values, indices)"""
    def before(av, ai, bv, bi):
        if ai < 0:
            return False
        if bi < 0:
            return True
        ak, bk = np.float32(sign) * np.float32(av), np.float32(sign) * np.float32(bv)
        an, bn = np.isnan(ak), np.isnan(bk)
        if an or bn:
            return ai < bi if (an and bn) else bool(bn)
        return ak > bk or (ak == bk and ai < bi)
    k = len(top_v)
    V = list(np.asarray(top_v, np.float32)) + list(np.asarray(seg_v, np.float32))
    I = list(np.asarray(top_i, np.int64)) + list(np.asarray(seg_i, np.int64))
    out_v, out_i = np.array(top_v, np.float32), np.array(top_i, np.int64)
    for e in range(len(V)):
        if e >= k and I[e] < 0:
            continue
        r = e if e < k else sum(1 for o in range(k) if before(V[o], I[o], V[e], I[e]))
        r += sum(1 for x in range(k, len(V)) if x != e and before(V[x], I[x], V[e], I[e]))
        if r < k:
            out_v[r], out_i[r] = V[e], I[e]
    return out_v, out_i


def readout_dot_host(fa, fb, F):
    """the readout block's share of <G_a, G_b> from two factor rows dhid [128] | feat [F] | hid [128] | dpred"""
    H = _lib.LIN1_OUT
    dd = float(np.dot(fa[:H], fb[:H]))
    ff = float(np.dot(fa[H:H + F], fb[H:H + F]))
    hh = float(np.dot(fa[H + F:2 * H + F], fb[H + F:2 * H + F]))
    return dd * (ff + 1.0) + float(fa[2 * H + F]) * float(fb[2 * H + F]) * (hh + 1.0)


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


def corated_users_host(row_ptr, col_idx, num_users, num_items, items, m, exclude_rated=True):
    """twin of igmc_corated_users: per query item v the ``m`` users with the most bridges, C[u][v] = (B B^T B)[u][v]
    - deg(u) B[u][v] (``corated_host``'s count of v for u), ordered by count descending then user ascending, users
    without a bridge dropped, ``exclude_rated`` dropping v's raters; (users [I, m], paths [I, m]) int32 padded with
    -1 / 0"""
    import scipy.sparse as ssp
    items = np.asarray(items, np.int64).reshape(-1)
    rp = np.asarray(row_ptr, np.int64)
    nnz = int(rp[num_users])
    Bm = ssp.csr_matrix((np.ones(nnz, np.int64), np.asarray(col_idx[:nnz], np.int64), rp[:num_users + 1]),
                        shape=(num_users, num_items))
    Bv = Bm[:, items].toarray()                              # [nu, I]
    P = np.asarray((Bm @ (Bm.T @ ssp.csr_matrix(Bv))).toarray(), np.int64) - np.diff(rp)[:num_users, None] * Bv
    if exclude_rated:
        P[Bv > 0] = 0
    users = np.full((len(items), m), -1, np.int32)
    paths = np.zeros((len(items), m), np.int32)
    for j in range(len(items)):
        o = np.argsort(-P[:, j], kind="stable")[:m]         # count descending, then user ascending
        o = o[P[o, j] > 0]
        users[j, :len(o)], paths[j, :len(o)] = o, P[o, j]
    return users, paths


def item_query_pairs_host(num_items, links_u, links_v):
    """twin of igmc_item_query_pairs: the (item, user) pairs of a run over the transposed view as (links_u = users,
    links_v = items, pair_id = u * num_items + v)"""
    u, v = np.asarray(links_v, np.int64), np.asarray(links_u, np.int64)
    return u, v, u * num_items + v


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


# ---- host twins of the cache repair kernels (csrc/recommend_cache.cu) ----------------------------------------------
def rescore_plan_host(row_ptr, col_idx, num_items, users, edit_u, edit_v, cand=None, exclude_rated=True):
    """twin of igmc_rescore_plan on the updated graph: (user_off [U+1] int64, items int32, full [U] uint8, candidate
    total).  Slot j's items: its candidates (``cand`` or every item, minus the user's rated items when
    ``exclude_rated``) that are b_i, or in row(a_i) when the user rated b_i; all of them when the user is some a_i"""
    rp, ci = np.asarray(row_ptr, np.int64), np.asarray(col_idx, np.int64)
    allowed = np.zeros(num_items, bool)
    allowed[np.arange(num_items) if cand is None else np.asarray(cand, np.int64)] = True
    out, full, total = [], [], 0
    for u in np.asarray(users, np.int64).reshape(-1):
        row = ci[rp[u]:rp[u + 1]]
        mark = np.zeros(num_items, bool)
        for a, b in zip(np.asarray(edit_u, np.int64).reshape(-1), np.asarray(edit_v, np.int64).reshape(-1)):
            if a == u:
                mark[:] = True
                continue
            mark[b] = True
            if b in row:
                mark[ci[rp[a]:rp[a + 1]]] = True
        ok = allowed.copy()
        if exclude_rated:
            ok[row] = False
        items = np.flatnonzero(mark & ok)
        out.append(items)
        full.append(len(items) == int(ok.sum()))
        total += int(ok.sum())
    user_off = np.concatenate([[0], np.cumsum([len(x) for x in out])]).astype(np.int64)
    items = (np.concatenate(out) if out else np.zeros(0)).astype(np.int32)
    return user_off, items, np.asarray(full, np.uint8), total


def cache_invalidate_host(user_off, resc, full, complete, top_s, top_i):
    """twin of igmc_cache_invalidate: (top_s, top_i, thr_s, thr_i) with the rescored items removed from every prefix
    (all of a fully rescored slot's: its own user's edits may have changed its candidates) and the threshold key (item -1: none, -2: an empty prefix of a slot that is not complete)"""
    top_s, top_i = np.array(top_s, np.float32), np.array(top_i, np.int64)
    U, D = top_i.shape
    thr_s, thr_i = np.full(U, -np.inf, np.float32), np.full(U, -1, np.int64)
    for j in range(U):
        n = int(np.argmin(np.r_[top_i[j] >= 0, False]))           # the leading entries with an item
        if not (complete[j] or full[j]):
            thr_i[j], thr_s[j] = (top_i[j, n - 1], top_s[j, n - 1]) if n else (-2, -np.inf)
        keep = ~np.isin(top_i[j, :n], np.asarray(resc[user_off[j]:user_off[j + 1]], np.int64)) & (full[j] == 0)
        s, i = top_s[j, :n][keep], top_i[j, :n][keep]
        top_s[j], top_i[j] = -np.inf, -1
        top_s[j, :len(s)], top_i[j, :len(i)] = s, i
    return top_s, top_i, thr_s, thr_i


def cache_settle_host(thr_s, thr_i, top_s, top_i, k):
    """twin of igmc_cache_settle: (top_s, top_i, complete, redo) with every list cut to its exact depth"""
    top_s, top_i = np.array(top_s, np.float32), np.array(top_i, np.int64)
    U, D = top_i.shape
    complete, redo = np.zeros(U, np.uint8), []
    for j in range(U):
        d = 0
        if thr_i[j] != -2:
            while d < D and top_i[j, d] >= 0 and (thr_i[j] == -1 or
                                                   not _before(thr_s[j], thr_i[j], top_s[j, d], top_i[j, d])):
                d += 1
        top_s[j, d:], top_i[j, d:] = -np.inf, -1
        complete[j] = thr_i[j] == -1 and d < D
        if thr_i[j] != -1 and d < k:
            redo.append(j)
    return top_s, top_i, complete, np.asarray(redo, np.int32)


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


def node_positions_host(node_label, n0, n1):
    """the nodes at positions 0, 1, ... of the graph with nodes [n0, n1): its nodes with node_label >= 2, in order"""
    return n0 + np.flatnonzero(np.asarray(node_label)[n0:n1] >= 2)


def node_count_host(node_ptr, tag, num_nodes):
    """twin of igmc_explain_node_count: num_nodes[tag[g]] = max(N_g - 2, 0) for every graph g with tag >= 0;
    ``num_nodes`` is updated in place and returned"""
    node_ptr = np.asarray(node_ptr, np.int64)
    for g in range(len(node_ptr) - 1):
        if tag[g] >= 0:
            num_nodes[tag[g]] = max(int(node_ptr[g + 1] - node_ptr[g]) - 2, 0)
    return num_nodes


def node_occlusion_mask_host(node_ptr, edge_ptr, src, dst, node_label, node_gid, tag, node_j):
    """twin of igmc_node_occlusion_mask: (edge_keep [edge_ptr[B]], and per graph the dropped node's global id, label
    and rating count, -1 / -1 / -1 where nothing is dropped).  Graph g with tag >= 0 drops every directed edge with its
    node at position node_j[g] as src or dst (``src`` / ``dst``: edge_index rows, batch node ids)"""
    node_ptr, edge_ptr = np.asarray(node_ptr, np.int64), np.asarray(edge_ptr, np.int64)
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    B = len(node_ptr) - 1
    keep = np.ones(int(edge_ptr[-1]), np.uint8)
    rec = np.full((3, B), -1, np.int64)
    for g in range(B):
        pos = node_positions_host(node_label, int(node_ptr[g]), int(node_ptr[g + 1]))
        if tag[g] < 0 or not 0 <= node_j[g] < len(pos):
            continue
        p = int(pos[node_j[g]])
        e = np.arange(edge_ptr[g], edge_ptr[g + 1])
        hit = e[(src[e] == p) | (dst[e] == p)]
        keep[hit] = 0
        rec[:, g] = (node_gid[p], node_label[p], len(hit) // 2)
    return keep, rec


def node_grad_scatter_host(node_ptr, edge_ptr, node_label, in_ptr, in_eid, tag, edge_grad, offsets, out, k=0, K=1):
    """twin of igmc_node_grad_scatter's values for checkpoint ``k`` of ``K``: graph g with tag q >= 0 writes, for its
    node n at position j, the fp32 sum over n's in-list in_eid[in_ptr[n]:in_ptr[n+1]] in list order (the first value
    as it is, then each next one added) of the rating values edge_grad[a] + edge_grad[a + E_g/2] (a the rating's
    user -> item edge) to out[offsets[q] + j] (k = 0), or adds it (k > 0), then divides by K (k = K - 1).  ``out`` [T]
    is updated in place and returned"""
    node_ptr, edge_ptr, offsets = (np.asarray(a, np.int64) for a in (node_ptr, edge_ptr, offsets))
    edge_grad = np.asarray(edge_grad, np.float32)
    for g in range(len(node_ptr) - 1):
        q = int(tag[g])
        if q < 0:
            continue
        e0, m = int(edge_ptr[g]), int(edge_ptr[g + 1] - edge_ptr[g]) // 2
        o = int(offsets[q])
        for j, n in enumerate(node_positions_host(node_label, int(node_ptr[g]), int(node_ptr[g + 1]))):
            v = np.float32(0)
            for t, e in enumerate(in_eid[in_ptr[n]:in_ptr[n + 1]]):
                a = int(e) if int(e) - e0 < m else int(e) - m
                r = np.float32(edge_grad[a] + edge_grad[a + m])
                v = r if t == 0 else np.float32(v + r)
            if k > 0:
                v = np.float32(out[o + j] + v)
            if k == K - 1:
                v = np.float32(v / np.float32(K))
            out[o + j] = v
    return out


# ---- Monte-Carlo-dropout draws (csrc/draws.cu) ----------------------------------------------------------------------
# The result of predict_draws, device tensors: value [P, S] fp32 (draw s of pair p), mean [P] and std [P] fp32 (the
# unbiased standard deviation over the S draws, 0 when S = 1).
Draws = collections.namedtuple("Draws", "value mean std")

DRAWS_HOP_TAG = 4    # sample_state's hop slot of the draw streams: side 0 the edges, side 1 the hidden units


def _check_draw_seed(draw_seed):
    if isinstance(draw_seed, (bool, np.bool_)) or not isinstance(draw_seed, (int, np.integer)):
        raise TypeError("draw_seed must be an integer, not %s" % type(draw_seed).__name__)
    if not 0 <= int(draw_seed) < 2 ** 64:
        raise ValueError("draw_seed must lie in [0, 2^64), not %d" % int(draw_seed))
    return int(draw_seed)


def _draw_inputs(draws, beta, draw_seed, batch_size):
    """None (``draws`` None: the eval scores) or dict(S, beta, draw_seed) of a run over draws, checked on the host:
    ValueError for draws < 1, draws > batch_size (all draws of a pair share one batch), a non-finite beta, or beta
    without draws; NotImplementedError above IGMC_DRAWS_MAX"""
    beta = float(beta)
    if not np.isfinite(beta):
        raise ValueError("beta must be finite, not %r" % beta)
    seed = _check_draw_seed(draw_seed)
    if draws is None:
        if beta != 0.0:
            raise ValueError("beta= ranks by mean + beta * std over draws: pass draws= as well")
        return None
    S = _check_count(draws, "draws", _lib.DRAWS_MAX)
    if S > int(batch_size):
        raise ValueError("draws = %d exceed batch_size = %d: every draw of a pair runs in one batch" % (S, batch_size))
    return dict(S=S, beta=beta, draw_seed=seed)


def draws_expand_host(S, B, pair_u, pair_v, pair_pid, pair_tag):
    """twin of igmc_draws_expand: (links_u, links_v, pair_id, tag, draw) [B] of the G = B // S pairs, S consecutive
    draws each; positions G*S..B-1 copy pair 0 with tag -1 and draw 0"""
    G = B // S
    i = np.arange(B)
    real = i < G * S
    g = np.where(real, i // S, 0)
    return (np.asarray(pair_u, np.int32)[g], np.asarray(pair_v, np.int32)[g], np.asarray(pair_pid, np.int64)[g],
            np.where(real, np.asarray(pair_tag, np.int64)[g], -1), np.where(real, i - g * S, 0).astype(np.int32))


def draw_states_host(draw_seed, pair_id, draw, side):
    """the stream state of each draw: splitmix64(sample_state(draw_seed, pair_id, side, DRAWS_HOP_TAG) + draw), uint64"""
    from oracle.extract_np import splitmix64
    with np.errstate(over="ignore"):
        tag = np.asarray(pair_id, np.int64).astype(np.uint64) * np.uint64(16) + np.uint64(DRAWS_HOP_TAG * 2 + side)
        state = splitmix64(np.uint64(int(draw_seed)) ^ splitmix64(tag))
        return splitmix64(state + np.asarray(draw, np.int64).astype(np.uint32).astype(np.uint64))


def draws_mask_host(edge_ptr, pair_id, tag, draw, adj_dropout, draw_seed):
    """twin of igmc_draws_mask: (edge_keep [edge_ptr[B]], hidden_keep [B * 128]) uint8.  Directed edge e of graph g is
    kept iff the high 32 bits of splitmix64(edge state + (e - edge_ptr[g])) reach keep_thresh(adj_dropout) (none at
    adj_dropout = 1), hidden unit o iff those of splitmix64(hidden state + o) reach keep_thresh(0.5); a graph with tag
    < 0 keeps everything"""
    from oracle.extract_np import splitmix64
    from .models import _keep_threshold
    edge_ptr = np.asarray(edge_ptr, np.int64)
    B = len(edge_ptr) - 1
    pad = np.asarray(tag, np.int64) < 0
    se, sh = draw_states_host(draw_seed, pair_id, draw, 0), draw_states_host(draw_seed, pair_id, draw, 1)
    g = np.repeat(np.arange(B), np.diff(edge_ptr))
    local = (np.arange(edge_ptr[0], edge_ptr[-1]) - edge_ptr[g]).astype(np.uint64)
    keep = np.ones(int(edge_ptr[-1]), np.uint8)
    with np.errstate(over="ignore"):
        ek = (splitmix64(se[g] + local) >> np.uint64(32)) >= np.uint64(_keep_threshold(adj_dropout))
        hk = (splitmix64(sh[:, None] + np.arange(_lib.LIN1_OUT, dtype=np.uint64)[None]) >> np.uint64(32)) >= \
            np.uint64(_keep_threshold(0.5))
    keep[edge_ptr[0]:] = ek | pad[g]
    return keep, (hk | pad[:, None]).reshape(-1).astype(np.uint8)


def _ckpt_mean_host(preds, K, B):
    """the fp32 checkpoint mean [B] of preds [K, B] (ckpt_mean in csrc/common.cuh): fp32 sum in checkpoint order / K"""
    preds = np.asarray(preds, np.float32).reshape(K, B)
    x = preds[0].copy()
    for q in range(1, K):
        x = (x + preds[q]).astype(np.float32)
    if K > 1:
        x = (x / np.float32(K)).astype(np.float32)
    return x


def draws_stats_host(preds, K, B, S, beta=0.0):
    """twin of igmc_draws_stats over one batch: (x [G, S], mean [G], std [G], key [G]) fp32 of its G = B // S pairs; x
    the fp32 checkpoint means, the statistics in fp64 in draw order (Python floats: no fma), each rounded once"""
    import math
    x = _ckpt_mean_host(preds, K, B)
    G = B // S
    x = x[:G * S].reshape(G, S)
    out = np.zeros((3, G), np.float64)
    for g in range(G):
        total = 0.0
        for v in x[g]:
            total += float(v)
        mean, sd = total / S, 0.0
        if S > 1:
            ss = 0.0
            for v in x[g]:
                d = float(v) - mean
                ss += d * d
            sd = math.sqrt(ss / (S - 1))
        out[:, g] = (mean, sd, mean + float(beta) * sd)
    mean, sd, key = out.astype(np.float32)
    return x, mean, sd, key


# ---- rating sessions (csrc/session.cu) ------------------------------------------------------------------------------
def session_rows_host(host, shape, users, session, items, values):
    """numpy twin of igmc_session_plan + _apply: (row_ptr [S+1], col_idx, rating) of the merged session rows.  Restates
    the kernels' steps: the base row of every session (the graph row of users[s], empty for a new user), the stable
    (session, item) order, the last edit of a run kept, classification against the base row and the merge of
    ``graph_update_host``."""
    from .util_functions import _merge_side_host
    users = np.asarray(users, np.int64).reshape(-1)
    session, items, values = (np.asarray(a, np.int64).reshape(-1) for a in (session, items, values))
    nu, _ = shape
    rp, ci, rt = (np.asarray(host[k], np.int64) for k in ("row_ptr", "col_idx", "rating"))
    S = len(users)
    base = [np.arange(rp[u], rp[u + 1]) if u < nu else np.zeros(0, np.int64) for u in users]
    bptr = np.concatenate([[0], np.cumsum([len(b) for b in base])]).astype(np.int64)
    bpos = np.concatenate(base).astype(np.int64) if S else np.zeros(0, np.int64)
    bidx, brt = ci[bpos], rt[bpos]
    if len(session) == 0:                                        # no edits: the base rows
        return bptr.astype(np.int32), bidx.astype(np.int32), brt.astype(np.uint8)
    o = np.lexsort((items, session))                             # stable
    sa, sb, sx = session[o], items[o], values[o]
    keep = np.r_[(sa[1:] != sa[:-1]) | (sb[1:] != sb[:-1]), True] if len(o) else np.zeros(0, bool)
    cls = np.zeros(len(o), np.int64)                             # 0 no-op, 1 insert, 2 change, 3 delete
    lab = np.zeros(len(o), np.int64)
    for i in np.flatnonzero(keep):
        a, b, x = sa[i], sb[i], sx[i]
        row = bidx[bptr[a]:bptr[a + 1]]
        q = int(np.searchsorted(row, b))
        p = bptr[a] + q if q < len(row) and row[q] == b else -1
        if x > 0:
            lab[i] = x - 1
            cls[i] = 1 if p < 0 else (2 if brt[p] != x - 1 else 0)
        elif p >= 0:
            cls[i] = 3
    new_rp, new_ci, new_rt = _merge_side_host(bptr, bidx, brt, S, S, sa, sb, cls, lab)
    return new_rp.astype(np.int32), new_ci.astype(np.int32), new_rt.astype(np.uint8)


class RatingSessions(object):
    """Users described by ratings passed with the query, scored without changing the rating graph.

    Session s is user ``users[s]`` with the edits ``(session[i] == s, items[i], values[i])`` applied to that user's
    row only: ``value`` = rating label + 1 (1..256) inserts or overwrites, 0 deletes (an absent rating: nothing), the
    last occurrence of (s, item) wins.  Ids below ``graph.num_users`` start from that user's graph row, larger ids are
    new users and start from an empty row; two sessions may share an id.  Items must exist.  The merged rows are one
    device CSR of S rows (``row_ptr``, ``col_idx`` ascending, ``rating``), built by csrc/session.cu with one host
    synchronisation (total length and longest row).  Host arrays are validated here (IndexError for ids, ValueError
    for values and lengths); int32 device tensors are checked by the kernel (RuntimeError).  The sessions belong to the
    graph as it was when they were built: using them after ``graph.update`` raises RuntimeError."""

    def __init__(self, graph, users, session=(), items=(), values=()):
        if not isinstance(graph, RatingGraph):
            raise TypeError("sessions are built on a RatingGraph")
        if graph.device is None:
            raise RuntimeError("igmc_b200 rating sessions run on a CUDA device (there is no CPU path)")
        self.graph, dev = graph, graph.device
        if torch.is_tensor(users) and users.device.type == "cuda":
            u = users.reshape(-1).clamp(-1, 2 ** 31 - 1).to(torch.int32).contiguous()
        else:
            u = _host_ids(users, "users", 2 ** 31 - 1)
            u = torch.from_numpy(u.astype(np.int32)).to(dev)
        S = int(u.numel())
        if S < 1:
            raise ValueError("a RatingSessions holds at least one session")
        sess, it, val, D = _update_inputs(session, items, values, S, graph.num_items, ("session", "items", "values"))
        sess, it, val = (_on_device_i32(a, dev) for a in (sess, it, val))
        lib = _lib.load()
        nbytes = C.c_int64(0)
        _lib.check(lib.igmc_session_ws_bytes(S, D, graph.num_items, C.byref(nbytes)), "igmc_session_ws_bytes")
        ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
        header = torch.zeros(2, dtype=torch.int64, device=dev)
        err = torch.zeros(1, dtype=torch.int32, device=dev)
        _lib.check(lib.igmc_session_plan(C.byref(graph._c), u.data_ptr(), S, _lib.ptr(sess), _lib.ptr(it),
                                         _lib.ptr(val), D, ws.data_ptr(), ws.numel(), header.data_ptr(),
                                         err.data_ptr(), _stream_ptr()), "igmc_session_plan")
        hv = torch.cat([header, err.to(torch.int64)]).cpu().numpy()      # the build's one host synchronisation
        _lib.check_kernel_error(int(hv[2]))
        self.nnz, self.max_row_deg = int(hv[0]), int(hv[1])
        if self.nnz > 2 ** 31 - 1:
            raise ValueError("the session rows hold %d ratings, beyond int32" % self.nnz)
        self.users = u
        self.row_ptr = torch.empty(S + 1, dtype=torch.int32, device=dev)
        self.col_idx = torch.empty(max(self.nnz, 1), dtype=torch.int32, device=dev)
        self.rating = torch.empty(max(self.nnz, 1), dtype=torch.uint8, device=dev)
        _lib.check(lib.igmc_session_apply(C.byref(graph._c), u.data_ptr(), S, D, ws.data_ptr(), ws.numel(),
                                          self.row_ptr.data_ptr(), self.col_idx.data_ptr(), self.rating.data_ptr(),
                                          _stream_ptr()), "igmc_session_apply")
        self.num_sessions = S
        self.version = graph.version
        self._c = _lib.Sessions(u.data_ptr(), self.row_ptr.data_ptr(), self.col_idx.data_ptr(),
                                self.rating.data_ptr(), S, self.max_row_deg)
        # the session rows as a CSR over query slots 0..S-1 (no columns): what the candidate kernels read
        self._view = _lib.CSR(self.row_ptr.data_ptr(), self.col_idx.data_ptr(), self.rating.data_ptr(), None, None,
                              S, graph.num_items)
        self._slots = torch.arange(S, dtype=torch.int32, device=dev)

    def __len__(self):
        return self.num_sessions

    def check(self, graph=None):
        """RuntimeError unless the sessions belong to ``graph`` (default: their own) as it is now"""
        if graph is not None and graph is not self.graph:
            raise ValueError("the sessions were built on another RatingGraph")
        if self.graph.version != self.version:
            raise RuntimeError("the rating graph was updated after these sessions were built: their base rows are "
                               "gone; build the sessions again")

    def rows(self):
        """host copies (row_ptr [S+1], col_idx [nnz], rating [nnz]) of the merged rows"""
        n = self.nnz
        return (self.row_ptr.cpu().numpy(), self.col_idx[:n].cpu().numpy(), self.rating[:n].cpu().numpy())


def _check_sessions(sessions, graph=None):
    """``sessions`` when it is a RatingSessions of ``graph`` (default: its own) as it is now"""
    if not isinstance(sessions, RatingSessions):
        raise TypeError("sessions must be a RatingSessions")
    sessions.check(graph)
    return sessions


# ---- counterfactual explanations (csrc/counterfactual.cu) -----------------------------------------------------------
# The result of counterfactual, per query (u, X, Y): found [Q] bool (X ends behind Y), size [Q] int32 (|R|), items and
# ratings [Q, max_removals] int32 (the removed items in greedy order and their labels, -1 past size), score and
# rival_score [Q, max_removals + 1] fp32 (s(u, X) and s(u, Y) before any removal and after each, NaN past size).
Counterfactual = collections.namedtuple("Counterfactual", "found size items ratings score rival_score")


def _counterfactual_inputs(shape, users, items, rivals, max_removals):
    """(users, items, rivals, max_removals) of a counterfactual run checked on the host: ids in range (IndexError),
    equal lengths, items[q] != rivals[q] and max_removals >= 1 (ValueError), max_removals <= IGMC_COUNTERFACTUAL_MAX
    (NotImplementedError)"""
    M = _check_count(max_removals, "max_removals", _lib.COUNTERFACTUAL_MAX)
    users, items, _ = _host_pairs(shape, users, items)
    rivals = _host_ids(rivals, "rivals", shape[1])
    if len(rivals) != len(items):
        raise ValueError("items and rivals must have the same length (%d vs %d)" % (len(items), len(rivals)))
    if np.any(items == rivals):
        q = int(np.flatnonzero(items == rivals)[0])
        raise ValueError("query %d names item %d as its own rival" % (q, int(items[q])))
    return users, items, rivals, M


def _no_counterfactual(Q, M, dev):
    """the Counterfactual of Q queries before any pass: nothing found, nothing removed"""
    i32 = dict(dtype=torch.int32, device=dev)
    nan = dict(fill_value=float("nan"), dtype=torch.float32, device=dev)
    return Counterfactual(torch.zeros(Q, dtype=torch.bool, device=dev), torch.zeros(Q, **i32),
                          torch.full((Q, M), -1, **i32), torch.full((Q, M), -1, **i32), torch.full((Q, M + 1), **nan),
                          torch.full((Q, M + 1), **nan))


def counterfactual_pairs_host(row_ptr, col_idx, rating, num_items, users, items, rivals, removed, size, offsets, step,
                              pos, B):
    """twin of igmc_counterfactual_pairs for positions [pos, pos + B): ((links_u, links_v, pair_id, tag) [4, B] int64,
    (row_users [B], row_ptr [B+1], row_col, row_rating)).  ``removed`` [Q, M]: R ascending in its first size[q]
    entries"""
    offsets = np.asarray(offsets, np.int64)
    Q, P2 = len(offsets) - 1, 2 * int(offsets[-1])
    out = np.zeros((4, B), np.int64)
    cols, rats = [], []
    for i in range(B):
        p = pos + i
        real = p < P2
        if not real:
            p = P2 - 1
        trial = p >> 1
        q = min(int(np.searchsorted(offsets, trial, side="right")) - 1, Q - 1)    # the last q with offsets[q] <= trial
        u, v = int(users[q]), int(rivals[q] if p & 1 else items[q])
        r0, deg = int(row_ptr[u]), int(row_ptr[u + 1] - row_ptr[u])
        keep = np.ones(deg, bool)
        keep[np.asarray(removed[q][:size[q]], np.int64)] = False
        if step > 0:
            keep[np.flatnonzero(keep)[trial - offsets[q]]] = False       # the candidate: the c-th position not in R
        cols.append(np.asarray(col_idx, np.int32)[r0 + np.flatnonzero(keep)])
        rats.append(np.asarray(rating, np.uint8)[r0 + np.flatnonzero(keep)])
        out[:, i] = (u, v, u * num_items + v, p if real else -1)
    rp = np.concatenate([[0], np.cumsum([len(c) for c in cols])]).astype(np.int32)
    return out, (out[0].astype(np.int32), rp, np.concatenate(cols).astype(np.int32),
                 np.concatenate(rats).astype(np.uint8))


def counterfactual_select_host(row_ptr, col_idx, rating, users, items, rivals, offsets, scores, step, state):
    """twin of igmc_counterfactual_select: ``state`` a dict of numpy arrays removed [Q, M] (ascending in its first
    size[q] entries), size [Q], count [Q], found [Q], items / ratings [Q, M], score / rival_score [Q, M + 1], updated in
    place.  ``scores`` [2T]: side s of trial t at 2t + s"""
    offsets = np.asarray(offsets, np.int64)
    scores = np.asarray(scores, np.float32)
    M = state["removed"].shape[1]
    for q in range(len(offsets) - 1):
        o, n = int(offsets[q]), int(offsets[q + 1] - offsets[q])
        if n == 0:
            state["count"][q] = 0
            continue
        u, X, Y = int(users[q]), int(items[q]), int(rivals[q])
        r0, deg, t = int(row_ptr[u]), int(row_ptr[u + 1] - row_ptr[u]), int(state["size"][q])
        sx, sy = scores[2 * o:2 * (o + n):2], scores[2 * o + 1:2 * (o + n):2]
        if step == 0:
            state["score"][q, 0], state["rival_score"][q, 0] = sx[0], sy[0]
            behind = _before(sy[0], Y, sx[0], X)
            state["found"][q] = behind
            state["count"][q] = 0 if behind else deg
            continue
        free = np.setdiff1d(np.arange(deg), state["removed"][q, :t])       # the candidates, ascending
        flip = np.array([_before(b, Y, a, X) for a, b in zip(sx, sy)], bool)
        margin = (sx - sy).astype(np.float32)
        item = np.asarray(col_idx, np.int64)[r0 + free]
        c = int(np.lexsort((item, np.where(np.isnan(margin), 0, margin), np.isnan(margin), ~flip))[0])
        pos = int(free[c])
        state["removed"][q, :t + 1] = np.sort(np.r_[state["removed"][q, :t], pos])
        state["items"][q, t], state["ratings"][q, t] = item[c], int(rating[r0 + pos])
        state["score"][q, t + 1], state["rival_score"][q, t + 1] = sx[c], sy[c]
        state["size"][q] = t + 1
        state["found"][q] = flip[c]
        state["count"][q] = 0 if (flip[c] or t + 1 == M or deg == t + 1) else deg - t - 1
    return state


def counterfactual_host(row_ptr, col_idx, rating, users, items, rivals, max_removals, scorer):
    """``counterfactual``'s greedy search restated on the host, one ``scorer`` call per step: scorer(users, deleted,
    targets) -> fp32 [n], the score of (users[i], targets[i]) with users[i]'s ratings of the items deleted[i] (a list)
    removed.  Returns a ``Counterfactual`` of numpy arrays."""
    users, items, rivals = (np.asarray(a, np.int64).reshape(-1) for a in (users, items, rivals))
    Q, M = len(users), int(max_removals)
    col_idx = np.asarray(col_idx, np.int64)
    found, size = np.zeros(Q, bool), np.zeros(Q, np.int32)
    out_i, out_r = np.full((Q, M), -1, np.int32), np.full((Q, M), -1, np.int32)
    score, rival = np.full((Q, M + 1), np.nan, np.float32), np.full((Q, M + 1), np.nan, np.float32)
    R = [[] for _ in range(Q)]               # removed row positions, in greedy order
    s = np.asarray(scorer(np.r_[users, users], [[]] * (2 * Q), np.r_[items, rivals]), np.float32)
    score[:, 0], rival[:, 0] = s[:Q], s[Q:]
    found[:] = [_before(s[Q + q], rivals[q], s[q], items[q]) for q in range(Q)]
    deg = np.asarray(row_ptr, np.int64)[users + 1] - np.asarray(row_ptr, np.int64)[users]
    active = [q for q in range(Q) if not found[q] and deg[q] > 0]
    while active:
        trials = []                          # (q, candidate position, deleted items)
        for q in active:
            r0 = int(row_ptr[users[q]])
            for pos in range(int(deg[q])):
                if pos not in R[q]:
                    trials.append((q, pos, list(col_idx[r0 + np.array(R[q] + [pos], np.int64)])))
        n = len(trials)
        tu = np.array([users[q] for q, _, _ in trials] * 2, np.int64)
        tt = np.r_[[items[q] for q, _, _ in trials], [rivals[q] for q, _, _ in trials]].astype(np.int64)
        s = np.asarray(scorer(tu, [d for _, _, d in trials] * 2, tt), np.float32)
        best = {}
        for k, (q, pos, d) in enumerate(trials):
            sx, sy = s[k], s[n + k]
            m = np.float32(sx - sy)
            key = (not _before(sy, rivals[q], sx, items[q]), bool(np.isnan(m)), 0.0 if np.isnan(m) else float(m),
                   int(d[-1]))
            if q not in best or key < best[q][0]:
                best[q] = (key, pos, sx, sy)
        for q in active:
            key, pos, sx, sy = best[q]
            t = len(R[q])
            r0 = int(row_ptr[users[q]])
            R[q].append(pos)
            out_i[q, t], out_r[q, t] = col_idx[r0 + pos], int(rating[r0 + pos])
            score[q, t + 1], rival[q, t + 1] = sx, sy
            size[q], found[q] = t + 1, not key[0]
        active = [q for q in active if not found[q] and size[q] < M and size[q] < deg[q]]
    return Counterfactual(found, size, out_i, out_r, score, rival)


# ---- question impact for rating sessions (csrc/elicit.cu) -----------------------------------------------------------
# The result of question_impact, per unit (session, question): impact [P] fp32 (the mean over the targets of the range
# of their scores over the answers) and answer_mean [P, A] fp32 (per answer the mean score of the targets).
QuestionImpact = collections.namedtuple("QuestionImpact", "impact answer_mean")


def _target_rows(targets):
    """``targets`` as a 2-D int64 array: one row (a 1-D list shared by every session) or one row per session"""
    t = np.asarray(targets, np.int64)
    return t.reshape(1, -1) if t.ndim == 1 else t


def _elicit_targets(targets, S, num_items, A, batch_size, queried):
    """(targets int32 [1, W] or [S, W], per_session) of a question-impact run over S sessions, checked on the host:
    IndexError for ids outside [0, num_items) (a 2-D array: [-1, num_items)), ValueError for a 2-D array without one
    row per session, no target slot, a session of ``queried`` whose row has no entry, or A * W > batch_size (every
    score of a question runs in one batch)"""
    if torch.is_tensor(targets):
        targets = targets.detach().cpu().numpy()
    per = _is_rows(targets)
    t = _user_rows(targets, S, num_items, "targets") if per else _host_ids(targets, "targets", num_items)
    t = _target_rows(t)
    W = t.shape[1]
    if W == 0:
        raise ValueError("targets is empty: a question is scored by its effect on at least one target")
    if per:
        bare = np.flatnonzero((t[np.asarray(queried, np.int64)] < 0).all(axis=1))
        if len(bare):
            raise ValueError("session %d has no target: its row of targets holds only -1"
                             % int(np.asarray(queried)[bare[0]]))
    if A * W > int(batch_size):
        raise ValueError("the %d answers x %d target slots of a question exceed batch_size = %d: every score of a "
                         "question runs in one batch; raise batch_size" % (A, W, int(batch_size)))
    return t.astype(np.int32), int(per)


def _question_units(sessions, session, questions):
    """(session, questions) host int64 vectors of explicit units: ids in range (IndexError), equal lengths"""
    sess = _host_ids(session, "session", sessions.num_sessions)
    q = _host_ids(questions, "questions", sessions.graph.num_items)
    if len(sess) != len(q):
        raise ValueError("session and questions must have the same length (%d vs %d)" % (len(sess), len(q)))
    return sess, q


def elicit_pairs_host(row_ptr, col_idx, rating, users, num_items, A, targets, unit_s, unit_q, unit_tag, B):
    """twin of igmc_elicit_pairs: ((links_u, links_v, pair_id, tag) [4, B] int64, sess [B] int32, (row_users [G*A],
    row_ptr [G*A+1], row_col, row_rating)).  ``row_ptr`` / ``col_idx`` / ``rating``: the session rows, ``users`` the
    sessions' user ids, ``targets`` one list [W] or a row per session [S, W] (-1 = empty slot)"""
    t2 = _target_rows(targets)
    W = t2.shape[1]
    U = A * W
    G = B // U
    out = np.zeros((4, B), np.int64)
    sess = np.zeros(B, np.int32)
    for i in range(B):
        real = i < G * U
        g, a = (i // U, (i % U) // W) if real else (0, 0)
        s, q = int(unit_s[g]), int(unit_q[g])
        t = int(t2[s if len(t2) > 1 else 0, i % W]) if real else -1
        u = int(users[s])
        v = t if t >= 0 else q
        out[:, i] = (u, v, u * num_items + v, int(unit_tag[g]) if t >= 0 else -1)
        sess[i] = g * A + a
    ru, cols, rats = [], [], []
    for r in range(G * A):
        g, a = divmod(r, A)
        s, q = int(unit_s[g]), int(unit_q[g])
        row = np.asarray(col_idx[row_ptr[s]:row_ptr[s + 1]], np.int64)
        p = int(np.searchsorted(row, q))
        ru.append(int(users[s]))
        cols.append(np.insert(row, p, q))
        rats.append(np.insert(np.asarray(rating[row_ptr[s]:row_ptr[s + 1]], np.int64), p, a))
    rp = np.concatenate([[0], np.cumsum([len(c) for c in cols])]).astype(np.int32)
    cat = lambda xs, dt: (np.concatenate(xs) if xs else np.zeros(0)).astype(dt)   # noqa: E731
    return out, sess, (np.asarray(ru, np.int32), rp, cat(cols, np.int32), cat(rats, np.uint8))


def _impact_of(x):
    """impact and answer means of one question from its scores x [A][n] (fp32, real targets in slot order): in fp64
    (Python floats: no fma) in slot order, each rounded once; a NaN score makes the impact NaN"""
    A, n = len(x), len(x[0])
    total, nan = 0.0, False
    for w in range(n):
        col = [float(x[a][w]) for a in range(A)]
        nan = nan or any(np.isnan(col))
        total += max(col) - min(col)
    means = []
    for a in range(A):
        m = 0.0
        for w in range(n):
            m += float(x[a][w])
        means.append(m / n)
    return np.float32(np.nan if nan else total / n), np.asarray(means).astype(np.float32)


def elicit_stats_host(preds, K, B, A, W, tag):
    """twin of igmc_elicit_stats over one batch: (impact [G], answer_mean [G, A], unit tag [G]) of its G = B // (A * W)
    units; a unit without real slots has impact 0, answer_mean NaN and tag -1"""
    x = _ckpt_mean_host(preds, K, B)
    tag = np.asarray(tag, np.int64)
    U = A * W
    G = B // U
    impact, mean, utag = np.zeros(G, np.float32), np.full((G, A), np.nan, np.float32), np.full(G, -1, np.int64)
    for g in range(G):
        real = [w for w in range(W) if tag[g * U + w] >= 0]
        if real:
            utag[g] = tag[g * U + real[-1]]
            impact[g], mean[g] = _impact_of([[x[g * U + a * W + w] for w in real] for a in range(A)])
    return impact, mean, utag


def question_impact_host(A, targets, session, questions, scorer):
    """``question_impact`` restated on the host, one ``scorer`` call: scorer(session, question, answer, target) ->
    fp32 [m], the score of (the user of session[i], target[i]) with session[i]'s row plus the rating (question[i],
    answer[i]) (label).  ``targets`` one list [W] or a row per session [S, W] (-1 = empty slot).  Returns
    (impact [P], answer_mean [P, A]) fp32"""
    t2 = _target_rows(targets)
    trials, spans = [], []
    for s, q in zip(np.asarray(session, np.int64), np.asarray(questions, np.int64)):
        ts = [int(t) for t in t2[s if len(t2) > 1 else 0] if t >= 0]
        spans.append(len(ts))
        trials += [(int(s), int(q), a, t) for a in range(A) for t in ts]
    x = np.asarray(scorer(*(np.array([tr[k] for tr in trials], np.int64) for k in range(4))), np.float32) \
        if trials else np.zeros(0, np.float32)
    impact, mean, o = np.zeros(len(spans), np.float32), np.zeros((len(spans), A), np.float32), 0
    for p, n in enumerate(spans):
        impact[p], mean[p] = _impact_of(x[o:o + A * n].reshape(A, n))
        o += A * n
    return impact, mean


def elicit_host(row_ptr, col_idx, num_items, A, n, targets, scorer, questions=None):
    """``elicit`` restated on the host: per session its questions (every item, one list [Q] or a row per session with
    -1 padding; minus the items of its row ``col_idx[row_ptr[s]:row_ptr[s+1]]``), their impacts by
    ``question_impact_host`` and the first n in ``recommend``'s order (impact descending, item ascending, NaN last).
    Returns (items [S, n] int64, impact [S, n] fp32) padded with -1 / -inf"""
    S = len(row_ptr) - 1
    qs = None if questions is None else _target_rows(questions)
    sess, qu = [], []
    for s in range(S):
        cand = np.arange(num_items) if qs is None else np.unique(qs[s if len(qs) > 1 else 0])
        cand = cand[(cand >= 0) & ~np.isin(cand, np.asarray(col_idx[row_ptr[s]:row_ptr[s + 1]], np.int64))]
        sess += [s] * len(cand)
        qu += list(cand)
    impact, _ = question_impact_host(A, targets, sess, qu, scorer)
    sess, qu = np.asarray(sess, np.int64), np.asarray(qu, np.int64)
    top_i, top_s = np.full((S, n), -1, np.int64), np.full((S, n), -np.inf, np.float32)
    for s in range(S):
        top_s[s], top_i[s] = rank_host(impact[sess == s], qu[sess == s], n)
    return top_i, top_s


class _TrialRows(object):
    """one batch slot's trial rows of a counterfactual or question-impact pass, and their igmc_sessions_t (``_c``):
    what ``SubgraphExtractor.extract`` takes as ``sessions``"""

    def __init__(self, users, row_ptr, col_idx, rating):
        self.users, self.row_ptr, self.col_idx, self.rating = users, row_ptr, col_idx, rating
        self.cap = int(col_idx.numel())
        self.max_row_deg = 0
        self._c = _lib.Sessions(users.data_ptr(), row_ptr.data_ptr(), col_idx.data_ptr(), rating.data_ptr(),
                                int(users.numel()), 0)


# ---- the engine -----------------------------------------------------------------------------------------------------
class InferenceEngine(object):
    """Pipelined, graph-replayed scoring of candidate pairs (module docstring).  ``checkpoints``: state_dict files of
    ``model``'s class, each scored and averaged (fp32 sum in checkpoint order / K); None scores ``model``'s own
    parameters as they are when a run starts.

        eng = InferenceEngine(model, graph, batch_size=256)
        eng.start_recommend(users, k)          # or start_pairs(users, items) / start_explain / start_attribute(users, items, m)
                                               # or start_recommend_users(items, k): per item its best users
                                               # or start_explain_nodes / start_attribute_nodes(users, items, m)
                                               # or start_draws(users, items, S): S dropout draws per pair
                                               # or start_counterfactual(users, items, rivals, max_removals)
                                               # or start_elicit(sessions, n, targets) / start_question_impact(...)
        while eng.step():
            pass
        top_items, top_scores = eng.finish()   # (predict: scores; explain: an Explanation; attribute: an Attribution;
                                               # counterfactual: a Counterfactual; question_impact: a QuestionImpact)

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
    def start_recommend(self, users, k, items=None, exclude_rated=True, retrieve=None, draws=None, beta=0.0,
                        draw_seed=0):
        """plan a ranking run (one host sync: the candidate total).  ``items``: one candidate list for every user, or
        a 2-D [U, width] array of per-user lists (-1 = empty slot); ``retrieve=M``: each user's M items with the most
        bridges (``corated_items``) are its candidates.  ``draws=S``: rank by mean + beta * std over S draws
        (``recommend``).  Returns the number of candidate pairs."""
        g = self.graph
        d = _draw_inputs(draws, beta, draw_seed, self.B)
        users = _host_ids(users, "users", g.num_users)
        k, m, cand, rows = _ranking_inputs(k, self.B, items, retrieve, len(users), g.num_items)
        slots = torch.from_numpy(users.astype(np.int32)).to(self.dev)

        def rated():     # the users' summed row lengths (host row pointers: a copy after an update)
            rp = g.host["row_ptr"]
            return int((rp[users + 1] - rp[users]).sum())
        return self._plan_ranking(slots, k, m, cand, rows, exclude_rated, rated,
                                  "igmc_corated_items", (C.byref(g._c), slots.data_ptr(), len(users)), draws=d)

    def start_session_recommend(self, sessions, k, items=None, exclude_rated=True, retrieve=None, draws=None,
                                beta=0.0, draw_seed=0):
        """plan a ranking run over the sessions (``recommend_sessions``): query slot s is session s, its candidates and
        rated items come from its session row.  Arguments as ``start_recommend``'s.  Returns the number of candidate
        pairs."""
        d = _draw_inputs(draws, beta, draw_seed, self.B)
        sessions = self._session_slots(sessions)
        k, m, cand, rows = _ranking_inputs(k, self.B, items, retrieve, sessions.num_sessions, self.graph.num_items)
        return self._plan_ranking(sessions._slots, k, m, cand, rows, exclude_rated, lambda: sessions.nnz,
                                  "igmc_corated_sessions", (C.byref(self.graph._c), C.byref(sessions._c)), sessions,
                                  draws=d)

    def start_recommend_users(self, items, k, users=None, exclude_rated=True, retrieve=None, draws=None, beta=0.0,
                              draw_seed=0):
        """plan an item-side ranking run (``recommend_users``): per query item its best users.  ``users``: one
        candidate list for every item, or a 2-D [I, width] array of per-item lists (-1 = empty slot); ``retrieve=M``:
        each item's M users with the most bridges (``corated_users``).  The candidate kernels run on the graph's
        transposed view.  ``draws`` / ``beta`` / ``draw_seed`` as ``start_recommend``'s.  Returns the number of
        candidate pairs."""
        g = self.graph
        d = _draw_inputs(draws, beta, draw_seed, self.B)
        items = _host_ids(items, "items", g.num_items)
        k, m, cand, rows = _ranking_inputs(k, self.B, users, retrieve, len(items), g.num_users, "users")
        slots = torch.from_numpy(items.astype(np.int32)).to(self.dev)

        def rated():     # the items' summed column lengths (host column pointers: a copy after an update)
            cp = g.host["col_ptr"]
            return int((cp[items + 1] - cp[items]).sum())
        return self._plan_ranking(slots, k, m, cand, rows, exclude_rated, rated,
                                  "igmc_corated_users", (C.byref(g._ct), slots.data_ptr(), len(items)), by_item=True,
                                  draws=d)

    def _plan_ranking(self, slots, k, m, cand, rows, exclude_rated, rated, retriever, args, sessions=None,
                      by_item=False, draws=None, **fields):
        """the plan of a ranking run over the query slots ``slots`` (int32, on the device) with ``_ranking_inputs``'
        (k, m, cand, rows): the candidate plan over every item or the list ``cand`` (``rated()``: the slots' summed row
        lengths, room for their rated positions in the list), or per-slot rows from ``rows`` or from the retriever entry
        ``retriever`` (leading arguments ``args``).  ``sessions``: the slots are these sessions.  ``by_item``: the
        slots are items and the candidates users - the plan runs on the graph's transposed view, whose rows are the
        items' columns.  ``draws``: ``_draw_inputs``' dict of a run ranked by draws.  ``fields``: further run fields
        (a question-ranking run's).  Returns the number of candidate pairs."""
        U, dev, g = int(slots.numel()), self.dev, self.graph
        run = dict(kind="recommend", U=U, k=k, version=g.version, sessions=sessions, users=slots, by_item=by_item,
                   top_s=torch.full((U, k), -float("inf"), dtype=torch.float32, device=dev),
                   top_i=torch.full((U, k), -1, dtype=torch.int64, device=dev), **self._draw_run(draws), **fields)
        self.run = run
        if U == 0 or (cand is not None and len(cand) == 0) or (rows is not None and rows.shape[1] == 0):
            run["P"] = 0
            return 0
        if m is not None:
            rows, _ = _corated(self.lib, g.shape[::-1] if by_item else g.shape, retriever, args, U, m, exclude_rated,
                               self.extractor.err, self._retrieve_ws)
        if rows is not None:
            return self._plan_lists(run, rows, exclude_rated)
        Cd = self._query_candidates(run, exclude_rated)
        run["cand"] = None if cand is None else torch.from_numpy(cand.astype(np.int32)).to(dev)
        if cand is not None and exclude_rated:
            run["rated_off"] = torch.zeros(U + 1, dtype=torch.int64, device=dev)
            run["rated_pos"] = torch.zeros(max(rated(), 1), dtype=torch.int32, device=dev)
        Cd.cand, Cd.num_cand = _lib.ptr(run["cand"]), 0 if cand is None else len(cand)
        Cd.rated_off, Cd.rated_pos = _lib.ptr(run.get("rated_off")), _lib.ptr(run.get("rated_pos"))
        _lib.check(self.lib.igmc_candidate_plan(C.byref(self._csr(run)), C.byref(Cd), self.extractor.err.data_ptr(),
                                                _stream_ptr()), "igmc_candidate_plan")
        return self._planned(run)

    def _plan_lists(self, run, rows, exclude_rated):
        """the plan of a run over per-slot candidate rows [U, width] (a host array or a device tensor):
        igmc_candidate_lists compacts them into run["lists"] and user_off"""
        U, dev, err = run["U"], self.dev, self.extractor.err
        rows = run["rows"] = torch.as_tensor(rows, device=dev).to(torch.int32).contiguous()
        width = int(rows.shape[1])
        run["lists"] = torch.empty(max(U * width, 1), dtype=torch.int32, device=dev)
        nbytes = C.c_int64(0)
        _lib.check(self.lib.igmc_candidate_lists_ws_bytes(U, width, C.byref(nbytes)), "igmc_candidate_lists_ws_bytes")
        run["lists_ws"] = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev)
        Cd = self._query_candidates(run, exclude_rated)
        _lib.check(self.lib.igmc_candidate_lists(C.byref(self._csr(run)), C.byref(Cd), rows.data_ptr(), width,
                                                 run["lists"].data_ptr(), run["lists_ws"].data_ptr(),
                                                 run["lists_ws"].numel(), err.data_ptr(), _stream_ptr()),
                   "igmc_candidate_lists")
        Cd.cand, Cd.per_user = run["lists"].data_ptr(), 1
        return self._planned(run)

    def _query_candidates(self, run, exclude_rated):
        """run["Cd"] over the query slots run["users"], with their count prefix run["user_off"] (zeroed)"""
        U = run["U"]
        run["user_off"] = torch.zeros(U + 1, dtype=torch.int64, device=self.dev)
        Cd = run["Cd"] = _lib.Candidates()
        Cd.users, Cd.user_off, Cd.num_query = run["users"].data_ptr(), run["user_off"].data_ptr(), U
        Cd.exclude_rated = int(bool(exclude_rated))
        return Cd

    def _planned(self, run):
        """after the plan of a ranking run: its pair total (the run's one host sync), the first batch primed.  Returns
        the total."""
        run["Cd"].num_pairs = run["P"] = int(run["user_off"][run["U"]].item())
        if run["P"] > 0:
            self._prime()
        return run["P"]

    def _start_rescore(self, slots, user_off, cand, P, top_s, top_i):
        """a ranking run over a plan made by the caller (``RecommendationCache``: igmc_rescore_plan): query slots
        ``slots`` (int32 on the device), per slot its items in ``cand`` at ``user_off`` (P pairs in all, known on the
        host), merged into the lists top_s / top_i [U, depth] as they stand instead of lists of -inf.  No host sync
        beyond the model's plan of a new batch shape."""
        run = self.run = dict(kind="recommend", U=int(slots.numel()), k=int(top_s.shape[1]), version=self.graph.version,
                              sessions=None, users=slots, by_item=False, top_s=top_s, top_i=top_i, user_off=user_off,
                              cand=cand, P=int(P))
        Cd = run["Cd"] = _lib.Candidates()
        Cd.users, Cd.user_off, Cd.num_query, Cd.cand = slots.data_ptr(), user_off.data_ptr(), run["U"], cand.data_ptr()
        Cd.per_user, Cd.num_pairs = 1, run["P"]
        if run["P"] > 0:
            self._prime()
        return run["P"]

    def start_pairs(self, users, items):
        """plan a run over the explicit pairs (users[i], items[i]).  Returns their number."""
        users, items, _ = _host_pairs(self.graph.shape, users, items)
        return self._start_explicit("pairs", users, items)

    def start_draws(self, users, items, draws, draw_seed=0):
        """plan a run of ``draws`` Monte-Carlo-dropout draws of each explicit pair (users[i], items[i])
        (``predict_draws``).  Returns the number of pairs."""
        d = _draw_inputs(draws, 0.0, draw_seed, self.B)
        users, items, _ = _host_pairs(self.graph.shape, users, items)
        P, S, f32 = len(users), d["S"], dict(dtype=torch.float32, device=self.dev)
        return self._start_explicit("draws", users, items, value=torch.empty(P, S, **f32),
                                    mean=torch.empty(P, **f32), std=torch.empty(P, **f32), **self._draw_run(d))

    def _draw_run(self, d):
        """the run fields of a run over draws (``_draw_inputs``' dict d, or None: none), the slots' draw buffers
        allocated: per slot the G pairs of a batch before their expansion, the draw index and the hidden mask"""
        if d is None:
            return {}
        i32, i64 = dict(dtype=torch.int32, device=self.dev), dict(dtype=torch.int64, device=self.dev)
        for s in self.slots:
            if "draw" not in s:
                s.update(gu=torch.zeros(self.B, **i32), gv=torch.zeros(self.B, **i32), gpid=torch.zeros(self.B, **i64),
                         gtag=torch.zeros(self.B, **i64), draw=torch.zeros(self.B, **i32),
                         hkeep=torch.ones(self.B * _lib.LIN1_OUT, dtype=torch.uint8, device=self.dev))
        return dict(d, G=self.B // d["S"], keys=torch.empty(self.B, dtype=torch.float32, device=self.dev))

    def _draw_masks(self):
        """each slot's edge mask sized for the extractor's batch edge capacity, and its dropout descriptor: the
        training-mode forward with both rates 0 and the slot's injected edge and hidden masks"""
        self.extractor._sync_graph()
        ecap = self.extractor._out_caps(self.B)[1]
        for s in self.slots:
            if s.get("keep") is None or s["keep"].numel() < ecap:
                s["keep"] = torch.ones(ecap, dtype=torch.uint8, device=self.dev)
            d = self.model.make_dropout(False)[0]
            d.edge_keep, d.hidden_keep = s["keep"].data_ptr(), s["hkeep"].data_ptr()
            s["drop"] = (d, [s["keep"], s["hkeep"]])

    # ---- rating sessions ----------------------------------------------------------------------------------------
    def _csr(self, run):
        """the rows the candidate kernels read: the graph's, its transposed view on an item-side run, or a session
        run's rows as a CSR over its sessions"""
        if run.get("by_item"):
            return self.graph._ct
        return run["sessions"]._view if run.get("sessions") is not None else self.graph._c

    def _session_slots(self, sessions):
        """``sessions`` checked against the engine's graph, and the per-slot session index buffers"""
        _check_sessions(sessions, self.graph)
        for s in self.slots:
            if "sess" not in s:
                s["sess"] = torch.zeros(self.B, dtype=torch.int32, device=self.dev)
        return sessions

    def start_session_pairs(self, sessions, session, items):
        """plan a run over the pairs (sessions.users[session[i]], items[i]), each scored with its target user's row
        taken from session ``session[i]`` (``predict_sessions``).  Returns their number."""
        sessions = self._session_slots(sessions)
        sess, items, _ = _host_pairs((sessions.num_sessions, self.graph.num_items), session, items, first="session")
        return self._start_explicit("pairs", sess, items, sessions=sessions)

    def start_explain(self, users, items, m=None):
        """plan an explanation run over the explicit pairs (users[i], items[i]) (``explain_pairs``): the base pass
        scores them and counts their subgraphs' ratings; once it is done, ``step`` reads the total (the run's one host
        sync) and goes on with the occlusion pass.  ``m``: keep each pair's first m ratings.  Returns the number of
        pairs."""
        m = _check_top(m)
        users, items, _ = _host_pairs(self.graph.shape, users, items)
        return self._start_explicit("explain", users, items, m=m, phase="base")

    def start_attribute(self, users, items, m=None):
        """plan an attribution run over the explicit pairs (users[i], items[i]) (``attribute_pairs``): the base pass of
        ``start_explain``, then (after the run's one host sync, the rating total) a gradient pass over the same pairs.
        ``m``: keep each pair's first m ratings.  Returns the number of pairs."""
        m = _check_top(m)
        users, items, _ = _host_pairs(self.graph.shape, users, items)
        return self._start_explicit("attribute", users, items, m=m, phase="base")

    def start_explain_nodes(self, users, items, m=None):
        """plan a node explanation run (``explain_nodes``): ``start_explain``'s two passes with the non-target nodes
        of each pair's subgraph as positions; the base pass counts them.  Returns the number of pairs."""
        m = _check_top(m)
        users, items, _ = _host_pairs(self.graph.shape, users, items)
        return self._start_explicit("explain_nodes", users, items, m=m, phase="base")

    def start_attribute_nodes(self, users, items, m=None):
        """plan a node attribution run (``attribute_nodes``): ``start_attribute``'s two passes, each node's gradient
        the sum of its ratings' gradients.  Returns the number of pairs."""
        m = _check_top(m)
        users, items, _ = _host_pairs(self.graph.shape, users, items)
        return self._start_explicit("attribute_nodes", users, items, m=m, phase="base")

    def start_counterfactual(self, users, items, rivals, max_removals=10):
        """plan a counterfactual run (``counterfactual``) over the queries (users[q], items[q], rivals[q]): a base pass
        scores each query's two pairs, then every trial pass scores each active query's trials (its row without R and
        without one more position, the pairs (u, X) and (u, Y)) and igmc_counterfactual_select appends the best one
        to R.  Each pass ends in one host sync (its trial total).  Returns the number of queries."""
        g, dev = self.graph, self.dev
        users, items, rivals, M = _counterfactual_inputs(g.shape, users, items, rivals, max_removals)
        Q = len(users)
        run = dict(kind="counterfactual", P=Q, version=g.version, M=M, step=0, row_deg=g.max_row_deg,
                   out=_no_counterfactual(Q, M, dev), removed=torch.zeros(Q, M, dtype=torch.int32, device=dev),
                   count=torch.ones(Q, dtype=torch.int32, device=dev),
                   offsets=torch.zeros(Q + 1, dtype=torch.int64, device=dev))
        self.run = run
        if Q == 0:
            return 0
        run["pu"], run["px"], run["py"] = (torch.from_numpy(a.astype(np.int32)).to(dev) for a in (users, items, rivals))
        run["Qd"] = _lib.Counterfactual(run["pu"].data_ptr(), run["px"].data_ptr(), run["py"].data_ptr(),
                                        run["out"].size.data_ptr(), run["removed"].data_ptr(), Q, M)
        self._trial_rows(self.B, g.max_row_deg)
        self._trial_pass()
        return Q

    def _trial_rows(self, rows, row_deg):
        """each slot's trial rows: room for ``rows`` rows of up to ``row_deg`` ratings, as the session rows
        igmc_extract_sessions reads (sess[g] of slot g names its trial row)"""
        n = rows * max(row_deg, 1)
        if n > 2 ** 31 - 1:
            raise NotImplementedError("%d trial rows of up to %d ratings = %d entries, beyond int32"
                                      % (rows, row_deg, n))
        i32 = dict(dtype=torch.int32, device=self.dev)
        for s in self.slots:
            t = s.get("trial")
            if t is None or t.cap < n:
                t = s["trial"] = _TrialRows(torch.zeros(self.B, **i32), torch.zeros(self.B + 1, **i32),
                                            torch.zeros(n, **i32), torch.zeros(n, dtype=torch.uint8, device=self.dev))
            if "sess" not in s:
                s["sess"] = torch.zeros(self.B, **i32)
            t.max_row_deg = row_deg
            t._c.max_row_deg = t.max_row_deg

    # ---- question impact ----------------------------------------------------------------------------------------
    def start_elicit(self, sessions, n, targets, questions=None):
        """plan a question-ranking run (``elicit``): the units (session s, question q) are the candidate pairs of a
        ranking run over the session rows (``questions`` as ``start_session_recommend``'s ``items``, rated items
        always excluded); each batch holds G units of A answers x W targets, and each unit's impact is merged into its
        session's top-n list.  One host sync (the unit total).  Returns the number of units."""
        sessions = self._session_slots(sessions)
        S = sessions.num_sessions
        n, _, cand, rows = _ranking_inputs(n, self.B, questions, None, S, self.graph.num_items, "questions")
        fields = self._elicit_run(sessions, targets, np.arange(S))
        return self._plan_ranking(sessions._slots, n, None, cand, rows, True, lambda: sessions.nnz, None, None,
                                  sessions, **fields)

    def start_question_impact(self, sessions, session, questions, targets):
        """plan a run over explicit units (session[i], questions[i]) (``question_impact``): per unit its impact and
        answer means.  ValueError for a question the session already rated.  Returns the number of units."""
        sessions = self._session_slots(sessions)
        sess, q = _question_units(sessions, session, questions)
        fields = self._elicit_run(sessions, targets, sess)
        if len(sess):
            rp, ci, _ = sessions.rows()
            for s, item in zip(sess, q):
                row = ci[rp[s]:rp[s + 1]]
                p = int(np.searchsorted(row, item))
                if p < len(row) and row[p] == item:
                    raise ValueError("session %d already rated item %d: a rated item is not a question"
                                     % (int(s), int(item)))
        f32 = dict(dtype=torch.float32, device=self.dev)
        return self._start_explicit("question_impact", sess, q, sessions=sessions,
                                    impact=torch.empty(len(sess), **f32),
                                    answer_mean=torch.empty(len(sess), fields["A"], **f32), **fields)

    def _elicit_run(self, sessions, targets, queried):
        """the run fields of a question-impact run (``_elicit_targets``' targets on the device, the answers A, target
        width W, units per batch G and the trial rows' longest row), the slots' unit and trial-row buffers allocated"""
        A, dev = self.model.num_relations, self.dev
        t, per = _elicit_targets(targets, sessions.num_sessions, self.graph.num_items, A, self.B, queried)
        W = t.shape[1]
        L = sessions.max_row_deg + 1            # a trial row: the session row and the question
        self._trial_rows(self.B // W, L)        # G * A <= B / W trial rows per batch
        i32, i64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.int64, device=dev)
        for s in self.slots:
            if "gu" not in s:
                s.update(gu=torch.zeros(self.B, **i32), gv=torch.zeros(self.B, **i32), gpid=torch.zeros(self.B, **i64),
                         gtag=torch.zeros(self.B, **i64))
        G = self.B // (A * W)
        return dict(A=A, W=W, G=G, targets=torch.from_numpy(t).to(dev), per_session=per, row_deg=L,
                    keys=torch.empty(G, dtype=torch.float32, device=dev))

    def _elicit_stats(self, preds, s):
        """a batch of units: per unit its impact merged into its session's top-n list (ranking), or its impact and
        answer means scattered to its index"""
        run, st = self.run, _stream_ptr()
        rank = run["kind"] == "recommend"
        outs = (run["keys"], None, None) if rank else (None, run["impact"], run["answer_mean"])
        _lib.check(self.lib.igmc_elicit_stats(preds.data_ptr(), self.K, self.B, run["A"], run["W"],
                                              s["tag"].data_ptr(), *(_lib.ptr(t) for t in outs), st),
                   "igmc_elicit_stats")
        if rank:
            _lib.check(self.lib.igmc_topk_merge(run["keys"].data_ptr(), 1, run["G"], s["gtag"].data_ptr(),
                                                s["gv"].data_ptr(), run["k"], run["top_s"].data_ptr(),
                                                run["top_i"].data_ptr(), st), "igmc_topk_merge")

    def _trial_pass(self):
        """the next pass of a counterfactual run: the offsets of the queries' trial counts, their total T (the pass's
        host sync) and its 2T positions primed.  Returns True when it has trials."""
        run = self.run
        _lib.check(self.lib.igmc_explain_offsets(run["count"].data_ptr(), run["P"], run["offsets"].data_ptr(),
                                                 _stream_ptr()), "igmc_explain_offsets")
        T = int(run["offsets"][run["P"]].item())
        if T == 0:
            run["steps"] = run["done"] = 0
            return False
        run["scores"] = torch.empty(2 * T, dtype=torch.float32, device=self.dev)
        self._prime(2 * T)
        return True

    def _select_trials(self):
        """after a pass of a counterfactual run: each query's best trial appended (igmc_counterfactual_select), then
        the next pass.  Returns True when it has trials."""
        run, out = self.run, self.run["out"]
        _lib.check(self.lib.igmc_counterfactual_select(C.byref(self.graph._c), C.byref(run["Qd"]),
                                                       run["offsets"].data_ptr(), run["scores"].data_ptr(),
                                                       run["step"], run["count"].data_ptr(), out.found.data_ptr(),
                                                       out.items.data_ptr(), out.ratings.data_ptr(),
                                                       out.score.data_ptr(), out.rival_score.data_ptr(),
                                                       self.extractor.err.data_ptr(), _stream_ptr()),
                   "igmc_counterfactual_select")
        run["step"] += 1
        return self._trial_pass()

    def start_pair_gradients(self, users, items, y=None):
        """plan a per-pair gradient run (``pair_gradients``) over the explicit pairs: per checkpoint the gradient of
        l_i = (f_i - y_i)^2 (``y`` given) or of the score f_i into run["out"] [K, P, param_count].  Returns P."""
        _check_per_pair_model(self.model)
        users, items, y = _host_pairs(self.graph.shape, users, items, y)
        out = torch.zeros(self.K, len(users), self.model._cmodel.param_count, dtype=torch.float32, device=self.dev)
        return self._start_explicit("pair_gradients", users, items, phase="pgrad", out=out, y=self._dev_y(y))

    def start_influence(self, train, test, k, lrs=None):
        """plan an influence run (``influence``): a test-gradient pass over ``test`` = (users, items[, y]) that stores
        every checkpoint's test gradients, then a training pass over ``train`` = (users, items, y) that accumulates
        S[b, t] = sum_k lrs[k] <G_b, G_t> per batch and merges it into each test pair's top-k lists.  Returns the
        number of test pairs."""
        _check_per_pair_model(self.model)
        k, tr, te, lrs = _influence_inputs(self.graph.shape, train, test, k, self.B, lrs, self.K)
        T, m, dev = len(te[0]), self.model._cmodel, self.dev
        f32, i64 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int64, device=dev)
        FW = self.lib.igmc_pair_factor_count(C.byref(m))
        extra = dict(phase="test", train=tr, lrs=lrs, k=k, T=T, y=self._dev_y(te[2]),
                     tconv=torch.zeros(self.K, T, m.conv_param_count, **f32), tfac=torch.zeros(self.K, T, FW, **f32),
                     pro_i=torch.full((T, k), -1, **i64), pro_v=torch.full((T, k), -float("inf"), **f32),
                     con_i=torch.full((T, k), -1, **i64), con_v=torch.full((T, k), float("inf"), **f32), self_out=None)
        return self._start_explicit("influence", te[0], te[1], **extra)

    def start_self_influence(self, train, lrs=None):
        """plan a self-influence run (``self_influence``) over ``train`` = (users, items, y).  Returns its size."""
        _check_per_pair_model(self.model)
        tr = _host_pairs(self.graph.shape, *_split_pairs(train, "train", True), name="train")
        lrs = _check_lrs(lrs, self.K)
        N = len(tr[0])
        self._start_explicit("self_influence", tr[0], tr[1], phase="train", lrs=lrs, T=0, y=self._dev_y(tr[2]),
                             self_out=torch.zeros(N, dtype=torch.float32, device=self.dev))
        if N:
            self._train_buffers()
        return N

    def _dev_y(self, y):
        return None if y is None else torch.from_numpy(y).to(self.dev)

    def _train_buffers(self):
        """the training pass's per-batch buffers: conv rows [B, PC], factor rows, S [B, T] and the GEMM workspace"""
        run, m, dev = self.run, self.model._cmodel, self.dev
        f32 = dict(dtype=torch.float32, device=dev)
        FW = self.lib.igmc_pair_factor_count(C.byref(m))
        nbytes = C.c_int64(0)
        _lib.check(self.lib.igmc_influence_ws_bytes(C.byref(m), self.B, run["T"], C.byref(nbytes)),
                   "igmc_influence_ws_bytes")
        run["bufs"] = dict(conv=torch.zeros(self.B, m.conv_param_count, **f32), fac=torch.zeros(self.B, FW, **f32),
                           S=torch.zeros(self.B, max(run["T"], 1), **f32),
                           ws=torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=dev))

    def _start_train_pass(self):
        """after the test-gradient pass of an influence run: the training pairs primed.  Returns True when there are
        any."""
        run = self.run
        users, items, y = run["train"]
        run["phase"], run["P"], run["y"] = "train", len(users), self._dev_y(y)
        if run["P"] == 0:
            run["steps"] = run["done"] = 0
            return False
        self._explicit_pairs(run, users, items)
        self._train_buffers()
        self._prime()
        return True

    def _pair_grad_step(self, slot):
        """per parameter set: the training-mode forward of batch ``slot`` without dropout, the seed (loss or score),
        the backward and the per-graph gradients - scattered to the pairs' rows (pair_gradients, the test-gradient
        pass) or kept per batch and accumulated into the influence values and / or self-influence (training pass);
        after the last checkpoint of a training batch the merge into the top-k lists"""
        m, b, s, run, lib = self.model, self.batches[slot], self.slots[slot], self.run, self.lib
        phase, tag, B = run["phase"], s["tag"].data_ptr(), self.B
        st = _stream_ptr()
        y = _lib.ptr(run["y"])
        bufs = run.get("bufs")
        dpred = self.preds[0]
        for j in range(self.K):
            with self._params(j):
                pred, saved = m._launch_forward(b, True, self.drop)
                ws = saved["ws"]
                _lib.check(lib.igmc_pair_seed(pred.data_ptr(), y, tag, B, float(m._cmodel.multiply_by),
                                              dpred.data_ptr(), st), "igmc_pair_seed")
                m._launch_backward(b, self.drop, saved, dpred)
                if phase == "pgrad":
                    grad, fac, scatter, full = run["out"][j], None, 1, 1
                elif phase == "test":
                    grad, fac, scatter, full = run["tconv"][j], run["tfac"][j], 1, 0
                else:
                    grad, fac, scatter, full = bufs["conv"], bufs["fac"], 0, 0
                cl = ws["cluster"]
                _lib.check(lib.igmc_pair_grad(C.byref(m._cmodel), m.flat_params.data_ptr(), B, _lib.ctas_per_graph(cl),
                                              ws["gpart"].data_ptr(), int(_lib.is_rs(cl)), ws["dhid"].data_ptr(),
                                              ws["feat"].data_ptr(), ws["hid"].data_ptr(), dpred.data_ptr(), tag,
                                              scatter, grad.data_ptr(), full, _lib.ptr(fac), st), "igmc_pair_grad")
            if phase != "train":
                continue
            eta = run["lrs"][j]
            if run["T"]:
                _lib.check(lib.igmc_influence_accum(C.byref(m._cmodel), B, run["T"], bufs["conv"].data_ptr(),
                                                    bufs["fac"].data_ptr(), run["tconv"][j].data_ptr(),
                                                    run["tfac"][j].data_ptr(), eta, int(j == 0),
                                                    bufs["ws"].data_ptr(), bufs["ws"].numel(), bufs["S"].data_ptr(),
                                                    st), "igmc_influence_accum")
            if run["self_out"] is not None:
                _lib.check(lib.igmc_self_influence(C.byref(m._cmodel), B, bufs["conv"].data_ptr(),
                                                   bufs["fac"].data_ptr(), tag, eta, run["self_out"].data_ptr(), st),
                           "igmc_self_influence")
        if phase == "train" and run["T"]:
            _lib.check(lib.igmc_influence_topk(bufs["S"].data_ptr(), B, run["T"], tag, run["k"],
                                               run["pro_v"].data_ptr(), run["pro_i"].data_ptr(),
                                               run["con_v"].data_ptr(), run["con_i"].data_ptr(), st),
                       "igmc_influence_topk")

    def _start_explicit(self, kind, users, items, **extra):
        """plan a run over the explicit pairs (users[i], items[i]), host arrays ``_host_pairs`` checked.  Returns their
        number."""
        P, dev = len(users), self.dev
        run = dict(kind=kind, P=P, version=self.graph.version, scores=torch.empty(P, dtype=torch.float32, device=dev),
                   **extra)
        self.run = run
        if kind in _EXPLAIN_RESULTS:
            # the positions per pair: its ratings, or its non-target nodes on a node run
            run["num_edges"] = torch.zeros(P, dtype=torch.int32, device=dev)
            run["offsets"] = torch.zeros(P + 1, dtype=torch.int64, device=dev)
            for s in self.slots:
                if kind in ("explain", "explain_nodes") and "j" not in s:
                    s["j"] = torch.zeros(self.B, dtype=torch.int32, device=dev)
        if P == 0:
            return 0
        self._explicit_pairs(run, users, items)
        self._prime()
        return P

    def _explicit_pairs(self, run, users, items):
        """run["pu"], run["pv"] and run["Cd"]: the explicit pairs (users[i], items[i]) on the device"""
        run["pu"] = torch.from_numpy(users.astype(np.int32)).to(self.dev)
        run["pv"] = torch.from_numpy(items.astype(np.int32)).to(self.dev)
        Cd = run["Cd"] = _lib.Candidates()
        Cd.pair_u, Cd.pair_v, Cd.num_pairs = run["pu"].data_ptr(), run["pv"].data_ptr(), len(users)

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
        sessions = run.get("sessions")
        # session rows served: the trial rows of a counterfactual run (never longer than the graph's rows) or of a
        # question-impact run (a session row and the question), else a session run's
        row_deg = run["row_deg"] if "row_deg" in run else sessions.max_row_deg if sessions is not None else 0
        self.extractor.serve_sessions(row_deg)
        per = run.get("G", self.B)      # pairs per batch: G on a run over draws, G units on a question-impact run
        run["steps"] = ((run["P"] if total is None else total) + per - 1) // per
        if run.get("S"):
            self._draw_masks()
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
        sessions = run.get("sessions")
        if run["kind"] == "counterfactual":
            # the trials' pairs, and per slot its trial row as session g, extracted in session mode
            t = sessions = s["trial"]
            _lib.check(self.lib.igmc_counterfactual_pairs(C.byref(self.graph._c), C.byref(run["Qd"]),
                                                          run["offsets"].data_ptr(), run["step"], self.cursor.data_ptr(),
                                                          self.B, s["u"].data_ptr(), s["v"].data_ptr(),
                                                          s["pid"].data_ptr(), s["tag"].data_ptr(), t.users.data_ptr(),
                                                          t.row_ptr.data_ptr(), t.col_idx.data_ptr(),
                                                          t.rating.data_ptr(), t.cap, s["sess"].data_ptr(), err,
                                                          _stream_ptr()), "igmc_counterfactual_pairs")
        elif occlude:
            _lib.check(self.lib.igmc_occlusion_pairs(C.byref(self.graph._c), run["pu"].data_ptr(),
                                                     run["pv"].data_ptr(), run["offsets"].data_ptr(), run["P"],
                                                     self.cursor.data_ptr(), self.B, s["u"].data_ptr(),
                                                     s["v"].data_ptr(), s["pid"].data_ptr(), s["tag"].data_ptr(),
                                                     s["j"].data_ptr(), err, _stream_ptr()), "igmc_occlusion_pairs")
        elif run.get("A"):
            # G units (session, question), then A x W positions each and per answer its trial row as session
            # g * A + a, extracted in session mode
            _lib.check(self.lib.igmc_candidate_pairs(C.byref(self._csr(run)), C.byref(run["Cd"]),
                                                     self.cursor.data_ptr(), run["G"], s["gu"].data_ptr(),
                                                     s["gv"].data_ptr(), s["gpid"].data_ptr(), s["gtag"].data_ptr(),
                                                     err, _stream_ptr()), "igmc_candidate_pairs")
            t = s["trial"]
            _lib.check(self.lib.igmc_elicit_pairs(C.byref(sessions._c), self.graph.num_items, run["A"],
                                                  run["targets"].data_ptr(), run["W"], run["per_session"],
                                                  s["gu"].data_ptr(), s["gv"].data_ptr(), s["gtag"].data_ptr(), self.B,
                                                  s["u"].data_ptr(), s["v"].data_ptr(), s["pid"].data_ptr(),
                                                  s["tag"].data_ptr(), t.users.data_ptr(), t.row_ptr.data_ptr(),
                                                  t.col_idx.data_ptr(), t.rating.data_ptr(), t.cap,
                                                  s["sess"].data_ptr(), err, _stream_ptr()), "igmc_elicit_pairs")
            sessions = t
        elif run.get("S"):
            # G pairs, then S consecutive draws of each over the B positions
            _lib.check(self.lib.igmc_candidate_pairs(C.byref(self._csr(run)), C.byref(run["Cd"]),
                                                     self.cursor.data_ptr(), run["G"], s["gu"].data_ptr(),
                                                     s["gv"].data_ptr(), s["gpid"].data_ptr(), s["gtag"].data_ptr(),
                                                     err, _stream_ptr()), "igmc_candidate_pairs")
            _lib.check(self.lib.igmc_draws_expand(run["S"], self.B, s["gu"].data_ptr(), s["gv"].data_ptr(),
                                                  s["gpid"].data_ptr(), s["gtag"].data_ptr(), s["u"].data_ptr(),
                                                  s["v"].data_ptr(), s["pid"].data_ptr(), s["tag"].data_ptr(),
                                                  s["draw"].data_ptr(), _stream_ptr()), "igmc_draws_expand")
        else:
            _lib.check(self.lib.igmc_candidate_pairs(C.byref(self._csr(run)), C.byref(run["Cd"]),
                                                     self.cursor.data_ptr(), self.B, s["u"].data_ptr(),
                                                     s["v"].data_ptr(), s["pid"].data_ptr(), s["tag"].data_ptr(), err,
                                                     _stream_ptr()), "igmc_candidate_pairs")
        if run.get("by_item"):
            # pairs over the transposed view are (item, user): back to (user, item) and the pair's own pair id
            _lib.check(self.lib.igmc_item_query_pairs(self.graph.num_items, self.B, s["u"].data_ptr(),
                                                      s["v"].data_ptr(), s["pid"].data_ptr(), err, _stream_ptr()),
                       "igmc_item_query_pairs")
        if run.get("sessions") is not None and not run.get("A"):
            # links_u holds the session: to the session's user id, its pair id and the per-pair session index
            _lib.check(self.lib.igmc_session_pairs(C.byref(sessions._c), self.graph.num_items, self.B,
                                                   s["u"].data_ptr(), s["v"].data_ptr(), s["pid"].data_ptr(),
                                                   s["sess"].data_ptr(), err, _stream_ptr()), "igmc_session_pairs")
        b = self.batches[slot] = self.extractor.extract(pairs=(s["u"], s["v"], None), pair_ids=s["pid"], reuse=True,
                                                        slot=slot, sessions=sessions,
                                                        sess=None if sessions is None else s["sess"])
        nodes = run["kind"] in _NODE_KINDS
        if occlude:
            mask = "igmc_node_occlusion_mask" if nodes else "igmc_occlusion_mask"
            _lib.check(getattr(self.lib, mask)(C.byref(b._lazy["_c"]), self.B, s["tag"].data_ptr(), s["j"].data_ptr(),
                                               s["keep"].data_ptr(), run["user"].data_ptr(), run["item"].data_ptr(),
                                               run["rating"].data_ptr(), err, _stream_ptr()), mask)
        elif run.get("S"):
            # the masks are keyed by the final (user, item) pair id: after the mapping kernels above
            _lib.check(self.lib.igmc_draws_mask(C.byref(b._lazy["_c"]), self.B, s["pid"].data_ptr(),
                                                s["tag"].data_ptr(), s["draw"].data_ptr(), float(self.model.adj_dropout),
                                                run["draw_seed"], s["keep"].data_ptr(), s["hkeep"].data_ptr(),
                                                _stream_ptr()), "igmc_draws_mask")
        elif run.get("phase") == "base":
            count, ptr = ("igmc_explain_node_count", "node_ptr") if nodes else ("igmc_explain_count", "edge_ptr")
            _lib.check(getattr(self.lib, count)(b._priv[ptr].data_ptr(), s["tag"].data_ptr(), self.B,
                                                run["num_edges"].data_ptr(), _stream_ptr()), count)

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
        if run.get("phase") in ("pgrad", "test", "train"):
            return self._pair_grad_step(slot)
        occlude = run.get("phase") == "occlude"
        training, drop = (True, s["drop"]) if occlude or run.get("S") else (False, self.drop)
        preds = None
        for j in range(self.K):
            with self._params(j):
                pred, _ = m._launch_forward(b, training, drop)
            if self.K == 1:
                preds = pred
            else:
                self.preds[j].copy_(pred)
                preds = self.preds
        if run.get("S"):
            return self._draw_stats(preds, s)
        if run.get("A"):
            return self._elicit_stats(preds, s)
        if run["kind"] == "recommend":
            ranked = s["u"] if run.get("by_item") else s["v"]      # the candidates: users on an item-side run
            _lib.check(self.lib.igmc_topk_merge(preds.data_ptr(), self.K, self.B, s["tag"].data_ptr(),
                                                ranked.data_ptr(), run["k"], run["top_s"].data_ptr(),
                                                run["top_i"].data_ptr(), _stream_ptr()), "igmc_topk_merge")
        else:
            out = run["occ"] if occlude else run["scores"]
            _lib.check(self.lib.igmc_score_scatter(preds.data_ptr(), self.K, self.B, s["tag"].data_ptr(),
                                                   out.data_ptr(), _stream_ptr()), "igmc_score_scatter")

    def _draw_stats(self, preds, s):
        """a batch of draws: per pair its statistics scattered to the run's outputs, or (ranking) its key
        mean + beta * std merged into the running top-k lists over the batch's G pairs"""
        run, st = self.run, _stream_ptr()
        rank = run["kind"] == "recommend"
        outs = (None, None, None, run["keys"]) if rank else (run["value"], run["mean"], run["std"], None)
        _lib.check(self.lib.igmc_draws_stats(preds.data_ptr(), self.K, self.B, run["S"], s["tag"].data_ptr(),
                                             run["beta"], *(_lib.ptr(t) for t in outs), st), "igmc_draws_stats")
        if rank:
            # the candidates before the mapping kernels: items, or users on an item-side run
            _lib.check(self.lib.igmc_topk_merge(run["keys"].data_ptr(), 1, run["G"], s["gtag"].data_ptr(),
                                                s["gv"].data_ptr(), run["k"], run["top_s"].data_ptr(),
                                                run["top_i"].data_ptr(), st), "igmc_topk_merge")

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
            scatter = "igmc_node_grad_scatter" if run["kind"] in _NODE_KINDS else "igmc_edge_grad_scatter"
            _lib.check(getattr(self.lib, scatter)(C.byref(b._lazy["_c"]), self.B, s["tag"].data_ptr(),
                                                  gw["edge_grad"].data_ptr(), run["offsets"].data_ptr(), j, self.K,
                                                  run["occ"].data_ptr(), run["user"].data_ptr(), run["item"].data_ptr(),
                                                  run["rating"].data_ptr(), self.extractor.err.data_ptr(), st), scatter)

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
        if run["kind"] == "counterfactual":
            return self._select_trials()
        if run.get("phase") == "test":
            return self._start_train_pass()
        if run.get("phase") != "base":
            return False
        return self._start_occlusion() if run["kind"] in ("explain", "explain_nodes") else self._start_gradient()

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
        if run["kind"] in _EXPLAIN_RESULTS:
            return self._order(run)
        if run["kind"] == "pair_gradients":
            return run["out"]
        if run["kind"] == "influence":
            return Influence(run["pro_i"], run["pro_v"], run["con_i"], run["con_v"])
        if run["kind"] == "self_influence":
            return run["self_out"]
        if run["kind"] == "draws":
            return Draws(run["value"], run["mean"], run["std"])
        if run["kind"] == "counterfactual":
            return run["out"]
        if run["kind"] == "question_impact":
            return QuestionImpact(run["impact"], run["answer_mean"])
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
        occlusion = run["kind"] in ("explain", "explain_nodes")
        _lib.check(self.lib.igmc_occlusion_order(run["scores"].data_ptr() if occlusion else None,
                                                 run["occ"].data_ptr(), run["offsets"].data_ptr(), P, T,
                                                 run["user"].data_ptr(), run["item"].data_ptr(),
                                                 run["rating"].data_ptr(), m or 0, ws.data_ptr(), ws.numel(),
                                                 out["user"].data_ptr(), out["item"].data_ptr(),
                                                 out["rating"].data_ptr(), out["delta"].data_ptr(), _stream_ptr()),
                   "igmc_occlusion_order")
        if m and run["kind"] in _NODE_KINDS:
            out["rating"].masked_fill_(out["user"] < 0, 0)      # a padded node has no ratings
        return _EXPLAIN_RESULTS[run["kind"]](run["scores"], run["num_edges"], run["offsets"], out["user"],
                                             out["item"], out["rating"], out["delta"])

    def recommend(self, users, k, items=None, exclude_rated=True, retrieve=None, draws=None, beta=0.0, draw_seed=0):
        self.start_recommend(users, k, items, exclude_rated, retrieve, draws, beta, draw_seed)
        return self.finish()

    def recommend_users(self, items, k, users=None, exclude_rated=True, retrieve=None, draws=None, beta=0.0,
                        draw_seed=0):
        self.start_recommend_users(items, k, users, exclude_rated, retrieve, draws, beta, draw_seed)
        return self.finish()

    def predict_pairs(self, users, items):
        self.start_pairs(users, items)
        return self.finish()

    def predict_draws(self, users, items, draws, draw_seed=0):
        self.start_draws(users, items, draws, draw_seed)
        return self.finish()

    def predict_sessions(self, sessions, session, items):
        self.start_session_pairs(sessions, session, items)
        return self.finish()

    def recommend_sessions(self, sessions, k, items=None, exclude_rated=True, retrieve=None, draws=None, beta=0.0,
                           draw_seed=0):
        self.start_session_recommend(sessions, k, items, exclude_rated, retrieve, draws, beta, draw_seed)
        return self.finish()

    def explain_pairs(self, users, items, m=None):
        self.start_explain(users, items, m)
        return self.finish()

    def attribute_pairs(self, users, items, m=None):
        self.start_attribute(users, items, m)
        return self.finish()

    def explain_nodes(self, users, items, m=None):
        self.start_explain_nodes(users, items, m)
        return self.finish()

    def counterfactual(self, users, items, rivals, max_removals=10):
        self.start_counterfactual(users, items, rivals, max_removals)
        return self.finish()

    def elicit(self, sessions, n, targets, questions=None):
        self.start_elicit(sessions, n, targets, questions)
        return self.finish()

    def question_impact(self, sessions, session, questions, targets):
        self.start_question_impact(sessions, session, questions, targets)
        return self.finish()

    def attribute_nodes(self, users, items, m=None):
        self.start_attribute_nodes(users, items, m)
        return self.finish()

    def pair_gradients(self, users, items, y=None):
        self.start_pair_gradients(users, items, y)
        return self.finish()

    def influence(self, train, test, k, lrs=None):
        self.start_influence(train, test, k, lrs)
        return self.finish()

    def self_influence(self, train, lrs=None):
        self.start_self_influence(train, lrs)
        return self.finish()

    def close(self):
        torch.cuda.synchronize()
        self.graphs = {}


# ---- public API -----------------------------------------------------------------------------------------------------
def _on_engine(model, graph, call, h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed):
    """``call(engine)`` on an InferenceEngine of ``model`` and ``graph`` built with the public functions' keywords,
    closed afterwards"""
    eng = InferenceEngine(model, graph, h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)
    try:
        return call(eng)
    finally:
        eng.close()


def _no_pairs_explained(cls, m, dev):
    """the Explanation or Attribution (``cls``) of no pairs: [0] / [1] offsets / [0] or [0, m] per-rating tensors"""
    shape = (0, m) if m else (0,)
    i32 = dict(dtype=torch.int32, device=dev)
    return cls(torch.zeros(0, dtype=torch.float32, device=dev), torch.zeros(0, **i32),
               torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(shape, **i32), torch.zeros(shape, **i32),
               torch.zeros(shape, **i32), torch.zeros(shape, dtype=torch.float32, device=dev))


def predict_pairs(model, graph, users, items, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None, batch_size=256,
                  checkpoints=None, sample_seed=0):
    """eval-mode scores [P] (fp32, on the model's device) of the pairs (users[i], items[i]); a pair rated in ``graph``
    is scored on its subgraph without the target edge, as in training.  ``checkpoints``: average of the checkpoints'
    scores (fp32 sum in checkpoint order / K)."""
    users, items, _ = _host_pairs(graph.shape, users, items)
    if len(users) == 0:
        return torch.zeros(0, dtype=torch.float32, device=model.flat_params.device)
    return _on_engine(model, graph, lambda eng: eng.predict_pairs(users, items),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def predict_draws(model, graph, users, items, draws, *, draw_seed=0, h=1, sample_ratio=1.0, max_nodes_per_hop=None,
                  batch_size=256, checkpoints=None, sample_seed=0):
    """``draws`` Monte-Carlo-dropout draws of the score of each pair (users[i], items[i]) and their statistics: a
    ``Draws`` of value [P, S], mean [P] and std [P] fp32 on the model's device.  Draw s of a pair is the training-mode
    forward of the subgraph ``predict_pairs`` scores, with each directed edge kept with probability 1 - adj_dropout
    and each of the 128 hidden units before lin2 kept with probability 0.5 (and scaled by 2), IGMC and DGCNN_RS alike:
    the dropout the model was trained with.  The masks are counter hashes of (draw_seed, u * num_items + v, s, the
    edge's offset in its subgraph or the unit's index), so a draw depends on the parameters, the graph, the pair, s and
    draw_seed only: not on the batch size, the batch position or the other pairs of the run.  ``checkpoints``: a draw
    is the fp32 checkpoint mean under the same masks.  mean and std (unbiased, 0 for S = 1) are taken in fp64 in draw
    order and rounded once; a NaN draw makes both NaN.  1 <= draws <= min(batch_size, IGMC_DRAWS_MAX = 256)."""
    d = _draw_inputs(draws, 0.0, draw_seed, batch_size)
    users, items, _ = _host_pairs(graph.shape, users, items)
    if len(users) == 0:
        dev = model.flat_params.device
        return Draws(*(torch.zeros(shape, dtype=torch.float32, device=dev) for shape in ((0, d["S"]), (0,), (0,))))
    return _on_engine(model, graph, lambda eng: eng.predict_draws(users, items, d["S"], d["draw_seed"]),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


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
    m = _check_top(m)
    users, items, _ = _host_pairs(graph.shape, users, items)
    if len(users) == 0:
        return _no_pairs_explained(Explanation, m, model.flat_params.device)
    return _on_engine(model, graph, lambda eng: eng.explain_pairs(users, items, m),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


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
    m = _check_top(m)
    users, items, _ = _host_pairs(graph.shape, users, items)
    if len(users) == 0:
        return _no_pairs_explained(Attribution, m, model.flat_params.device)
    return _on_engine(model, graph, lambda eng: eng.attribute_pairs(users, items, m),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def explain_nodes(model, graph, users, items, m=None, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None, batch_size=256,
                  checkpoints=None, sample_seed=0):
    """why each pair (users[i], items[i]) got its score, one node at a time: for every node of the pair's enclosing
    subgraph other than its two targets (the users and items with node_label >= 2, in the subgraph's node order),
    delta = the score of that subgraph with every rating of the node removed (both directed edges; same nodes, labels
    and sampling) - the pair's score.  For IGMC an isolated node sends no message, so this is the node removed;
    DGCNN_RS still sorts it into its SortPooling.  Returns a ``NodeExplanation`` of device tensors: score [P] (bit for
    bit ``predict_pairs``), num_nodes [P], offsets [P+1] and per node node (global user or item id) / label
    (node_label) / ratings (its ratings in the subgraph) / delta, ordered within a pair by |delta| descending, NaN
    after every number, ties by position; flat with pair p at [offsets[p], offsets[p+1]) when ``m`` is None, else the
    first ``m`` per pair [P, m], padded with node / label -1 and ratings / delta 0.  A pair whose subgraph holds only
    its targets (a cold-start pair) has no entries.  ``checkpoints``: every score is the fp32 checkpoint mean."""
    m = _check_top(m)
    users, items, _ = _host_pairs(graph.shape, users, items)
    if len(users) == 0:
        return _no_pairs_explained(NodeExplanation, m, model.flat_params.device)
    return _on_engine(model, graph, lambda eng: eng.explain_nodes(users, items, m),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def attribute_nodes(model, graph, users, items, m=None, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None,
                    batch_size=256, checkpoints=None, sample_seed=0):
    """why each pair (users[i], items[i]) got its score, one node at a time and to first order: every non-target node
    n of the pair's enclosing subgraph gets a gate g_n that multiplies the weight m_e (``attribute_pairs``) of each of
    its ratings; grad = d score / d g_n at g = 1 = the sum of ``attribute_pairs``' grad over n's ratings, summed in n's
    in-list order (its ratings sorted by (label, neighbour)).  -grad estimates ``explain_nodes``' delta.  Returns a
    ``NodeAttribution`` in ``NodeExplanation``'s layout and order with grad in place of delta.  The gradient pass runs
    the L2 kernel plan whatever plan the model uses.  ``checkpoints``: score and grad are fp32 checkpoint means."""
    m = _check_top(m)
    users, items, _ = _host_pairs(graph.shape, users, items)
    if len(users) == 0:
        return _no_pairs_explained(NodeAttribution, m, model.flat_params.device)
    return _on_engine(model, graph, lambda eng: eng.attribute_nodes(users, items, m),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def counterfactual(model, graph, users, items, rivals, max_removals=10, *, h=1, sample_ratio=1.0,
                   max_nodes_per_hop=None, batch_size=256, checkpoints=None, sample_seed=0):
    """which of user u's own ratings, removed together, put item X behind the rival item Y: per query (users[q],
    items[q], rivals[q]) a greedy search over u's ratings with every candidate scored exactly.  s_R(u, v) is the eval
    score of (u, v) on the graph with u's ratings of the items in R deleted (``predict_sessions`` on a session of u
    that deletes R: same pair id, sample_seed and checkpoint mean); "X ahead of Y" is ``recommend``'s order (score
    descending, item ascending, NaN last).  From R = {}: if X is not ahead of Y the answer has size 0.  Otherwise each
    step scores the trial R + {i} for every item i of u's row not in R and adds the first by (trials that put X
    behind Y first, then the margin s(u,X) - s(u,Y) (fp32) ascending with NaN after every number, then item
    ascending).  The search stops when X is behind Y (found), when |R| = ``max_removals`` or when u's row has no item
    left (not found; the path taken is still reported).  u's ratings of X and Y are candidates like any other; a pair's
    own rating is never in its own subgraph, as in ``predict_pairs``.  Returns a ``Counterfactual`` of device
    tensors: found [Q] bool, size [Q] int32, items / ratings [Q, max_removals] int32 (the removed items in greedy order
    and their labels, -1 past size), score / rival_score [Q, max_removals + 1] fp32 (s(u, X) / s(u, Y) before any
    removal and after each, NaN past size).  The results do not depend on batch_size, graph replay or the other
    queries.  A step costs 2 (deg(u) - |R|) forwards per query; 1 <= max_removals <= IGMC_COUNTERFACTUAL_MAX = 256.
    The graph is not changed."""
    users, items, rivals, M = _counterfactual_inputs(graph.shape, users, items, rivals, max_removals)
    if len(users) == 0:
        return _no_counterfactual(0, M, model.flat_params.device)
    return _on_engine(model, graph, lambda eng: eng.counterfactual(users, items, rivals, M),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def pair_gradients(model, graph, users, items, y=None, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None,
                   batch_size=256, checkpoints=None, sample_seed=0):
    """per-example gradients [K, P, param_count] fp32 on the model's device, in the ``flat_params`` layout (conv
    parameters, then lin1 and lin2), one row per pair and checkpoint (K = 1 without ``checkpoints``).  With ``y``: the
    gradient of l_i = (f_i - y_i)^2, the squared error of ONE pair - the batch mean and the ARR regulariser are not
    per-example terms and are left out; the backward's seed is 2 (f_i - y_i) * multiply_by.  Without ``y``: the gradient
    of the score f_i (seed multiply_by).  Pair i's subgraph is the one ``predict_pairs`` scores (its own rating removed,
    sampled by its pair id); the forward is the eval forward, run as a training-mode launch with both dropout rates 0,
    on the model's own kernel plan.  Needs 4 * param_count bytes per pair and checkpoint (197 KB at R = 5): meant for
    thousands of pairs; ``influence`` / ``self_influence`` never materialise them.  IGMC only (DGCNN_RS:
    NotImplementedError)."""
    _check_per_pair_model(model)
    users, items, y = _host_pairs(graph.shape, users, items, y)
    if len(users) == 0:
        K = len(checkpoints) if checkpoints else 1
        return torch.zeros(K, 0, model._cmodel.param_count, dtype=torch.float32, device=model.flat_params.device)
    return _on_engine(model, graph, lambda eng: eng.pair_gradients(users, items, y),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def influence(model, graph, train, test, k, *, checkpoints=None, lrs=None, h=1, sample_ratio=1.0,
              max_nodes_per_hop=None, batch_size=256, sample_seed=0):
    """TracIn-CP influence of every training pair on every test pair:
        influence(i, t) = sum over checkpoints k of lrs[k] * < grad l_i(theta_k), grad q_t(theta_k) >
    with l_i = (f_i - y_i)^2 of one training pair (``pair_gradients``' definition: no batch mean, no ARR term) and q_t =
    l_t for a labelled test pair, f_t (the score) otherwise.  ``train`` = (users, items, y) with y the value the model
    was trained against; ``test`` = (users, items) or (users, items, y), at most INFLUENCE_T_MAX = 1024 pairs
    (NotImplementedError above: split the test set).  ``lrs``: eta_k per checkpoint, default 1.  Sign: with test labels
    a positive value marks a proponent - a gradient step on i lowers t's loss; without, a step theta <- theta - eta
    grad l_i changes f_t by -eta * influence to first order.  Returns an ``Influence`` of [T, k] device tensors: the k
    largest values (pro_*) and the k smallest (con_*) per test pair, index = position in ``train``; ties by index, NaN
    after every number, empty slots -1 / -inf (pro) and -1 / +inf (con).  Conv block by a split-K FFMA GEMM, readout
    block from its rank-1 factors; bit-identical across runs, batch sizes and graph replay.  IGMC only."""
    _check_per_pair_model(model)
    k, tr, te, lrs = _influence_inputs(graph.shape, train, test, k, batch_size, lrs,
                                       len(checkpoints) if checkpoints else 1)
    if len(te[0]) == 0:
        dev = model.flat_params.device
        return Influence(*(torch.zeros(0, k, dtype=t, device=dev) for t in (torch.int64, torch.float32) * 2))
    return _on_engine(model, graph, lambda eng: eng.influence(tr, te, k, lrs),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def self_influence(model, graph, train, *, checkpoints=None, lrs=None, h=1, sample_ratio=1.0, max_nodes_per_hop=None,
                   batch_size=256, sample_seed=0):
    """self_influence(i) = sum over checkpoints k of lrs[k] * ||grad l_i(theta_k)||^2 for every training pair of
    ``train`` = (users, items, y), [N] fp32 on the model's device (``influence``'s definitions).  The usual detector
    of mislabelled training examples: large values first.  IGMC only."""
    _check_per_pair_model(model)
    tr = _host_pairs(graph.shape, *_split_pairs(train, "train", True), name="train")
    lrs = _check_lrs(lrs, len(checkpoints) if checkpoints else 1)
    if len(tr[0]) == 0:
        return torch.zeros(0, dtype=torch.float32, device=model.flat_params.device)
    return _on_engine(model, graph, lambda eng: eng.self_influence(tr, lrs),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def recommend(model, graph, users, k, *, items=None, exclude_rated=True, retrieve=None, draws=None, beta=0.0,
              draw_seed=0, h=1, sample_ratio=1.0, max_nodes_per_hop=None, batch_size=256, checkpoints=None,
              sample_seed=0):
    """for every query user the ``k`` best candidate items: (top_items [U, k] int64, top_scores [U, k] fp32), on the
    model's device.  Candidates: ``items`` (sorted, deduplicated), a 2-D ``items`` [U, width] of per-user lists (-1 =
    empty slot; each row sorted and deduplicated), the user's ``retrieve`` items with the most bridges
    (``corated_items``), or every item; minus the user's rated items when ``exclude_rated``.  Order: score
    descending, then item ascending; a NaN score ranks last; a user with fewer than ``k`` candidates gets item -1 /
    score -inf in the empty slots.  A pair's score does not depend on the candidates it was ranked among.
    ``draws=S``: every candidate is ranked by its key mean + beta * std over S draws (``predict_draws``, seeded by
    ``draw_seed``), and the returned scores are those keys: S = 1 is Thompson sampling (std = 0), beta > 0 UCB and
    beta < 0 a risk-averse ranking.  ``draws=None`` ranks by the eval score."""
    d = _draw_inputs(draws, beta, draw_seed, batch_size)
    users = _host_ids(users, "users", graph.shape[0])
    k = _ranking_inputs(k, batch_size, items, retrieve, len(users), graph.shape[1])[0]
    if len(users) == 0:
        dev = model.flat_params.device
        return (torch.zeros(0, k, dtype=torch.int64, device=dev), torch.zeros(0, k, dtype=torch.float32, device=dev))
    return _on_engine(model, graph, lambda eng: eng.recommend(users, k, items, exclude_rated, retrieve, draws, beta,
                                                              draw_seed),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


class RecommendationCache(object):
    """``recommend``'s lists for a fixed set of users, kept exact as ratings arrive (h = 1; DESIGN.md §19).

        cache = RecommendationCache(model, graph, users, k=10, depth=50)
        cache.update(u, v, values)             # graph.update, then only the pairs the edits can reach are rescored
        top_items, top_scores = cache.lists()  # == recommend(model, graph, users, 10, ...) on the updated graph

    An edit (a, b) changes the enclosing subgraph of (u, v) only when u = a, v = b, or u rated b and a rated v: every
    other cached score stays what ``recommend`` computes, bit for bit.  Each slot keeps its ``depth`` best entries as an
    exact prefix; a repair drops the rescored items from it, merges their new scores and keeps the entries that still
    rank before every unlisted item.  A slot left with fewer than k exact entries is re-ranked in full.  Keywords as
    ``recommend``'s (one shared ``items`` list or none); ``depth`` (k..IGMC_TOPK_MAX, default k): kept entries per
    slot, a deeper list outlives more invalidations.

    Host synchronisations of an ``update`` that needs no full rebuild or fallback: the parameter check, graph.update's,
    the rescore total and the fallback count, four in all (three without rescored pairs; with ``checkpoints`` the
    parameter check compares the files' stamps on the host).  Every list is rebuilt in full - ``update`` returns
    full=True - when the item count grows (every pair id changes), the model's parameters or the checkpoint files
    changed since the last build, the extractor's node capacity n_cap changes (it sets the kernel plan, and scores are
    bit-identical on one batch shape), or the rescore plan reaches the pairs of a full run."""

    def __init__(self, model, graph, users, k, *, depth=None, items=None, exclude_rated=True, h=1, sample_ratio=1.0,
                 max_nodes_per_hop=None, batch_size=256, checkpoints=None, sample_seed=0, use_graph=True,
                 retrieve=None, draws=None):
        if draws is not None:
            raise NotImplementedError("a cache keeps lists ranked by the eval score: a ranking by draws= is drawn anew "
                                      "for every pair")
        if int(h) != 1:
            raise NotImplementedError("a cache repairs lists with h = 1 only: at h >= 2 an update reaches further by "
                                      "a hop per hop")
        users = _host_ids(users, "users", graph.shape[0])
        k, m, cand, rows = _ranking_inputs(k, batch_size, items, retrieve, len(users), graph.shape[1])
        if m is not None or rows is not None:
            raise NotImplementedError("a cache takes one shared items list or none: per-user rows and retrieve= "
                                      "candidates change with the graph")
        depth = k if depth is None else _check_count(depth, "depth", _lib.TOPK_MAX)
        if depth < k:
            raise ValueError("depth must be at least k (%d), not %d" % (k, depth))
        _check_merge_fits(depth, batch_size)
        self.k, self.depth, self.exclude_rated = k, depth, bool(exclude_rated)
        self._users, self._cand, self._checkpoints = users, cand, list(checkpoints or [])
        self._args = [model, graph, h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed,
                      use_graph]
        self.eng = InferenceEngine(*self._args)
        self.graph = self._args[1] = self.eng.graph
        U, dev = len(users), self.eng.dev
        i32, i64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.int64, device=dev)
        self._slots = torch.from_numpy(users.astype(np.int32)).to(dev)
        self._cand_dev = None if cand is None else torch.from_numpy(cand.astype(np.int32)).to(dev)
        self._user_off, self._totals = torch.zeros(U + 1, **i64), torch.zeros(2, **i64)
        self._full = torch.zeros(max(U, 1), dtype=torch.uint8, device=dev)
        self._thr_s = torch.zeros(max(U, 1), dtype=torch.float32, device=dev)
        self._thr_i, self._redo, self._redo_count = torch.zeros(max(U, 1), **i64), torch.zeros(max(U, 1), **i32), \
            torch.zeros(1, **i32)
        self._resc, self._ws = torch.zeros(1, **i32), torch.zeros(1, dtype=torch.uint8, device=dev)
        self.refresh()

    def _stamp(self):
        return [(os.stat(p).st_mtime_ns, os.stat(p).st_size) for p in self._checkpoints]

    def _stale_params(self):
        """the scored parameters changed since the last build: the checkpoint files' stamps (host), or the model's
        flat_params against the device copy taken then (one host sync)"""
        if self._checkpoints:
            return self._stamp() != self._built_from
        return not torch.equal(self.eng.model.flat_params, self._built_from)

    def _check_version(self):
        if self.graph.version != self._version:
            raise RuntimeError("the rating graph was updated outside this cache (graph.update): its lists belong to "
                               "the old graph; call refresh()")

    def refresh(self):
        """rebuild every list with a full ranking run (also after an update made outside the cache).  Returns the
        number of pairs scored."""
        if self._checkpoints and self._stamp() != getattr(self, "_built_from", None):
            self.eng.close()
            self.eng = InferenceEngine(*self._args)     # reads the checkpoint files again
        eng, g = self.eng, self.graph
        self._built_from = self._stamp() if self._checkpoints else eng.model.flat_params.detach().clone()
        P = eng.start_recommend(self._users, self.depth, self._cand, self.exclude_rated)
        self._top_i, self._top_s = eng.finish()
        self._complete = ((self._top_i >= 0).sum(1) < self.depth).to(torch.uint8)
        eng.extractor._sync_graph()
        self._version, self._num_items, self._cap = g.version, g.num_items, eng.extractor.cap
        need = len(self._users) * (g.num_items if self._cand is None else len(self._cand))
        if self._resc.numel() < need:
            self._resc = torch.empty(need, dtype=torch.int32, device=eng.dev)
        return P

    def lists(self):
        """(top_items [U, k] int64, top_scores [U, k] fp32) on the device: ``recommend``'s layout and order"""
        self._check_version()
        return self._top_i[:, :self.k].clone(), self._top_s[:, :self.k].clone()

    def update(self, users, items, values, shape=None):
        """``graph.update(users, items, values, shape)``, then the lists repaired.  Returns graph.update's counts and
        rescored_pairs (pairs scored: the rescore plan's, or a full run's), rebuilt_users (slots re-ranked in full)
        and full (every list rebuilt)."""
        self._check_version()
        g, eng, U = self.graph, self.eng, len(self._users)
        stale = U > 0 and self._stale_params()
        u, v, x, D = _update_inputs(users, items, values, g.capacity.users, g.capacity.items)
        if any(torch.is_tensor(t) for t in (u, v, x)):
            u, v, x = (_on_device_i32(t, eng.dev) for t in (u, v, x))
        else:       # checked above: one pinned upload, no stream sync, and graph.update takes the edits as they are
            up = torch.from_numpy(np.stack([u, v, x]).astype(np.int32)).pin_memory().to(eng.dev, non_blocking=True)
            u, v, x = up[0], up[1], up[2]
        out = dict(g.update(u, v, x, shape), rescored_pairs=0, rebuilt_users=0, full=False)
        if U == 0 or (g.version == self._version and not stale):
            self._version = g.version
            return out
        eng.extractor._sync_graph()
        if stale or g.num_items != self._num_items or eng.extractor.cap != self._cap:
            return dict(out, rescored_pairs=self.refresh(), full=True)
        nbytes, chunk = C.c_int64(0), C.c_int(0)
        lib, err = eng.lib, eng.extractor.err
        _lib.check(lib.igmc_rescore_plan_ws_bytes(U, g.num_items, 0, C.byref(nbytes), C.byref(chunk)),
                   "igmc_rescore_plan_ws_bytes")
        if self._ws.numel() < nbytes.value:
            self._ws = torch.empty(nbytes.value, dtype=torch.uint8, device=eng.dev)
        _lib.check(lib.igmc_rescore_plan(C.byref(g._c), self._slots.data_ptr(), U, u.data_ptr(), v.data_ptr(), D,
                                         _lib.ptr(self._cand_dev), 0 if self._cand is None else len(self._cand),
                                         int(self.exclude_rated), self._ws.data_ptr(), self._ws.numel(),
                                         self._user_off.data_ptr(), self._resc.data_ptr(), self._resc.numel(),
                                         self._full.data_ptr(), self._totals.data_ptr(), err.data_ptr(),
                                         _stream_ptr()), "igmc_rescore_plan")
        P, total, code = (int(x) for x in torch.cat([self._totals, err.long()]).cpu())   # the rescore total
        self._check_error(code)
        if P > 0 and P >= total:
            return dict(out, rescored_pairs=self.refresh(), full=True)
        self._version = g.version
        if P == 0:
            return out
        args = (U, self.depth)
        _lib.check(lib.igmc_cache_invalidate(*args, self._user_off.data_ptr(), self._resc.data_ptr(),
                                             self._full.data_ptr(), self._complete.data_ptr(), self._top_s.data_ptr(),
                                             self._top_i.data_ptr(), self._thr_s.data_ptr(), self._thr_i.data_ptr(),
                                             _stream_ptr()), "igmc_cache_invalidate")
        eng._start_rescore(self._slots, self._user_off, self._resc, P, self._top_s, self._top_i)
        while eng.step():
            pass
        eng.run = None
        _lib.check(lib.igmc_cache_settle(*args, self.k, self._thr_s.data_ptr(), self._thr_i.data_ptr(),
                                         self._top_s.data_ptr(), self._top_i.data_ptr(), self._complete.data_ptr(),
                                         self._redo.data_ptr(), self._redo_count.data_ptr(), _stream_ptr()),
                   "igmc_cache_settle")
        F, code = (int(x) for x in torch.cat([self._redo_count, err]).cpu())          # the fallback count
        self._check_error(code)
        if F:
            redo = self._redo[:F].long()
            ti, ts = eng.recommend(self._users[redo.cpu().numpy()], self.depth, self._cand, self.exclude_rated)
            self._top_i[redo], self._top_s[redo] = ti, ts
            self._complete[redo] = ((ti >= 0).sum(1) < self.depth).to(torch.uint8)
        return dict(out, rescored_pairs=P, rebuilt_users=F)

    def _check_error(self, code):
        if code:
            self.eng.extractor.err.zero_()
            self._version = None        # the lists are not known to be exact: refresh() rebuilds them
            _lib.check_kernel_error(code)

    def close(self):
        """wait for the device and release the engine and the lists"""
        self.eng.close()
        self._top_i = self._top_s = self._resc = self._ws = None


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
    m = _check_count(m, "m", g.num_items, ValueError)
    users = _host_ids(users, "users", g.num_users)
    err = torch.zeros(1, dtype=torch.int32, device=g.device)
    du = torch.from_numpy(users.astype(np.int32)).to(g.device)
    items, paths = _corated(_lib.load(), g.shape, "igmc_corated_items", (C.byref(g._c), du.data_ptr(), len(users)),
                            len(users), m, exclude_rated, err, {})
    _lib.check_kernel_error(int(err.item()))
    return items, paths


def recommend_users(model, graph, items, k, *, users=None, exclude_rated=True, retrieve=None, draws=None, beta=0.0,
                    draw_seed=0, h=1, sample_ratio=1.0, max_nodes_per_hop=None, batch_size=256, checkpoints=None,
                    sample_seed=0):
    """for every query item the ``k`` best candidate users - the audience of a new or promoted item: (top_users [I, k]
    int64, top_scores [I, k] fp32), on the model's device.  Candidates: ``users`` (sorted, deduplicated), a 2-D
    ``users`` [I, width] of per-item lists (-1 = empty slot), the item's ``retrieve`` users with the most bridges
    (``corated_users``), or every user; minus the item's raters when ``exclude_rated``.  Order: score descending, then
    user ascending; a NaN score ranks last; an item with fewer than ``k`` candidates gets user -1 / score -inf in the
    empty slots.  A pair's score is ``predict_pairs``' score of (u, v) bit for bit at the same batch size and kernel
    plan (pair id u * num_items + v): the lists filter those scores and compute nothing new.  An item added with
    ``graph.update`` and a few ratings is ranked against every user without retraining.  ``draws`` / ``beta`` /
    ``draw_seed``: ranked by mean + beta * std over draws, as in ``recommend``."""
    _draw_inputs(draws, beta, draw_seed, batch_size)
    items = _host_ids(items, "items", graph.shape[1])
    k = _ranking_inputs(k, batch_size, users, retrieve, len(items), graph.shape[0], "users")[0]
    if len(items) == 0:
        dev = model.flat_params.device
        return (torch.zeros(0, k, dtype=torch.int64, device=dev), torch.zeros(0, k, dtype=torch.float32, device=dev))
    return _on_engine(model, graph, lambda eng: eng.recommend_users(items, k, users, exclude_rated, retrieve, draws,
                                                                    beta, draw_seed),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def corated_users(graph, items, m, exclude_rated=True):
    """per query item the ``m`` users with the most bridges to it: (users [I, m], paths [I, m]) int32 on the graph's
    device.  The count for user u is exactly the count ``corated_items`` gives item v for u, C[u][v] = (B B^T B)[u][v]
    - deg(u) B[u][v] (B the 0/1 rating matrix): the 3-paths u - i - u' - v with u' != u.  Ordered by count descending,
    then user ascending; users without a bridge are never returned, the rest of a row is user -1 / paths 0;
    ``exclude_rated`` drops the item's raters.  Exact integer counts: runs are bit-identical.  ``graph``: a RatingGraph
    or a rating matrix (copied to the current CUDA device).  One host synchronisation (the error word)."""
    g = graph if isinstance(graph, RatingGraph) else RatingGraph(graph)
    m = _check_count(m, "m", g.num_users, ValueError)
    items = _host_ids(items, "items", g.num_items)
    if g.device is None:
        raise RuntimeError("igmc_b200 retrieval runs on a CUDA device (there is no CPU path)")
    err = torch.zeros(1, dtype=torch.int32, device=g.device)
    dv = torch.from_numpy(items.astype(np.int32)).to(g.device)
    users, paths = _corated(_lib.load(), g.shape[::-1], "igmc_corated_users", (C.byref(g._ct), dv.data_ptr(),
                                                                                len(items)),
                            len(items), m, exclude_rated, err, {})
    _lib.check_kernel_error(int(err.item()))
    return users, paths


# ---- rating sessions: public API ------------------------------------------------------------------------------------
def predict_sessions(model, sessions, session, items, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None,
                     batch_size=256, checkpoints=None, sample_seed=0):
    """eval-mode scores [P] (fp32, on the model's device) of the pairs (sessions.users[session[i]], items[i]), each
    with its target user's row taken from session ``session[i]`` (``RatingSessions``) and every other row and column
    from the graph, which is not changed.  Bit for bit ``predict_pairs`` of the same pair on the graph with that
    session's edits applied (same kernel plan and batch size); pair ids stay u * num_items + v.  Keywords as
    ``predict_pairs``'."""
    sessions = _check_sessions(sessions)
    sess, items, _ = _host_pairs((sessions.num_sessions, sessions.graph.num_items), session, items, first="session")
    if len(sess) == 0:
        return torch.zeros(0, dtype=torch.float32, device=model.flat_params.device)
    return _on_engine(model, sessions.graph, lambda eng: eng.predict_sessions(sessions, sess, items),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def recommend_sessions(model, sessions, k, *, items=None, exclude_rated=True, retrieve=None, draws=None, beta=0.0,
                       draw_seed=0, h=1, sample_ratio=1.0, max_nodes_per_hop=None, batch_size=256, checkpoints=None,
                       sample_seed=0):
    """per session the ``k`` best candidate items: (top_items [S, k] int64, top_scores [S, k] fp32), row s for
    session s.  Candidates and order as ``recommend``'s, with the session row as the user's ratings (``exclude_rated``,
    ``retrieve=M``); a 2-D ``items`` has one row per session.  Row s is bit for bit ``recommend`` for sessions.users[s]
    on the graph with session s's edits applied (same kernel plan and batch size); the graph is not changed.
    ``draws`` / ``beta`` / ``draw_seed``: ranked by mean + beta * std over draws, as in ``recommend``."""
    _draw_inputs(draws, beta, draw_seed, batch_size)
    sessions = _check_sessions(sessions)
    k = _ranking_inputs(k, batch_size, items, retrieve, sessions.num_sessions, sessions.graph.num_items)[0]
    return _on_engine(model, sessions.graph,
                      lambda eng: eng.recommend_sessions(sessions, k, items, exclude_rated, retrieve, draws, beta,
                                                         draw_seed),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def corated_items_sessions(sessions, m, exclude_rated=True):
    """``corated_items`` for sessions: per session the ``m`` items with the most bridges to its user, with N(u) the
    session row (and ``exclude_rated`` dropping its items) and the columns from the graph: (items [S, m], paths
    [S, m]) int32, row s bit for bit ``corated_items`` for sessions.users[s] on the graph with session s's edits
    applied.  One host synchronisation (the error word)."""
    sessions = _check_sessions(sessions)
    g = sessions.graph
    m = _check_count(m, "m", g.num_items, ValueError)
    err = torch.zeros(1, dtype=torch.int32, device=g.device)
    items, paths = _corated(_lib.load(), g.shape, "igmc_corated_sessions", (C.byref(g._c), C.byref(sessions._c)),
                            sessions.num_sessions, m, exclude_rated, err, {})
    _lib.check_kernel_error(int(err.item()))
    return items, paths


def elicit(model, sessions, n, targets, *, questions=None, h=1, sample_ratio=1.0, max_nodes_per_hop=None,
           batch_size=256, checkpoints=None, sample_seed=0):
    """per session the ``n`` items it should be asked to rate: (items [S, n] int64, impact [S, n] fp32) on the model's
    device, row s for session s.  A question asks session s about an item q not in its row; its answers are the rating
    labels a = 0..A-1 (A = model.num_relations).  x_a(t) is the eval score of (sessions.users[s], t) with the rating
    (q, a) added to s's row: bit for bit ``predict_sessions`` of a session with s's edits plus the edit (q, a + 1)
    (same pair id, sample_seed and checkpoint mean).  impact = the mean over s's real targets t, in slot order, of
    max_a x_a(t) - min_a x_a(t), in fp64 and rounded once; a NaN score makes it NaN.  ``targets``: one list for every
    session, or a 2-D array with a row per session (-1 = empty slot); duplicates count each time and rated items are
    allowed (a target equal to q has range 0: a pair's own rating is never in its subgraph).  ``questions``: every
    item (None), one list, or a 2-D array of per-session rows (-1 = empty slot); items of the session's row are never
    questions.  Order: ``recommend``'s (impact descending, item ascending, NaN last); empty slots -1 / -inf.  The
    results do not depend on batch_size, graph replay or the other sessions.  A question costs A x |targets| forwards;
    A x the target width <= batch_size, 1 <= n <= IGMC_TOPK_MAX = 256.  The graph is not changed."""
    sessions = _check_sessions(sessions)
    S, ni = sessions.num_sessions, sessions.graph.num_items
    _ranking_inputs(n, batch_size, questions, None, S, ni, "questions")
    _elicit_targets(targets, S, ni, model.num_relations, batch_size, np.arange(S))
    return _on_engine(model, sessions.graph, lambda eng: eng.elicit(sessions, n, targets, questions),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)


def question_impact(model, sessions, session, questions, targets, *, h=1, sample_ratio=1.0, max_nodes_per_hop=None,
                    batch_size=256, checkpoints=None, sample_seed=0):
    """what asking session ``session[i]`` about item ``questions[i]`` would do: a ``QuestionImpact`` of impact [P]
    (``elicit``'s key) and answer_mean [P, A] (per answer a the mean of x_a(t) over the session's real targets, in fp64
    in slot order, rounded once; a NaN score makes that answer's mean NaN) fp32 on the model's device.  ``targets`` and
    the keywords as ``elicit``'s.  ValueError for a question the session already rated."""
    sessions = _check_sessions(sessions)
    sess, q = _question_units(sessions, session, questions)
    A = model.num_relations
    _elicit_targets(targets, sessions.num_sessions, sessions.graph.num_items, A, batch_size, sess)
    if len(sess) == 0:
        dev = model.flat_params.device
        return QuestionImpact(torch.zeros(0, dtype=torch.float32, device=dev),
                              torch.zeros(0, A, dtype=torch.float32, device=dev))
    return _on_engine(model, sessions.graph, lambda eng: eng.question_impact(sessions, sess, q, targets),
                      h, sample_ratio, max_nodes_per_hop, batch_size, checkpoints, sample_seed)
