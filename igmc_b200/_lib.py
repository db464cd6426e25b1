"""ctypes binding of libigmc_b200.so (the C-ABI declared in include/igmc_b200.h).

There is NO fallback: if the shared library is missing or an entry point is absent the import of
the hot path fails loudly.  Build it with ``python -m igmc_b200.build`` (or
``__graft_entry__.build()``).
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libigmc_b200.so")

MAX_LAYERS = 8
REDUCE_WS_FLOATS = MAX_LAYERS * 32 * 64 + MAX_LAYERS * 32 + 64   # IGMC_REDUCE_WS_FLOATS
MAX_HOP = 3
HIDDEN = 32
LIN1_OUT = 128

ERR_NAMES = {
    0: "ok",
    1: "a subgraph side exceeded the node-list capacity (cap)",
    2: "batch edge capacity exceeded",
    3: "batch node capacity exceeded",
    4: "subgraph larger than the shared-memory plan of the model kernels (n_cap)",
    5: "malformed batch (edges not grouped by graph / node outside its graph / no target node)",
    6: "subgraph of more than 65535 nodes (beyond the 16-bit neighbour field of the edge lists)",
    7: "inference candidates: a user / item id outside the rating matrix or an inconsistent candidate plan",
    8: "graph update: a user / item id outside the graph's capacity or a value outside 0..256",
    9: "rating sessions: a session / item id out of range, a negative user id or a value outside 0..256",
    10: "online training draw: the rating graph has no ratings",
    11: "extraction: a rating label or a pair label outside 0..num_classes-1 (more ratings than class_values / "
        "the model's relations)",
}

TOPK_MAX = 256       # IGMC_TOPK_MAX
DRAWS_MAX = 256      # IGMC_DRAWS_MAX
COUNTERFACTUAL_MAX = 256   # IGMC_COUNTERFACTUAL_MAX
GROUP_MAX = 64       # IGMC_GROUP_MAX
GROUP_AGGREGATES = ("mean", "min", "max")   # IGMC_GROUP_AGG_MEAN, _MIN, _MAX

# Kernel plan values (igmc_model_plan): 0 generic kernels, 1..4 relation-space cluster kernels (CTAs per subgraph),
# PLAN_L2_BASE + c (c = 1, 2, 4, 8) the L2 plan with c CTAs per subgraph (IGMC_PLAN_L2 in include/igmc_b200.h).
PLAN_L2_BASE = 16
L2_MAX_NODES = 65535


def plan_l2(c):
    return PLAN_L2_BASE + int(c)


def l2_csize(plan):
    """CTAs per subgraph of an L2 plan value, 0 for every other plan"""
    c = int(plan) - PLAN_L2_BASE
    return c if c in (1, 2, 4, 8) else 0


def is_rs(plan):
    """a relation-space cluster plan (raw gradient rows, prepared weights, list images)"""
    return 0 < int(plan) <= 4


def ctas_per_graph(plan):
    return l2_csize(plan) or max(int(plan), 1)

p_i32 = C.c_void_p  # all device pointers travel as raw addresses
vp = C.c_void_p


class CSR(C.Structure):
    _fields_ = [("row_ptr", vp), ("col_idx", vp), ("rating", vp), ("col_ptr", vp), ("row_idx", vp),
                ("num_users", C.c_int32), ("num_items", C.c_int32)]


class Pairs(C.Structure):
    _fields_ = [("idx", vp), ("links_u", vp), ("links_v", vp), ("links_label", vp), ("pair_id", vp)]


class ExtractWS(C.Structure):
    _fields_ = [("nodes_u", vp), ("nodes_v", vp), ("n_u", vp), ("n_v", vp), ("row_cnt", vp), ("m_cnt", vp),
                ("col_cnt", vp), ("hop_off", vp), ("sync", vp)]


class BatchOut(C.Structure):
    _fields_ = [("node_cap", C.c_int32), ("edge_cap", C.c_int32), ("feat_dim", C.c_int32),
                ("x", vp), ("node_label", vp), ("batch", vp), ("node_gid", vp), ("edge_index", vp),
                ("edge_type", vp), ("y", vp), ("node_ptr", vp), ("edge_ptr", vp), ("graph_nu", vp),
                ("counts", vp), ("adj_in_ptr", vp), ("adj_in", vp), ("adj_eid", vp), ("adj_tmp", vp)]


class Store(C.Structure):
    _fields_ = [(k, vp) for k in ("node_off", "edge_off", "node_label", "node_gid", "edge_src", "edge_dst",
                                  "edge_type", "y", "graph_nu", "adj_ptr", "adj_in", "adj_eid")]


class Adj(C.Structure):
    _fields_ = [("in_ptr", vp), ("in_adj", vp), ("in_eid", vp), ("out_ptr", vp), ("out_adj", vp),
                ("out_eid", vp), ("tmp", vp), ("symmetric", C.c_int32)]


class Model(C.Structure):
    _fields_ = [("num_layers", C.c_int32), ("num_relations", C.c_int32), ("num_bases", C.c_int32),
                ("in_dim0", C.c_int32),
                ("off_att", C.c_int32 * MAX_LAYERS), ("off_basis", C.c_int32 * MAX_LAYERS),
                ("off_root", C.c_int32 * MAX_LAYERS), ("off_bias", C.c_int32 * MAX_LAYERS),
                ("off_lin1_w", C.c_int32), ("off_lin1_b", C.c_int32), ("off_lin2_w", C.c_int32),
                ("off_lin2_b", C.c_int32), ("conv_param_count", C.c_int32), ("param_count", C.c_int32),
                ("multiply_by", C.c_float), ("readout", C.c_int32), ("list_hint", C.c_int32)]


class Dropout(C.Structure):
    _fields_ = [("adj_dropout", C.c_float), ("hidden_dropout", C.c_float), ("seed", C.c_uint64),
                ("seed_dev", vp), ("edge_keep", vp), ("hidden_keep", vp)]


class Saved(C.Structure):
    _fields_ = [("states", vp), ("zsave", vp), ("inv_deg", vp), ("feat", vp), ("hid", vp),
                ("hid_gscale", vp), ("pred", vp), ("target", vp), ("node_cap", C.c_int32), ("dstate", vp), ("wprep", vp), ("prof", vp),
                ("gate", vp), ("l2_scratch", vp), ("rel_inv_deg", vp)]


class Stage(C.Structure):
    _fields_ = [("tab", vp), ("ent", vp), ("inv_deg", vp), ("tab_ints", C.c_int32), ("lcap", C.c_int32),
                ("chunk", C.c_int32), ("cluster", C.c_int32)]


class Candidates(C.Structure):
    _fields_ = [("users", vp), ("cand", vp), ("pair_u", vp), ("pair_v", vp), ("user_off", vp), ("rated_off", vp),
                ("rated_pos", vp), ("num_pairs", C.c_int64), ("num_query", C.c_int32), ("num_cand", C.c_int32),
                ("exclude_rated", C.c_int32), ("per_user", C.c_int32)]


class Sessions(C.Structure):
    _fields_ = [("users", vp), ("row_ptr", vp), ("col_idx", vp), ("rating", vp), ("num_sessions", C.c_int32),
                ("max_row_deg", C.c_int32)]


class Counterfactual(C.Structure):
    _fields_ = [("users", vp), ("items", vp), ("rivals", vp), ("size", vp), ("removed", vp), ("num_query", C.c_int32),
                ("max_removals", C.c_int32)]


GRAPH_UPDATE_HEADER = ("nnz", "num_users", "num_items", "max_row_deg", "max_col_deg", "inserted", "changed",
                       "removed")   # igmc_graph_update_header_t: these int64 fields, then int32 status, int32 err
GRAPH_UPDATE_OVER_CAPACITY, GRAPH_UPDATE_OVER_INT32 = 1, 2


MAX_RANKS = 8


class Comm(C.Structure):
    _fields_ = [("grad", vp * MAX_RANKS), ("flag", vp * MAX_RANKS), ("state", vp), ("world", C.c_int32),
                ("rank", C.c_int32), ("stride", C.c_int32), ("pad_", C.c_int32)]


class SortPool(C.Structure):
    _fields_ = [(k, C.c_int32) for k in ("k", "width", "state_stride", "c1", "c2", "kw2", "t1", "t2", "dense_dim",
                                         "off_conv1_w", "off_conv1_b", "off_conv2_w", "off_conv2_b", "off_lin1_w",
                                         "off_lin1_b", "off_lin2_w", "off_lin2_b", "param_begin", "param_end")]


class SortPoolSaved(C.Structure):
    _fields_ = [(k, vp) for k in ("rank", "perm", "act1", "pool", "flat", "hid", "hid_gscale", "pred", "dhid",
                                  "gpart")]


_SIGS = {
    "igmc_extract_batch": [C.POINTER(CSR), C.POINTER(Pairs), C.c_int, C.c_int, C.c_int, C.c_double, C.c_uint64, vp, C.c_int,
                           vp, vp, vp, vp, C.POINTER(ExtractWS), vp, C.c_int, C.c_int, C.POINTER(BatchOut), vp, vp],
    "igmc_extract_plan": [C.c_int] * 10,
    "igmc_assemble_batch": [C.POINTER(Store), vp, C.c_int, C.POINTER(BatchOut), vp, vp],
    "igmc_batch_ptrs": [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp],
    "igmc_batch_prepare": [vp, C.c_int64, vp, vp, vp, C.c_int, C.c_int, C.POINTER(Adj), vp, vp],
    "igmc_forward": [C.POINTER(Model), vp, vp, vp, vp, C.POINTER(Adj), C.c_int, C.c_int, C.POINTER(Dropout),
                     C.c_int, C.POINTER(Saved), vp, C.c_float, vp, vp, C.c_int, C.POINTER(Stage), vp, vp],
    "igmc_backward": [C.POINTER(Model), vp, vp, vp, vp, C.POINTER(Adj), C.c_int, C.c_int, C.POINTER(Dropout),
                      C.POINTER(Saved), vp, vp, vp, C.c_int, C.POINTER(Stage), vp, vp],
    "igmc_forward_backward": [C.POINTER(Model), vp, vp, vp, vp, C.POINTER(Adj), C.c_int, C.c_int, C.POINTER(Dropout),
                              C.POINTER(Saved), vp, C.c_float, vp, vp, vp, vp, C.c_int, C.POINTER(Stage),
                              C.POINTER(Stage), vp, vp],
    "igmc_raw_grad_count": [C.POINTER(Model)],
    "igmc_stage_plan": [C.POINTER(Model), C.c_int, C.c_int, C.c_int, C.POINTER(Stage)],
    "igmc_stage_lists": [C.POINTER(Model), vp, vp, C.POINTER(Adj), C.c_int, C.c_int, C.POINTER(Dropout), C.c_int,
                         C.POINTER(Stage), C.POINTER(Stage), vp, vp],
    "igmc_grad_reduce": [C.POINTER(Model), vp, C.c_int, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, C.c_float, C.c_float,
                         C.c_float, vp, vp, vp, vp],
    "igmc_adam_step": [vp, vp, vp, vp, vp, C.c_int, C.c_float, vp, C.c_float, C.c_float, C.c_float, C.c_float,
                       C.c_float, vp, vp, C.c_float, vp],
    "igmc_reduce_update": [C.POINTER(Model), vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, C.c_float, C.c_float,
                           C.POINTER(Comm), vp, vp, vp, C.c_float, vp, C.c_float, C.c_float, C.c_float, C.c_float,
                           C.c_float, vp, vp, C.c_float, vp, vp, vp, C.c_int, vp, vp],
    "igmc_reduce_update_grid": [C.POINTER(Model), C.POINTER(C.c_int), C.POINTER(C.c_int)],
    "igmc_comm_alloc": [C.c_int64, C.POINTER(C.c_void_p), C.c_char_p],
    "igmc_comm_open": [C.c_char_p, C.POINTER(C.c_void_p)],
    "igmc_comm_close": [vp],
    "igmc_comm_free": [vp],
    "igmc_prep_weights": [C.POINTER(Model), vp, vp, vp],
    "igmc_gate_wait": [vp, C.c_int, C.c_int, vp],
    "igmc_candidate_plan": [C.POINTER(CSR), C.POINTER(Candidates), vp, vp],
    "igmc_candidate_pairs": [C.POINTER(CSR), C.POINTER(Candidates), vp, C.c_int, vp, vp, vp, vp, vp, vp],
    "igmc_item_query_pairs": [C.c_int, C.c_int, vp, vp, vp, vp, vp],
    "igmc_topk_merge": [vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp],
    "igmc_score_scatter": [vp, C.c_int, C.c_int, vp, vp, vp],
    "igmc_topk_fits": [C.c_int, C.c_int],
    "igmc_candidate_lists_ws_bytes": [C.c_int, C.c_int, C.POINTER(C.c_int64)],
    "igmc_candidate_lists": [C.POINTER(CSR), C.POINTER(Candidates), vp, C.c_int, vp, vp, C.c_int64, vp, vp],
    "igmc_explain_count": [vp, vp, C.c_int, vp, vp],
    "igmc_explain_offsets": [vp, C.c_int, vp, vp],
    "igmc_occlusion_pairs": [C.POINTER(CSR), vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, vp, vp],
    "igmc_occlusion_mask": [C.POINTER(BatchOut), C.c_int, vp, vp, vp, vp, vp, vp, vp, vp],
    "igmc_occlusion_order_ws_bytes": [C.c_int, C.c_int64, C.POINTER(C.c_int64)],
    "igmc_occlusion_order": [vp, vp, vp, C.c_int, C.c_int64, vp, vp, vp, C.c_int, vp, C.c_int64, vp, vp, vp, vp, vp],
    "igmc_edge_grad": [C.POINTER(Model), vp, vp, vp, vp, C.POINTER(Adj), C.c_int, C.c_int, C.POINTER(Dropout),
                       C.POINTER(Saved), vp, vp, C.c_int, vp, vp],
    "igmc_edge_grad_scatter": [C.POINTER(BatchOut), C.c_int, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp],
    "igmc_explain_node_count": [vp, vp, C.c_int, vp, vp],
    "igmc_node_occlusion_mask": [C.POINTER(BatchOut), C.c_int, vp, vp, vp, vp, vp, vp, vp, vp],
    "igmc_node_grad_scatter": [C.POINTER(BatchOut), C.c_int, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp],
    "igmc_pair_factor_count": [C.POINTER(Model)],
    "igmc_pair_seed": [vp, vp, vp, C.c_int, C.c_float, vp, vp],
    "igmc_pair_grad": [C.POINTER(Model), vp, C.c_int, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, C.c_int, vp, C.c_int,
                       vp, vp],
    "igmc_self_influence": [C.POINTER(Model), C.c_int, vp, vp, vp, C.c_float, vp, vp],
    "igmc_influence_ws_bytes": [C.POINTER(Model), C.c_int, C.c_int, C.POINTER(C.c_int64)],
    "igmc_influence_accum": [C.POINTER(Model), C.c_int, C.c_int, vp, vp, vp, vp, C.c_float, C.c_int, vp, C.c_int64,
                             vp, vp],
    "igmc_influence_topk": [vp, C.c_int, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp],
    "igmc_corated_ws_bytes":[C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int64)],
    "igmc_corated_items": [C.POINTER(CSR), vp, C.c_int, C.c_int, C.c_int, vp, C.c_int64, vp, vp, vp, vp],
    "igmc_corated_users": [C.POINTER(CSR), vp, C.c_int, C.c_int, C.c_int, vp, C.c_int64, vp, vp, vp, vp],
    "igmc_graph_update_ws_bytes": [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int64)],
    "igmc_graph_update_plan": [C.POINTER(CSR), C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_int, C.c_int,
                               C.c_int, vp, C.c_int64, vp, vp, vp],
    "igmc_graph_update_apply": [C.POINTER(CSR), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int64, C.c_int,
                                C.c_int, C.c_int, vp],
    "igmc_session_ws_bytes": [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int64)],
    "igmc_session_plan": [C.POINTER(CSR), vp, C.c_int, vp, vp, vp, C.c_int, vp, C.c_int64, vp, vp, vp],
    "igmc_session_apply": [C.POINTER(CSR), vp, C.c_int, C.c_int, vp, C.c_int64, vp, vp, vp, vp],
    "igmc_session_pairs": [C.POINTER(Sessions), C.c_int, C.c_int, vp, vp, vp, vp, vp, vp],
    "igmc_extract_sessions": [C.POINTER(CSR), C.POINTER(Sessions), vp, C.POINTER(Pairs), C.c_int, C.c_int, C.c_int,
                              C.c_double, C.c_uint64, vp, C.c_int, C.POINTER(ExtractWS), vp, C.c_int, C.c_int,
                              C.POINTER(BatchOut), vp, vp],
    "igmc_corated_sessions": [C.POINTER(CSR), C.POINTER(Sessions), C.c_int, C.c_int, vp, C.c_int64, vp, vp, vp, vp],
    "igmc_online_draw": [C.POINTER(CSR), vp, vp, C.c_int, vp, C.c_int64, vp, C.c_int, C.c_uint64, C.c_uint64, C.c_int,
                         vp, vp, vp, vp, vp, vp, vp],
    "igmc_online_recent_append": [vp, vp, vp, C.c_int, vp, vp, C.c_int, vp, vp, vp],
    "igmc_draws_expand": [C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp],
    "igmc_draws_mask": [C.POINTER(BatchOut), C.c_int, vp, vp, vp, C.c_float, C.c_uint64, vp, vp, vp],
    "igmc_draws_stats": [vp, C.c_int, C.c_int, C.c_int, vp, C.c_double, vp, vp, vp, vp, vp],
    "igmc_counterfactual_pairs": [C.POINTER(CSR), C.POINTER(Counterfactual), vp, C.c_int, vp, C.c_int, vp, vp, vp, vp,
                                  vp, vp, vp, vp, C.c_int, vp, vp, vp],
    "igmc_counterfactual_select": [C.POINTER(CSR), C.POINTER(Counterfactual), vp, vp, C.c_int, vp, vp, vp, vp, vp, vp,
                                   vp, vp],
    "igmc_elicit_pairs": [C.POINTER(Sessions), C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp,
                          vp, vp, vp, vp, vp, C.c_int, vp, vp, vp],
    "igmc_elicit_stats": [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp],
    "igmc_group_rows": [C.POINTER(CSR), vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp],
    "igmc_group_pairs": [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp],
    "igmc_group_stats": [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp],
    "igmc_diverse_ws_bytes": [C.c_int, C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int)],
    "igmc_item_union": [vp, C.c_int64, C.c_int, vp, vp, vp, vp, vp, vp],
    "igmc_cocount": [C.POINTER(CSR), vp, C.c_int, vp, C.c_int64, vp],
    "igmc_diverse_select": [C.POINTER(CSR), vp, vp, C.c_int, C.c_int, C.c_int, C.c_float, vp, C.c_int, vp, vp, vp, vp,
                            vp, vp],
    "igmc_item_cosine": [C.POINTER(CSR), vp, C.c_int, vp, C.c_int, vp, vp, vp, vp],
    "igmc_rescore_plan_ws_bytes":[C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int)],
    "igmc_rescore_plan": [C.POINTER(CSR), vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, C.c_int, vp, C.c_int64, vp, vp,
                          C.c_int64, vp, vp, vp, vp],
    "igmc_cache_invalidate": [C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, vp],
    "igmc_cache_settle": [C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp],
    "igmc_build_info": [],
    "igmc_model_plan": [C.POINTER(Model), C.c_int, C.c_int, C.c_int],
    "igmc_sortpool_plan": [C.POINTER(SortPool), C.c_int, C.c_int],
    "igmc_sortpool_forward": [C.POINTER(SortPool), vp, vp, vp, C.c_int, C.c_int, C.POINTER(Dropout), C.c_int,
                              C.POINTER(SortPoolSaved), vp, C.c_float, vp, vp, vp, vp],
    "igmc_sortpool_backward": [C.POINTER(SortPool), vp, vp, vp, C.c_int, C.c_int, C.POINTER(SortPoolSaved), vp, vp,
                               C.c_float, vp, vp, vp],
}

EXPORTS = tuple(_SIGS)
_lib = None


def load():
    """dlopen the library once; raises if it (or a declared symbol) is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "igmc_b200: %s not found - build the CUDA extension first (python -m igmc_b200.build). "
            "There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in _SIGS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.argtypes = argtypes
        fn.restype = C.c_int
    if lib.igmc_build_info() != 90:
        raise RuntimeError("igmc_b200: library was not built for sm_90a")
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        raise RuntimeError("igmc_b200: %s failed with code %d" % (what, rc))


def check_kernel_error(code):
    """raise for a nonzero code read from a kernel error word (the caller reads, and if it wants clears, the word)"""
    if code:
        raise RuntimeError("igmc_b200 kernel error %d: %s" % (code, ERR_NAMES.get(code, "?")))


def ptr(t):
    """device address of a torch tensor (or None -> NULL)."""
    return None if t is None else t.data_ptr()
