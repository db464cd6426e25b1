"""Drop-in for the hot-path half of the reference's ``util_functions.py``.

Same public names and signatures as the reference (``MyDynamicDataset`` util_functions.py:113-145,
``MyDataset`` :69-110, ``SparseRowIndexer``/``SparseColIndexer`` :20-66 replaced by ``RatingGraph``),
but ``get``/batching run as CUDA kernels over a device-resident CSR/CSC through the C-ABI in
include/igmc_b200.h.  The ``Data``/``Batch`` objects expose the PyG attribute surface the reference's
model and train loop touch (``x, edge_index, edge_type, y, batch, num_graphs, to()``).

No CPU fallback: constructing a dataset or extracting without a CUDA device raises.
"""
import collections
import ctypes as C
import os

import numpy as np
import torch

from . import _lib

__all__ = ["RatingGraph", "GraphCapacity", "graph_update_host", "Data", "Batch", "SubgraphExtractor", "MyDynamicDataset", "MyDataset"]


def _require_cuda(device=None):
    if not torch.cuda.is_available():
        raise RuntimeError("igmc_b200 needs a CUDA device (H100); there is no CPU path")
    return torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)


def _stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _on_device(a, dtype, dev):
    """``a`` (host array or tensor) as a contiguous ``dtype`` tensor on ``dev``; a tensor that already is one is
    returned as is (no copy)."""
    if not torch.is_tensor(a):
        a = torch.as_tensor(np.asarray(a), dtype=dtype)
    return a.to(device=dev, dtype=dtype).contiguous()


class DevView(object):
    """Device-visible window of a PINNED host tensor: ``data_ptr()`` is the address the kernels use (under unified
    addressing a cudaHostAlloc'd buffer has the same address on the host and on the device), so they read / write the
    host memory directly and no copy is ever launched.  Carries just what the launch code needs (``data_ptr``,
    ``numel``, slicing).  Used for the per-step inputs (a few hundred bytes of indices and seeds) and the per-step
    loss read-back of the train engine."""

    def __init__(self, pinned, off=0, n=None):
        assert pinned.is_pinned() and pinned.is_contiguous() and pinned.dim() == 1
        self.pinned, self.off = pinned, int(off)
        self.n = int(pinned.numel() - off if n is None else n)

    def data_ptr(self):
        return self.pinned.data_ptr() + self.off * self.pinned.element_size()

    def numel(self):
        return self.n

    def __len__(self):
        return self.n

    def __getitem__(self, sl):
        assert isinstance(sl, slice) and sl.step in (None, 1)
        lo, hi, _ = sl.indices(self.n)
        return DevView(self.pinned, self.off + lo, max(0, hi - lo))


def _device_index(idx, dev):
    """dataset indices as an int64 device tensor; a ``DevView`` (int64 indices in mapped host memory) is used as is"""
    if isinstance(idx, DevView):
        return idx
    if not torch.is_tensor(idx):
        idx = torch.as_tensor(np.asarray(idx), dtype=torch.int64)
    return idx.to(device=dev, dtype=torch.int64)


GraphCapacity = collections.namedtuple("GraphCapacity", "users items nnz")

_GRAPH_ARRAYS = (("row_ptr", np.int32), ("col_idx", np.int32), ("rating", np.uint8), ("col_ptr", np.int32),
                 ("row_idx", np.int32))


class RatingGraph(object):
    """Flat device CSR + CSC of ``adj_train`` (scipy CSR, stored value = rating label + 1,
    preprocessing.py:190-197).  Replaces SparseRowIndexer/SparseColIndexer (util_functions.py:20-66).

    The device arrays are allocated at capacity (``reserve_*`` beyond the matrix) so that ``update`` can insert ratings
    and add users / items in place; the five device pointers never change.  ``version`` counts the updates that
    changed the graph; ``host`` is a mirror refreshed on its first access after one."""

    def __init__(self, A, device=None, *, reserve_nnz=0, reserve_users=0, reserve_items=0):
        import scipy.sparse as ssp
        if min(int(reserve_nnz), int(reserve_users), int(reserve_items)) < 0:
            raise ValueError("reserve_nnz / reserve_users / reserve_items must be >= 0")
        A = ssp.csr_matrix(A)
        A.sum_duplicates()
        A.sort_indices()
        self.shape = A.shape
        self.nnz = int(A.nnz)
        self.num_users, self.num_items = int(A.shape[0]), int(A.shape[1])
        lab = np.rint(A.data).astype(np.int64) - 1
        if self.nnz and (lab.min() < 0 or lab.max() > 255):
            raise ValueError("rating labels must lie in 0..255")
        Cc = A.tocsc()
        Cc.sort_indices()
        self.max_row_deg = int(np.diff(A.indptr).max()) if self.nnz else 0
        self.max_col_deg = int(np.diff(Cc.indptr).max()) if self.nnz else 0
        self._host = dict(row_ptr=A.indptr.astype(np.int32), col_idx=A.indices.astype(np.int32),
                          rating=lab.astype(np.uint8), col_ptr=Cc.indptr.astype(np.int32),
                          row_idx=Cc.indices.astype(np.int32))
        self._cap = GraphCapacity(self.num_users + int(reserve_users), self.num_items + int(reserve_items),
                                  self.nnz + int(reserve_nnz))
        self.version = 0
        self._host_version = 0
        self._upd = None           # update workspace, header and error word (allocated on the first update)
        self.device = None
        self.dev = {}
        if device is not None or torch.cuda.is_available():
            self.to(_require_cuda(device))

    @property
    def capacity(self):
        """(users, items, nnz) the device arrays hold: ids up to users - 1 / items - 1 and nnz ratings"""
        return self._cap

    @property
    def host(self):
        """host copies of the five arrays, cut to the current shape and nnz (one device-to-host copy per array on the
        first access after an update)"""
        if self._host_version != self.version:
            d, n = self.dev, self.nnz
            self._host = dict(row_ptr=d["row_ptr"][:self.num_users + 1].cpu().numpy(),
                              col_idx=d["col_idx"][:n].cpu().numpy(), rating=d["rating"][:n].cpu().numpy(),
                              col_ptr=d["col_ptr"][:self.num_items + 1].cpu().numpy(),
                              row_idx=d["row_idx"][:n].cpu().numpy())
            self._host_version = self.version
        return self._host

    def to(self, device):
        h = self.host
        self.device = torch.device(device)
        cu, ci, cn = self._cap
        size = dict(row_ptr=cu + 1, col_idx=cn, rating=cn, col_ptr=ci + 1, row_idx=cn)
        self.dev = {}
        for k, dt in _GRAPH_ARRAYS:
            # a zero-length index array still needs a valid pointer
            t = torch.zeros(max(size[k], 1), dtype=_TORCH_OF[dt], device=self.device)
            if len(h[k]):
                t[:len(h[k])] = torch.from_numpy(h[k]).to(self.device)
            self.dev[k] = t
        self._upd = None
        self._make_c()
        return self

    def _make_c(self):
        d = self.dev
        self._c = _lib.CSR(d["row_ptr"].data_ptr(), d["col_idx"].data_ptr(), d["rating"].data_ptr(),
                           d["col_ptr"].data_ptr(), d["row_idx"].data_ptr(), self.num_users, self.num_items)
        # the transposed view: rows are items, columns users (no ratings: they are not in column order).  What the
        # candidate kernels and the retriever read on item-side runs (include/igmc_b200.h: igmc_item_query_pairs)
        self._ct = _lib.CSR(d["col_ptr"].data_ptr(), d["row_idx"].data_ptr(), None, d["row_ptr"].data_ptr(),
                            d["col_idx"].data_ptr(), self.num_items, self.num_users)

    def node_cap(self, max_nodes_per_hop, h=1, max_row_deg=None):
        """capacity of one side's node list: target + per hop min(mnph, largest possible fringe) (hop 1: a row or
        a column of the matrix; later hops: up to the whole side).  ``max_row_deg``: the longest target row when it
        may be longer than the graph's (rating sessions)."""
        d = max(self.max_row_deg if max_row_deg is None else max(self.max_row_deg, int(max_row_deg)),
                self.max_col_deg)
        side = max(self.num_users, self.num_items)
        if max_nodes_per_hop is not None:
            d = min(d, int(max_nodes_per_hop))
            side = min(side, int(max_nodes_per_hop))
        return min(1 + d + (int(h) - 1) * side, 1 + max(self.num_users, self.num_items))

    # ---- in-place update (igmc_graph_update_plan / _apply, csrc/graph_update.cu) ------------------------------------
    def update(self, users, items, values, shape=None):
        """Apply ratings in place: ``values[i]`` = rating label + 1 (1..256) inserts or overwrites the rating of
        (users[i], items[i]), 0 deletes it (an absent rating: nothing); the last occurrence of a pair wins.  Ids below
        ``capacity`` grow ``shape`` to cover them, ``shape=`` grows it further (users / items without ratings); the
        shape never shrinks.  Host arrays are validated here; int32 device tensors are used in place and validated by
        the kernel (RuntimeError with IGMC_ERR_GRAPH_UPDATE, nothing changed).  ValueError, with nothing changed, if
        the result would exceed the nnz capacity.  One host synchronisation.  Returns dict(inserted=, changed=,
        removed=): the ratings added, relabelled and deleted."""
        cu, ci, cn = self._cap
        u, v, x, D = _update_inputs(users, items, values, cu, ci)
        req = _update_shape(shape, self.shape, self._cap)
        counts = dict(inserted=0, changed=0, removed=0)
        if D == 0 and req == self.shape:
            return counts
        if self.device is None:
            raise RuntimeError("igmc_b200 graph updates run on a CUDA device (there is no CPU path)")
        if D == 0:      # shape only: the new rows / columns are empty
            self.dev["row_ptr"][self.num_users + 1:req[0] + 1] = self.nnz
            self.dev["col_ptr"][self.num_items + 1:req[1] + 1] = self.nnz
            self._commit(self.nnz, req[0], req[1], self.max_row_deg, self.max_col_deg)
            return counts
        lib, dev = _lib.load(), self.device
        u, v, x = (_on_device_i32(a, dev) for a in (u, v, x))
        nbytes = C.c_int64(0)
        _lib.check(lib.igmc_graph_update_ws_bytes(D, cu, ci, cn, C.byref(nbytes)), "igmc_graph_update_ws_bytes")
        if self._upd is None:
            self._upd = dict(ws=torch.empty(0, dtype=torch.uint8, device=dev),
                             header=torch.zeros(len(_lib.GRAPH_UPDATE_HEADER) + 1, dtype=torch.int64, device=dev),
                             err=torch.zeros(1, dtype=torch.int32, device=dev))
        w = self._upd
        if w["ws"].numel() < nbytes.value:
            w["ws"] = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        args = (C.byref(self._c), self.nnz, cu, ci, cn)
        _lib.check(lib.igmc_graph_update_plan(*args, u.data_ptr(), v.data_ptr(), x.data_ptr(), D, req[0], req[1],
                                              w["ws"].data_ptr(), w["ws"].numel(), w["header"].data_ptr(),
                                              w["err"].data_ptr(), _stream_ptr()), "igmc_graph_update_plan")
        hdr = w["header"].cpu().numpy()             # the update's one host synchronisation
        h = dict(zip(_lib.GRAPH_UPDATE_HEADER, (int(a) for a in hdr)))
        status, err = (int(a) for a in hdr[-1:].view(np.int32))
        if err:
            w["err"].zero_()
        _lib.check_kernel_error(err)
        if status:
            raise ValueError("the update would leave %d ratings, beyond the graph's capacity of %d%s (reserve_nnz "
                             "makes room)" % (h["nnz"], cn, " and int32" if status == _lib.GRAPH_UPDATE_OVER_INT32
                                              else ""))
        counts = dict(inserted=h["inserted"], changed=h["changed"], removed=h["removed"])
        if any(counts.values()) or (h["num_users"], h["num_items"]) != self.shape:
            _lib.check(lib.igmc_graph_update_apply(*args, D, w["ws"].data_ptr(), w["ws"].numel(), h["nnz"],
                                                   h["num_users"], h["num_items"], _stream_ptr()),
                       "igmc_graph_update_apply")
            self._commit(h["nnz"], h["num_users"], h["num_items"], h["max_row_deg"], h["max_col_deg"])
        return counts

    def _commit(self, nnz, nu, ni, max_row_deg, max_col_deg):
        self.nnz, self.max_row_deg, self.max_col_deg = int(nnz), int(max_row_deg), int(max_col_deg)
        if (nu, ni) != self.shape:
            self.num_users, self.num_items = int(nu), int(ni)
            self.shape = (self.num_users, self.num_items)
            self._make_c()
        self.version += 1


_TORCH_OF = {np.int32: torch.int32, np.uint8: torch.uint8}


def _cuda_ints(a, name):
    """True for a CUDA tensor, which must hold integers (TypeError for a float, complex or bool dtype); False for host
    data"""
    if not (torch.is_tensor(a) and a.device.type == "cuda"):
        return False
    if a.is_floating_point() or a.is_complex() or a.dtype == torch.bool:
        raise TypeError("%s must be integers, not %s" % (name, a.dtype))
    return True


def _update_inputs(users, items, values, hi_users, hi_items, names=("users", "items", "values")):
    """(users, items, values, D) of edits in ``RatingGraph.update``'s encoding, the arrays called ``names``: host arrays
    validated here (IndexError for an id outside [0, hi_users) / [0, hi_items), ValueError for a value outside 0..256 or
    unequal lengths); device tensors are passed on unchecked (the kernel checks them)"""
    arrs = []
    for name, a in zip(names, (users, items, values)):
        if _cuda_ints(a, name):
            arrs.append(a.reshape(-1))
            continue
        a = np.asarray(a.cpu().numpy() if torch.is_tensor(a) else a).reshape(-1)
        if a.size and not np.issubdtype(a.dtype, np.integer):
            raise TypeError("%s must be integers, not %s" % (name, a.dtype))
        arrs.append(a.astype(np.int64))
    n = [int(a.numel()) if torch.is_tensor(a) else len(a) for a in arrs]
    if len(set(n)) != 1:
        raise ValueError("%s, %s and %s must have the same length (%d, %d, %d)" % (names + tuple(n)))
    for a, name, hi in zip(arrs, names, (hi_users, hi_items)):
        if not torch.is_tensor(a) and a.size and (a.min() < 0 or a.max() >= hi):
            bad = int(a.min()) if a.min() < 0 else int(a.max())
            raise IndexError("%s: id %d out of range [0, %d)" % (name, bad, hi))
    x = arrs[2]
    if not torch.is_tensor(x) and x.size and (x.min() < 0 or x.max() > 256):
        raise ValueError("%s must be rating label + 1 (1..256) or 0 (delete), got %d"
                         % (names[2], int(x.min()) if x.min() < 0 else int(x.max())))
    return arrs[0], arrs[1], arrs[2], n[0]


def _update_shape(shape, cur, cap):
    if shape is None:
        return tuple(cur)
    shape = tuple(int(a) for a in shape)
    if len(shape) != 2:
        raise ValueError("shape must be (num_users, num_items)")
    if shape[0] < cur[0] or shape[1] < cur[1]:
        raise ValueError("shape %s would shrink the graph's %s: the id space never shrinks" % (shape, tuple(cur)))
    if shape[0] > cap.users or shape[1] > cap.items:
        raise ValueError("shape %s beyond the graph's capacity (%d, %d)" % (shape, cap.users, cap.items))
    return shape


def _on_device_i32(a, dev):
    """int32 device tensor (an int32 device tensor is used in place; wider ones are clamped first, so that an id
    beyond int32 stays invalid)"""
    if torch.is_tensor(a) and a.device.type == "cuda":
        if a.dtype != torch.int32:
            a = a.clamp(-1, 2 ** 31 - 1).to(torch.int32)
        return a.contiguous()
    return torch.from_numpy(np.clip(a, -1, 2 ** 31 - 1).astype(np.int32)).to(dev)


def graph_update_host(host, shape, users, items, values, shape_req=None):
    """numpy twin of igmc_graph_update_plan + _apply on the host arrays of a graph of ``shape``: (new host arrays,
    header dict).  Restates the kernels' steps: stable (u, v) order, last entry of a pair kept, classification by
    binary search in the row, new lengths and pointers from the net counts, merge positions
    n0 + (j - o0) + (inserted - deleted with a smaller id) for old entries and n0 + q + the same for inserted ones."""
    users, items, values = (np.asarray(a, np.int64).reshape(-1) for a in (users, items, values))
    nu, ni = shape
    rp, ci, rt = (np.asarray(host[k], np.int64) for k in ("row_ptr", "col_idx", "rating"))
    cp, ri = (np.asarray(host[k], np.int64) for k in ("col_ptr", "row_idx"))
    D = len(users)
    req = (0, 0) if shape_req is None else shape_req
    if D == 0:
        raise ValueError("the twin models a non-empty delta")
    o = np.lexsort((items, users))                             # stable
    su, sv, sx = users[o], items[o], values[o]
    keep = np.r_[(su[1:] != su[:-1]) | (sv[1:] != sv[:-1]), True]
    cls = np.zeros(D, np.int64)                                # 0 no-op, 1 insert, 2 change, 3 delete
    lab = np.zeros(D, np.int64)
    for i in np.flatnonzero(keep):
        a, b, x = su[i], sv[i], sx[i]
        p = -1
        if a < nu and b < ni:
            q = rp[a] + np.searchsorted(ci[rp[a]:rp[a + 1]], b)
            if q < rp[a + 1] and ci[q] == b:
                p = q
        if x > 0:
            lab[i] = x - 1
            cls[i] = 1 if p < 0 else (2 if rt[p] != x - 1 else 0)
        elif p >= 0:
            cls[i] = 3
    nu2 = max(nu, req[0], int(su.max()) + 1)
    ni2 = max(ni, req[1], int(sv.max()) + 1)
    # the column side: the same entries stably ordered by (v, u)
    oc = np.lexsort((su, sv))
    new_rp, new_ci, new_rt = _merge_side_host(rp, ci, rt, nu, nu2, su, sv, cls, lab)
    new_cp, new_ri, _ = _merge_side_host(cp, ri, None, ni, ni2, sv[oc], su[oc], cls[oc], None)
    nnz = int(new_rp[-1])
    hdr = dict(nnz=nnz, num_users=nu2, num_items=ni2, max_row_deg=int(np.diff(new_rp).max(initial=0)),
               max_col_deg=int(np.diff(new_cp).max(initial=0)), inserted=int((cls == 1).sum()),
               changed=int((cls == 2).sum()), removed=int((cls == 3).sum()))
    out = dict(row_ptr=new_rp.astype(np.int32), col_idx=new_ci.astype(np.int32), rating=new_rt.astype(np.uint8),
               col_ptr=new_cp.astype(np.int32), row_idx=new_ri.astype(np.int32))
    return out, hdr


def _merge_side_host(ptr, idx, rating, n_old, n_new, a, b, cls, lab):
    """one side of the twin: rows r < n_new from the old rows (ptr, idx[, rating]) and the delta entries (a = row,
    b = other id, ascending (a, b)) classified ``cls``"""
    pk = np.where(cls == 1, 1, np.where(cls == 3, -1, 0))
    scan = np.concatenate([[0], np.cumsum(pk)])                 # exclusive net counts, scan[D] = total
    ds = np.searchsorted(a, np.arange(n_new), "left")
    de = np.searchsorted(a, np.arange(n_new), "right")
    old_len = np.zeros(n_new, np.int64)
    old_len[:n_old] = np.diff(ptr)
    new_ptr = np.concatenate([[0], np.cumsum(old_len + scan[de] - scan[ds])])
    optr = np.concatenate([ptr, np.full(n_new - n_old, ptr[-1], np.int64)])    # rows past the old shape: empty
    M = int(max(idx.max(initial=0), b.max(initial=0))) + 1
    rows = np.repeat(np.arange(n_old), np.diff(ptr))
    key_old, key_d = rows * M + idx, a * M + b
    out_idx = np.full(int(new_ptr[-1]), -1, np.int64)
    out_rt = np.zeros(int(new_ptr[-1]), np.int64) if rating is not None else None
    # old entry j: dropped when deleted, else n0 + (j - o0) + net count of the run's entries with a smaller id
    lo, hi = np.searchsorted(key_d, key_old, "left"), np.searchsorted(key_d, key_old, "right")
    k = np.where(hi > lo, cls[np.maximum(hi - 1, 0)], 0)
    j = np.arange(len(idx))
    dst = new_ptr[rows] + (j - ptr[rows]) + scan[lo] - scan[ds[rows]]
    live = k != 3
    out_idx[dst[live]] = idx[live]
    if rating is not None:
        out_rt[dst[live]] = np.where(k == 2, lab[np.maximum(hi - 1, 0)], rating)[live]
    # inserted entry p: n0 + (old entries of the row with a smaller id) + the same count
    p = np.flatnonzero(cls == 1)
    r = a[p]
    q = np.searchsorted(key_old, key_d[p]) - optr[r]
    dst = new_ptr[r] + q + scan[p] - scan[ds[r]]
    out_idx[dst] = b[p]
    if rating is not None:
        out_rt[dst] = lab[p]
    assert (out_idx >= 0).all()
    return new_ptr, out_idx, out_rt


class Data(object):
    """Minimal stand-in for ``torch_geometric.data.Data`` (reference util_functions.py:13,287)."""

    def __init__(self, x=None, edge_index=None, edge_type=None, y=None, **kw):
        self.x, self.edge_index, self.edge_type, self.y = x, edge_index, edge_type, y
        for k, v in kw.items():
            setattr(self, k, v)

    @property
    def num_nodes(self):
        return int(self.x.shape[0])

    @property
    def num_features(self):
        return int(self.x.shape[1])

    def keys(self):
        return [k for k, v in self.__dict__.items() if not k.startswith("_") and torch.is_tensor(v)]

    def to(self, device):
        for k in self.keys():
            setattr(self, k, getattr(self, k).to(device))
        return self


class Batch(Data):
    """A collated mini-batch (PyG ``Batch.from_data_list`` semantics, SURVEY.md A.3) plus the private
    device structures the fused kernels consume (graph offsets, labels, message-passing adjacency).

    Batches produced by ``SubgraphExtractor`` live in capacity-sized buffers; the public tensors
    (``x``, ``edge_index`` ...) are views cut to the true sizes, which costs one host sync the first
    time one of them is touched (the training loop never touches them).
    """

    def __init__(self, num_graphs, device, **kw):
        super().__init__(**kw)
        self.num_graphs = int(num_graphs)
        self.device = device
        self.batch = None
        self._priv = {}      # node_label, node_ptr, edge_ptr, node_cap, edge_cap, n_cap, symmetric ...
        self._adj = None
        self._lazy = None    # capacity buffers of an extracted batch
        self._err = None

    # ---- lazily cut public views of an extracted batch -------------------------------------------
    def _materialize(self):
        if self._lazy is None:
            return
        lz, self._lazy = self._lazy, None
        counts = lz["counts"].cpu()
        self.check()
        N, E = int(counts[0]), int(counts[1])
        self.__dict__["x"] = lz["x"][:N]
        self.__dict__["edge_index"] = lz["edge_index"][:, :E]
        self.__dict__["edge_type"] = lz["edge_type"][:E]
        self.__dict__["batch"] = lz["batch"][:N]
        self.__dict__["node_label"] = lz["node_label"][:N]
        self.__dict__["node_gid"] = lz["node_gid"][:N]

    def __getattribute__(self, name):
        if name in ("x", "edge_index", "edge_type", "batch", "node_label", "node_gid"):
            d = object.__getattribute__(self, "__dict__")
            if d.get("_lazy") is not None:
                object.__getattribute__(self, "_materialize")()
        return object.__getattribute__(self, name)

    def check(self):
        """raise if a kernel flagged a data-dependent error (host sync)."""
        if self._err is not None:
            _lib.check_kernel_error(int(self._err.item()))

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("igmc_b200 batches live on the GPU")
        return self

    # ---- foreign batches (PyG-collated tensors from anywhere) ------------------------------------
    @staticmethod
    def from_arrays(x, edge_index, edge_type, batch, y, num_graphs=None, device=None):
        """Wrap already-collated arrays (e.g. the oracle's) and derive graph offsets on the GPU.  Records the range of
        the edge types (``_priv["type_range"]``, None without edges), which the models compare with their relation
        count before they launch anything on the batch."""
        device = _require_cuda(device)
        lib = _lib.load()
        x = torch.as_tensor(x, dtype=torch.float32).to(device).contiguous()
        edge_index = torch.as_tensor(edge_index, dtype=torch.int64).to(device).contiguous()
        edge_type = torch.as_tensor(edge_type, dtype=torch.int64).to(device).contiguous()
        batch = torch.as_tensor(batch, dtype=torch.int64).to(device).contiguous()
        y = torch.as_tensor(y, dtype=torch.float32).to(device).contiguous().view(-1)
        B = int(num_graphs) if num_graphs is not None else int(y.numel())
        N, E = int(x.shape[0]), int(edge_index.shape[1])
        b = Batch(B, device, x=x, edge_index=edge_index, edge_type=edge_type, y=y)
        b.batch = batch
        lab = torch.argmax(x, 1).to(torch.uint8)
        node_ptr = torch.zeros(B + 1, dtype=torch.int32, device=device)
        edge_ptr = torch.zeros(B + 1, dtype=torch.int32, device=device)
        err = torch.zeros(1, dtype=torch.int32, device=device)
        src = edge_index[0] if E else torch.zeros(1, dtype=torch.int64, device=device)
        _lib.check(lib.igmc_batch_ptrs(batch.data_ptr() if N else None, src.data_ptr(), N, E, B,
                                       node_ptr.data_ptr(), edge_ptr.data_ptr(), err.data_ptr(), _stream_ptr()),
                   "igmc_batch_ptrs")
        # the largest graph and the edge-type range in one device-to-host copy
        zero = torch.zeros(1, dtype=torch.int64, device=device)
        stats = torch.cat([(node_ptr[1:] - node_ptr[:-1]).max().long().view(1) if B else zero,
                           edge_type.min().view(1) if E else zero, edge_type.max().view(1) if E else zero]).tolist()
        n_max = stats[0]
        b._err = err
        b._priv = dict(node_label=lab, node_ptr=node_ptr, edge_ptr=edge_ptr, node_cap=max(N, 1),
                       edge_cap=max(E, 1), n_cap=max(n_max, 2), symmetric=0, edge_row_stride=E,
                       type_range=(stats[1], stats[2]) if E else None)
        b.__dict__["node_label"] = lab
        b.check()
        return b

    @staticmethod
    def from_data_list(data_list, device=None):
        """PyG collate of ``Data`` objects (offset-concat edge_index, concat the rest)."""
        xs, eis, ets, ys, bs = [], [], [], [], []
        off = 0
        for gi, d in enumerate(data_list):
            n = int(d.x.shape[0])
            xs.append(d.x)
            eis.append(d.edge_index + off)
            ets.append(d.edge_type)
            ys.append(d.y.view(-1))
            bs.append(torch.full((n,), gi, dtype=torch.int64, device=d.x.device))
            off += n
        return Batch.from_arrays(torch.cat(xs, 0), torch.cat(eis, 1), torch.cat(ets), torch.cat(bs),
                                 torch.cat(ys), len(data_list), device)

    # ---- message-passing adjacency ------------------------------------------------------------------
    def adjacency(self):
        """(lazily) build the (type, neighbour)-sorted in/out edge lists with igmc_batch_prepare."""
        if self._adj is not None:
            return self._adj
        lib = _lib.load()
        p = self._priv
        dev = self.device
        ecap, ncap = p["edge_cap"], p["node_cap"]
        cache = getattr(self, "_adj_cache", None)
        if self._lazy is not None:
            ei, et = self._lazy["edge_index"], self._lazy["edge_type"]
        else:
            ei, et = self.edge_index, self.edge_type
        sym = int(p["symmetric"])
        if cache is not None and "t" in cache:
            t = cache["t"]
        else:
            t = dict(in_ptr=torch.zeros(ncap + 1, dtype=torch.int32, device=dev),
                     in_adj=torch.empty(ecap, dtype=torch.int32, device=dev),
                     in_eid=torch.empty(ecap, dtype=torch.int32, device=dev),
                     tmp=torch.empty(ecap, dtype=torch.int64, device=dev))
            if cache is not None:
                cache["t"] = t
        if not sym and "out_ptr" not in t:
            t.update(out_ptr=torch.zeros(ncap + 1, dtype=torch.int32, device=dev),
                     out_adj=torch.empty(ecap, dtype=torch.int32, device=dev),
                     out_eid=torch.empty(ecap, dtype=torch.int32, device=dev))
        c = _lib.Adj(t["in_ptr"].data_ptr(), t["in_adj"].data_ptr(), t["in_eid"].data_ptr(),
                     _lib.ptr(t.get("out_ptr")), _lib.ptr(t.get("out_adj")), _lib.ptr(t.get("out_eid")),
                     t["tmp"].data_ptr(), sym)
        _lib.check(lib.igmc_batch_prepare(ei.data_ptr(), p["edge_row_stride"], et.data_ptr(),
                                          p["node_ptr"].data_ptr(), p["edge_ptr"].data_ptr(), self.num_graphs,
                                          p["n_cap"], C.byref(c), self._err.data_ptr(), _stream_ptr()),
                   "igmc_batch_prepare")
        self._adj = (c, t)
        return self._adj


class _BatchWriter(object):
    """Output side of ``SubgraphExtractor`` and ``StaticStore``, so that the train engine treats both alike: the
    capacity-sized buffers a batch kernel writes (one cached set per (batch size, slot) with ``reuse``), the
    ``BatchOut`` struct that points at them and the ``Batch`` that wraps them.  A subclass sets ``device``,
    ``feat_dim``, ``emit_x``, ``cap``, ``err`` and ``_out_cache`` and defines ``_out_caps(B)``."""

    def _out_caps(self, B):
        """(node capacity, edge capacity, length of adj_tmp) of a batch of ``B`` subgraphs"""
        raise NotImplementedError

    def _alloc_out(self, B, reuse=False, slot=0):
        if reuse and (B, slot) in self._out_cache:
            return self._out_cache[(B, slot)]
        dev = self.device
        ncap, ecap, tmp = self._out_caps(B)
        o = dict(x=torch.empty(ncap, self.feat_dim, dtype=torch.float32, device=dev) if self.emit_x else None,
                 node_label=torch.empty(ncap, dtype=torch.uint8, device=dev),
                 batch=torch.empty(ncap, dtype=torch.int64, device=dev),
                 node_gid=torch.empty(ncap, dtype=torch.int32, device=dev),
                 edge_index=torch.empty(2, ecap, dtype=torch.int64, device=dev),
                 edge_type=torch.empty(ecap, dtype=torch.int64, device=dev),
                 y=torch.empty(B, dtype=torch.float32, device=dev),
                 node_ptr=torch.zeros(B + 1, dtype=torch.int32, device=dev),
                 edge_ptr=torch.zeros(B + 1, dtype=torch.int32, device=dev),
                 graph_nu=torch.zeros(B, dtype=torch.int32, device=dev),
                 counts=torch.zeros(2, dtype=torch.int32, device=dev),
                 adj_in_ptr=torch.zeros(ncap + 1, dtype=torch.int32, device=dev),
                 adj_in=torch.empty(ecap, dtype=torch.int32, device=dev),
                 adj_eid=torch.empty(ecap, dtype=torch.int32, device=dev),
                 adj_tmp=torch.empty(tmp, dtype=torch.int64, device=dev),
                 err=self.err)
        o["_caps"] = (ncap, ecap)
        o["_c"] = _lib.BatchOut(ncap, ecap, self.feat_dim, _lib.ptr(o["x"]), o["node_label"].data_ptr(),
                                o["batch"].data_ptr(), o["node_gid"].data_ptr(), o["edge_index"].data_ptr(),
                                o["edge_type"].data_ptr(), o["y"].data_ptr(), o["node_ptr"].data_ptr(),
                                o["edge_ptr"].data_ptr(), o["graph_nu"].data_ptr(), o["counts"].data_ptr(),
                                o["adj_in_ptr"].data_ptr(), o["adj_in"].data_ptr(), o["adj_eid"].data_ptr(),
                                o["adj_tmp"].data_ptr())
        if reuse:
            self._out_cache[(B, slot)] = o
        return o

    def _batch(self, B, o, keep):
        """the ``Batch`` of ``B`` subgraphs written into ``o``; ``keep``: inputs the launch reads, kept alive with it"""
        ncap, ecap = o["_caps"]
        b = Batch(B, self.device, y=o["y"])
        b._lazy = o
        b._err = o["err"]
        b._keep = keep
        b._priv = dict(node_label=o["node_label"], node_ptr=o["node_ptr"], edge_ptr=o["edge_ptr"],
                       node_cap=ncap, edge_cap=ecap, n_cap=2 * self.cap, symmetric=1, edge_row_stride=ecap,
                       graph_nu=o["graph_nu"], counts=o["counts"])
        # the batch kernel already built the (symmetric) message-passing adjacency in the same pass
        b._adj = (_lib.Adj(o["adj_in_ptr"].data_ptr(), o["adj_in"].data_ptr(), o["adj_eid"].data_ptr(), None, None,
                           None, o["adj_tmp"].data_ptr(), 1), o)
        return b


class SubgraphExtractor(_BatchWriter):
    """Owns the workspace for batches of up to ``max_batch`` pairs and runs igmc_extract_batch.

    One instance per dataset; ``extract(idx)`` is what the reference's DataLoader workers do with
    ``MyDynamicDataset.get`` + collate (train_eval.py:40-45), as two kernel launches.
    """

    def __init__(self, graph, links_u, links_v, labels, class_values, h=1, sample_ratio=1.0,
                 max_nodes_per_hop=None, max_batch=64, seed=0, emit_x=True, fast=True):
        if not 1 <= int(h) <= _lib.MAX_HOP:
            raise NotImplementedError("igmc_b200 extraction implements hop = 1..%d (Main.py:88 default 1)" % _lib.MAX_HOP)
        self.lib = _lib.load()
        self.graph = graph
        self.fast = bool(fast)    # h = 1: one-launch extraction (False forces the generic two-launch kernels)
        self.device = graph.device if graph.device is not None else _require_cuda()
        if graph.device is None:
            graph.to(self.device)
        dev = self.device
        self.h = int(h)
        self.sample_ratio = float(sample_ratio)
        self.mnph = -1 if max_nodes_per_hop is None else int(max_nodes_per_hop)
        self._mnph_arg = max_nodes_per_hop
        self.seed = int(seed)
        self.num_links = len(links_u)
        self.links_u = torch.as_tensor(np.asarray(links_u), dtype=torch.int32).to(dev)
        self.links_v = torch.as_tensor(np.asarray(links_v), dtype=torch.int32).to(dev)
        self.links_label = torch.as_tensor(np.asarray(labels), dtype=torch.int32).to(dev)
        self.class_values = torch.as_tensor(np.asarray(class_values, dtype=np.float32)).to(dev)
        self.session_row_deg = 0   # the longest rating-session row the extractor serves (0: none)
        self.cap = graph.node_cap(max_nodes_per_hop, self.h)
        self._graph_version = graph.version
        self.feat_dim = 2 * self.h + 2
        self.emit_x = emit_x
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)   # shared device error word
        self._out_cache = {}
        self.max_batch = 0
        self._reserve(max_batch)

    def _row_deg(self):
        """the longest user row a batch can read: the graph's, or a rating session's"""
        return max(self.graph.max_row_deg, self.session_row_deg)

    def _edges_per_graph(self):
        g = self.graph
        return 2 * min(self.cap * min(self.cap, max(self._row_deg(), 1)), max(g.nnz + self.session_row_deg, 1))

    def serve_sessions(self, row_deg):
        """size the capacities for target rows of up to ``row_deg`` ratings (a ``RatingSessions``' longest row; 0:
        the graph's rows only), re-reserving as after a graph update"""
        if int(row_deg) != self.session_row_deg:
            self.session_row_deg = int(row_deg)
            self._graph_version = None

    def _sync_graph(self):
        """after an update of the graph (or of the session rows served): re-derive ``cap`` and the edge capacity, and
        re-reserve the workspace if they grew beyond what it holds (a smaller cap uses the larger buffers as they
        are)"""
        g = self.graph
        if g.version == self._graph_version:
            return
        self._graph_version = g.version
        self.cap = g.node_cap(self._mnph_arg, self.h, self._row_deg())
        if self.cap > self._ws_cap or self._edges_per_graph() > self._ws_edges:
            self._reserve(self.max_batch, regrow=True)

    def _reserve(self, B, regrow=False):
        if B <= self.max_batch and not regrow:
            return
        B = max(B, self.max_batch)
        dev, cap = self.device, self.cap
        if self.max_batch:
            # captured CUDA graphs hold raw pointers into the workspace of the batch sizes seen so far: keep the old
            # buffers alive instead of handing them back to the allocator
            self.__dict__.setdefault("_retired_ws", []).append((self.ws, self._out_cache))
            self._out_cache = {}
        self.max_batch = B
        per_graph_edges = self._edges_per_graph()
        self._ws_cap, self._ws_edges = cap, per_graph_edges
        self.node_cap = B * 2 * cap
        self.edge_cap = max(B * per_graph_edges, 2)
        i32 = dict(dtype=torch.int32, device=dev)
        self.ws = dict(nodes_u=torch.empty(B * cap, **i32), nodes_v=torch.empty(B * cap, **i32),
                       n_u=torch.zeros(B, **i32), n_v=torch.zeros(B, **i32),
                       row_cnt=torch.empty(B * cap, **i32), m_cnt=torch.zeros(B, **i32),
                       col_cnt=torch.empty(B * cap, **i32),
                       hop_off=torch.zeros(B * 2 * (_lib.MAX_HOP + 1), **i32),
                       sync=torch.zeros(B + 1, **i32))
        ptrs = [self.ws[k].data_ptr() for k in ("nodes_u", "nodes_v", "n_u", "n_v", "row_cnt", "m_cnt", "col_cnt",
                                                "hop_off", "sync")]
        if not self.fast:
            ptrs[-1] = None      # no flags -> the generic two-launch path
        self._ws_c = _lib.ExtractWS(*ptrs)

    def _out_caps(self, B):
        ecap = max(B * (self.edge_cap // self.max_batch), 2)
        return B * 2 * self.cap, ecap, ecap

    def extract(self, idx=None, pairs=None, pair_ids=None, out=None, inject=None, seed=None, seed_dev=None,
                reuse=False, slot=0, sessions=None, sess=None):
        """Extract + collate.  ``idx``: int64 tensor/array of dataset indices (device tensor preferred),
        or ``pairs=(u, v, label)`` explicit arrays.  ``inject=(nodes_u, nodes_v, n_u, n_v)`` supplies the
        per-graph node lists ([B,cap] int32, target first) instead of sampling (parity tests).
        ``reuse=True`` writes into one cached buffer set per batch size (training loop / CUDA graphs:
        the previous batch of that size is overwritten).  ``seed_dev``: device uint64 overriding the seed.
        ``sessions`` (a ``RatingSessions``, with ``pairs``) and ``sess`` [B] (int32 device tensor): graph g takes its
        target user's row from session row sess[g] (igmc_extract_sessions; ``serve_sessions`` first).
        Returns a ``Batch`` whose public tensors are materialised lazily."""
        dev = self.device
        self._sync_graph()
        keep = []
        if pairs is not None:
            # (device tensors of the right type are used in place: the inference engine's candidate buffers, read by
            # a captured CUDA graph; a label array of None extracts with label 0)
            pu = _on_device(pairs[0], torch.int32, dev)
            pv = _on_device(pairs[1], torch.int32, dev)
            pl = None if pairs[2] is None else _on_device(pairs[2], torch.int32, dev)
            B = int(pu.numel())
            pid = None
            if pair_ids is not None:
                pid = _on_device(pair_ids, torch.int64, dev)
            P = _lib.Pairs(None, pu.data_ptr(), pv.data_ptr(), _lib.ptr(pl), _lib.ptr(pid))
            keep += [pu, pv, pl, pid]
        else:
            idx = _device_index(idx, dev)
            B = int(idx.numel())
            P = _lib.Pairs(idx.data_ptr(), self.links_u.data_ptr(), self.links_v.data_ptr(),
                           self.links_label.data_ptr(), None)
            keep += [idx]
        self._reserve(B)
        o = out if out is not None else self._alloc_out(B, reuse, slot)
        inj = [None] * 4
        if inject is not None:
            inj_t = [torch.as_tensor(np.asarray(a), dtype=torch.int32).to(dev).contiguous() for a in inject]
            assert inj_t[0].shape == (B, self.cap) and inj_t[1].shape == (B, self.cap)
            inj = [t.data_ptr() for t in inj_t]
            keep += inj_t
        if sessions is not None:
            if inject is not None or pairs is None or sess is None:
                raise ValueError("session extraction takes pairs= and sess=, and no injected node lists")
            if sessions.max_row_deg > self.session_row_deg:
                raise ValueError("the extractor is sized for session rows of up to %d ratings, not %d "
                                 "(serve_sessions)" % (self.session_row_deg, sessions.max_row_deg))
            sess = _on_device(sess, torch.int32, dev)
            keep += [sess, sessions]
        head = (C.byref(P), B, self.h, self.mnph, self.sample_ratio, self.seed if seed is None else int(seed),
                _lib.ptr(seed_dev), self.cap)
        tail = (C.byref(self._ws_c), self.class_values.data_ptr(), int(self.class_values.numel()),
                int(self._row_deg()), C.byref(o["_c"]), o["err"].data_ptr(), _stream_ptr())
        if sessions is not None:
            _lib.check(self.lib.igmc_extract_sessions(C.byref(self.graph._c), C.byref(sessions._c), sess.data_ptr(),
                                                      *head, *tail), "igmc_extract_sessions")
        else:
            _lib.check(self.lib.igmc_extract_batch(C.byref(self.graph._c), *head, *inj, *tail), "igmc_extract_batch")
        return self._batch(B, o, keep)

    def plan(self, B):
        """the path ``extract`` takes for a batch of ``B`` pairs (igmc_extract_plan on this extractor's graph, cap,
        rating classes, longest row and edge capacity): the dynamic shared memory of the one-launch h = 1 kernel, 0
        for the generic kernels, < 0 when neither fits.  Sizes the workspace for ``B`` pairs as ``extract`` does."""
        self._sync_graph()
        self._reserve(B)
        g = self.graph
        return int(self.lib.igmc_extract_plan(g.num_users, g.num_items, int(B), self.h, self.cap,
                                              int(self.class_values.numel()), int(self._row_deg()),
                                              self._out_caps(B)[1], int(self.fast), 1))

    def node_lists(self, B):
        """(nodes_u [B,cap], nodes_v [B,cap], n_u [B], n_v [B]) of the last extract (host copies)."""
        cap = self.cap
        return (self.ws["nodes_u"][:B * cap].view(B, cap).cpu().numpy(),
                self.ws["nodes_v"][:B * cap].view(B, cap).cpu().numpy(),
                self.ws["n_u"][:B].cpu().numpy(), self.ws["n_v"][:B].cpu().numpy())


class MyDynamicDataset(object):
    """Reference signature (util_functions.py:114-115).  ``get(idx)`` extracts one enclosing subgraph on
    the GPU; the train loop uses ``extract_batch(indices)`` to get a whole collated mini-batch."""

    def __init__(self, root, A, links, labels, h, sample_ratio, max_nodes_per_hop, u_features, v_features,
                 class_values, max_num=None, seed=0):
        if u_features is not None or v_features is not None:
            raise NotImplementedError("side features (--use-features) are outside the hot path (SURVEY.md §2)")
        self.root = root
        self.links = (np.asarray(links[0]), np.asarray(links[1]))
        self.labels = np.asarray(labels)
        self.h, self.sample_ratio, self.max_nodes_per_hop = int(h), sample_ratio, max_nodes_per_hop
        self.class_values = np.asarray(class_values)
        if max_num is not None:  # reference :127-133
            np.random.seed(123)
            perm = np.random.permutation(len(self.links[0]))[:max_num]
            self.links = (self.links[0][perm], self.links[1][perm])
            self.labels = self.labels[perm]
        self.graph = A if isinstance(A, RatingGraph) else RatingGraph(A)
        self.extractor = SubgraphExtractor(self.graph, self.links[0], self.links[1], self.labels,
                                           self.class_values, self.h, sample_ratio, max_nodes_per_hop,
                                           seed=seed)

    def __len__(self):
        return len(self.links[0])

    @property
    def num_features(self):
        return 2 * self.h + 2

    def extract_batch(self, indices):
        return self.extractor.extract(idx=indices)

    def get(self, idx):
        b = self.extractor.extract(idx=np.asarray([self._index(idx)], dtype=np.int64))
        return Data(b.x, b.edge_index, edge_type=b.edge_type, y=b.y)

    def _index(self, idx):
        """PyG ``Dataset.__getitem__`` semantics for an int: negative indices count from the end, anything outside
        raises IndexError - which is what ends the reference's ``for g in dataset`` loops (models.py:71)."""
        idx = int(idx)
        n = len(self)
        if idx < -n or idx >= n:
            raise IndexError("index %d out of range for a dataset of %d subgraphs" % (idx, n))
        return idx + n if idx < 0 else idx

    def __getitem__(self, idx):
        return self.get(idx)

    def __iter__(self):
        for k in range(len(self)):
            yield self.get(k)

    def pair_cost(self):
        """a-priori size estimate of every pair's subgraph from the matrix degrees alone (hop 1: raters of the item
        + items of the user, each capped by max_nodes_per_hop): what the data-parallel sharding balances the ranks'
        batches by (train_eval.deal_balanced).  Host arrays, computed once per version of the graph."""
        c = getattr(self, "_pair_cost", None)
        if c is None or self._pair_cost_version != self.graph.version:
            self._pair_cost_version = self.graph.version
            h = self.graph.host
            du, dv = np.diff(h["row_ptr"]), np.diff(h["col_ptr"])
            cap = self.max_nodes_per_hop if self.max_nodes_per_hop is not None else (1 << 30)
            c = np.minimum(du[self.links[0]], cap) + np.minimum(dv[self.links[1]], cap)
            self._pair_cost = c = c.astype(np.float64)
        return c

    def node_counts(self, chunk=2048):
        """number of nodes of every subgraph (what ``[g.num_nodes for g in dataset]`` gives, models.py:71), extracted
        in large batches instead of one by one"""
        out = []
        for s0 in range(0, len(self), chunk):
            idx = np.arange(s0, min(s0 + chunk, len(self)), dtype=np.int64)
            b = self.extract_batch(idx)
            b.check()
            out.append(np.diff(b._priv["node_ptr"][:len(idx) + 1].cpu().numpy()))
        return np.concatenate(out) if out else np.zeros(0, np.int64)


class StaticStore(_BatchWriter):
    """Device-resident store of pre-extracted subgraphs + batch assembly (igmc_assemble_batch).  Has the
    ``extract`` / ``err`` / ``cap`` surface of ``SubgraphExtractor`` so that the train engine treats both alike."""

    def __init__(self, extractor, num_graphs, chunk=512):
        self.lib = _lib.load()
        self.device = dev = extractor.device
        self.feat_dim, self.emit_x = extractor.feat_dim, extractor.emit_x
        parts = {k: [] for k in ("node_label", "node_gid", "edge_src", "edge_dst", "edge_type", "y", "graph_nu",
                                 "adj_ptr", "adj_in", "adj_eid", "ncnt", "ecnt")}
        for s0 in range(0, num_graphs, chunk):
            idx = np.arange(s0, min(s0 + chunk, num_graphs), dtype=np.int64)
            b = extractor.extract(idx=idx)
            b.check()
            nptr, eptr = b._priv["node_ptr"].long(), b._priv["edge_ptr"].long()
            N, E = int(nptr[-1]), int(eptr[-1])
            gi_n = b.batch[:N]
            ei = b.edge_index
            gi_e = gi_n[ei[0]] if E else torch.zeros(0, dtype=torch.int64, device=dev)
            adj = b._adj[1]
            parts["node_label"].append(b.node_label[:N].clone())
            parts["node_gid"].append(b.node_gid[:N].clone())
            parts["edge_src"].append((ei[0] - nptr[gi_e]).int())
            parts["edge_dst"].append((ei[1] - nptr[gi_e]).int())
            parts["edge_type"].append(b.edge_type[:E].to(torch.uint8))
            parts["y"].append(b.y.clone())
            parts["graph_nu"].append(b._priv["graph_nu"][:len(idx)].clone())
            # adjacency: list offsets / edge ids relative to the graph; positions coincide with the edge slots
            ap = adj["adj_in_ptr"][:N + 1].long()
            loc = ap[:N] - eptr[gi_n]
            ends = (eptr[1:] - eptr[:-1])                      # per graph: last offset = its edge count
            # interleave: for graph g its n offsets followed by its total
            cnt_n = (nptr[1:] - nptr[:-1])
            out = torch.empty(N + len(idx), dtype=torch.int32, device=dev)
            pos = torch.arange(N, device=dev) + gi_n              # node t of graph g sits at t + g
            out[pos] = loc.int()
            out[nptr[1:] + torch.arange(len(idx), device=dev)] = ends.int()
            parts["adj_ptr"].append(out)
            parts["adj_in"].append(adj["adj_in"][:E].clone())
            parts["adj_eid"].append((adj["adj_eid"][:E].long() - eptr[gi_e]).int())   # list slot e belongs to graph gi_e
            parts["ncnt"].append(cnt_n)
            parts["ecnt"].append(ends)
        cat = {k: torch.cat(v) for k, v in parts.items()}
        self._finish(cat, num_graphs)

    @classmethod
    def from_arrays(cls, device, feat_dim, x, edge_index, edge_type, y, node_off, edge_off, emit_x=True):
        """Build the store from collated per-graph-LOCAL arrays (the content of the reference's ``data.pt``,
        pyg_cache.load_processed) instead of extracting: labels from the one-hot ``x``, message-passing lists by one
        device-wide sort of the edges by (destination node, rating, source).  The edge layout must be the reference's
        ``[u | v ; v | u]`` per graph (construct_pyg_graph, util_functions.py:283-285): the kernels find an edge's
        reverse at +-half the graph's edge count."""
        self = cls.__new__(cls)
        self.lib = _lib.load()
        self.device = dev = torch.device(device)
        self.feat_dim, self.emit_x = int(feat_dim), emit_x
        x, y = x.to(dev), y.to(dev).float().view(-1)
        ei, et = edge_index.to(dev).long(), edge_type.to(dev).long()
        noff, eoff = node_off.to(dev).long(), edge_off.to(dev).long()
        G = int(y.numel())
        if et.numel() and (int(et.min()) < 0 or int(et.max()) > 255):
            raise ValueError("edge types must lie in 0..255 (the stored type is one byte), got %d..%d"
                             % (int(et.min()), int(et.max())))
        if int(x.shape[1]) != self.feat_dim:
            raise ValueError("cached node features have width %d, expected %d (hop mismatch)" % (x.shape[1], feat_dim))
        ncnt, ecnt = noff[1:] - noff[:-1], eoff[1:] - eoff[:-1]
        E, N = int(eoff[-1]), int(noff[-1])
        ge = torch.repeat_interleave(torch.arange(G, device=dev), ecnt)          # graph of every edge
        gn = torch.repeat_interleave(torch.arange(G, device=dev), ncnt)
        if E:
            half = (ecnt // 2)[ge]
            k = torch.arange(E, device=dev) - eoff[ge]
            mirror = torch.where(k < half, torch.arange(E, device=dev) + half, torch.arange(E, device=dev) - half)
            if bool((ecnt % 2 != 0).any()) or not torch.equal(ei[0], ei[1][mirror]) or not torch.equal(et, et[mirror]) \
                    or int(ei.max()) >= int(ncnt.max()) or bool((ei >= ncnt[ge].unsqueeze(0)).any()):
                raise ValueError("the cache is not in the reference's [u|v ; v|u] per-graph edge layout")
        label = torch.argmax(x, 1)
        gnu = torch.zeros(G, dtype=torch.int64, device=dev).index_add_(0, gn, (label % 2 == 0).long())
        # in-lists: edges sorted by (global destination node, rating, local source); graphs stay contiguous
        gdst = noff[ge] + ei[1]
        key = (gdst * 256 + et) * 65536 + ei[0]
        order = torch.argsort(key)
        deg = torch.zeros(N, dtype=torch.int64, device=dev).index_add_(0, gdst, torch.ones(E, dtype=torch.int64, device=dev))
        start = torch.cumsum(deg, 0) - deg                                         # first list slot of every node
        adj_ptr = torch.empty(N + G, dtype=torch.int32, device=dev)
        adj_ptr[torch.arange(N, device=dev) + gn] = (start - eoff[gn]).int()
        adj_ptr[noff[1:] + torch.arange(G, device=dev)] = ecnt.int()
        cat = dict(node_label=label.to(torch.uint8), node_gid=torch.zeros(N, dtype=torch.int32, device=dev),
                   edge_src=ei[0].int(), edge_dst=ei[1].int(), edge_type=et.to(torch.uint8), y=y, graph_nu=gnu.int(),
                   adj_ptr=adj_ptr, adj_in=(ei[0][order] | (et[order] << 16)).int(),
                   adj_eid=(order - eoff[ge[order]]).int(), ncnt=ncnt, ecnt=ecnt)
        self._finish(cat, G)
        return self

    def arrays(self):
        """collated per-graph-local arrays of the store: (x one-hot, edge_index, edge_type, y, node_off, edge_off)"""
        lab = self.t["node_label"].long()
        n = int(self.node_off[-1])
        x = torch.zeros(n, self.feat_dim, dtype=torch.float32, device=self.device)
        if n:
            x[torch.arange(n, device=self.device), lab[:n]] = 1.0
        e = int(self.edge_off[-1])
        ei = torch.stack([self.t["edge_src"][:e].long(), self.t["edge_dst"][:e].long()])
        return x, ei, self.t["edge_type"][:e].long(), self.t["y"][:self.num_graphs], self.node_off.long(), \
            self.edge_off.long()

    def _finish(self, cat, num_graphs):
        dev = self.device
        z = torch.zeros(1, dtype=torch.int64, device=dev)
        self.node_off = torch.cat([z, torch.cumsum(cat["ncnt"], 0)]).int()
        self.edge_off = torch.cat([z, torch.cumsum(cat["ecnt"], 0)]).int()
        self.t = {k: cat[k] for k in ("node_label", "node_gid", "edge_src", "edge_dst", "edge_type", "y", "graph_nu",
                                       "adj_ptr", "adj_in", "adj_eid")}
        for k, v in self.t.items():   # valid pointers even for empty stores
            if v.numel() == 0:
                self.t[k] = torch.zeros(1, dtype=v.dtype, device=dev)
        self.num_graphs = num_graphs
        self.max_n = int(cat["ncnt"].max()) if num_graphs else 2
        self.max_e = int(cat["ecnt"].max()) if num_graphs else 2
        et = cat["edge_type"]
        # every batch assembled from the store carries the store's edge-type range: the models compare it with their
        # relation count before they launch (Batch.from_arrays records the same for foreign batches)
        self.type_range = tuple(torch.stack([et.min(), et.max()]).long().tolist()) if et.numel() else None
        self.cap = (self.max_n + 1) // 2 + 1          # n_cap = 2*cap >= max_n (the model plans by 2*cap)
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)
        self._c = _lib.Store(self.node_off.data_ptr(), self.edge_off.data_ptr(),
                             *[self.t[k].data_ptr() for k in ("node_label", "node_gid", "edge_src", "edge_dst",
                                                              "edge_type", "y", "graph_nu", "adj_ptr", "adj_in",
                                                              "adj_eid")])
        self._out_cache = {}

    def _out_caps(self, B):
        return max(B * self.max_n, 2), max(B * self.max_e, 2), 1

    def extract(self, idx=None, seed_dev=None, reuse=False, slot=0, **unused):
        idx = _device_index(idx, self.device)
        B = int(idx.numel())
        o = self._alloc_out(B, reuse, slot)
        _lib.check(self.lib.igmc_assemble_batch(C.byref(self._c), idx.data_ptr(), B, C.byref(o["_c"]),
                                                self.err.data_ptr(), _stream_ptr()), "igmc_assemble_batch")
        b = self._batch(B, o, [idx])
        b._priv["type_range"] = self.type_range
        return b


class MyDataset(MyDynamicDataset):
    """Static variant (reference util_functions.py:69-110): every subgraph is extracted ONCE (in large GPU batches
    instead of an mp.Pool) and kept device-resident in the reference's ``(data, slices)`` spirit — per-graph LOCAL
    node ids + per-graph boundaries (SURVEY.md A.5b), in compact types, with the message-passing adjacency;
    mini-batches are assembled from it by one kernel (igmc_assemble_batch)."""

    def __init__(self, root, A, links, labels, h, sample_ratio, max_nodes_per_hop, u_features, v_features,
                 class_values, max_num=None, parallel=True, seed=0, chunk=512):
        super().__init__(root, A, links, labels, h, sample_ratio, max_nodes_per_hop, u_features, v_features,
                         class_values, max_num, seed)
        self.parallel = parallel
        self.max_num = max_num
        self.dynamic_extractor = self.extractor
        # the reference's cache contract (util_functions.py:91-99,108-109): <root>/processed/data.pt (data_<max_num>.pt)
        # holding (data, slices) is used when present, written otherwise - files interchange with the reference's
        from . import pyg_cache
        path = pyg_cache.processed_path(root, max_num) if root else None
        if path is not None and os.path.isfile(path):
            c = pyg_cache.load_processed(path)
            if int(c["y"].numel()) != len(self):
                raise ValueError("%s holds %d subgraphs, the dataset has %d pairs (stale cache: delete it or pass "
                                 "--reprocess)" % (path, int(c["y"].numel()), len(self)))
            self.store = StaticStore.from_arrays(self.dynamic_extractor.device, self.num_features, c["x"],
                                                 c["edge_index"], c["edge_type"], c["y"], c["node_off"], c["edge_off"])
            self.extractor = self.store
            self.loaded_from = path
        else:
            self.process(chunk)
            self.loaded_from = None
            if path is not None:
                pyg_cache.save_processed(path, *self.store.arrays())

    @property
    def processed_file_names(self):
        return ["data.pt"] if self.max_num is None else ["data_{}.pt".format(self.max_num)]

    def process(self, chunk=512):
        self.store = StaticStore(self.dynamic_extractor, len(self), chunk)
        self.extractor = self.store          # the train / eval loops batch through the store from now on

    def extract_batch(self, indices):
        return self.store.extract(idx=indices)

    def get(self, idx):
        b = self.store.extract(idx=np.asarray([self._index(idx)], dtype=np.int64))
        return Data(b.x, b.edge_index, edge_type=b.edge_type, y=b.y)

    def node_counts(self, chunk=2048):
        return np.diff(self.store.node_off.cpu().numpy()).astype(np.int64)
