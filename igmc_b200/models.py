"""Drop-in for the reference's ``models.IGMC`` (models.py:170-217) on the fused sm_90a (H100) kernels.

``IGMC(dataset, gconv, latent_dim, num_relations, num_bases, regression, adj_dropout, ...)`` keeps the
reference constructor, ``forward(data) -> Tensor[B]``, ``reset_parameters()``, the attribute surface
``convs[l].{att, basis, root, bias, num_bases, num_relations, in_channels, out_channels}``, ``lin1``,
``lin2`` and therefore the reference's ``state_dict`` keys, so its checkpoints load.  ``rgcn="pyg-2"`` swaps in the
RGCNConv of PyG >= 1.6 (``convs[l].{comp, weight, root, bias}``, one mean per relation) on the same kernels.

All parameters are views into ONE flat fp32 buffer (``flat_params``), gradients into ``flat_grad``:
that buffer is what the kernels read, what the single NCCL all-reduce per step moves and what the fused
Adam updates.  ``forward`` is autograd-capable (custom Function over the C-ABI); the training loop in
``train_eval`` uses ``fused_step`` which skips autograd altogether.
"""
import ctypes as C
import math
import os

import torch
import torch.nn as nn

from . import _lib
from .util_functions import Batch, _stream_ptr

HID = _lib.HIDDEN
SMEM_LIMIT = 227 * 1024


def _align4(x):
    return (x + 3) & ~3


def splitmix64(x):
    M = (1 << 64) - 1
    x = (x + 0x9E3779B97F4A7C15) & M
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M
    return x ^ (x >> 31)


def _keep_threshold(p):
    """Host twin of ``keep_thresh`` in csrc/lists.cuh and ``edge_keep``'s reading of it: a draw keeps its unit iff its
    high 32 bits >= the returned p * 2^32, which is 2^32 (nothing kept) for p >= 1."""
    import numpy as np
    t = float(np.float32(p)) * 4294967296.0   # the kernel sees p as fp32
    return 1 << 32 if t >= 4294967295.0 else int(t)


def edge_keep_reference(seed, num_edges, p):
    """Host twin of ``edge_keep`` in csrc/common.cuh: bool keep mask for directed edges 0..E-1."""
    thresh = _keep_threshold(p)
    return torch.tensor([(splitmix64((seed + e) & ((1 << 64) - 1)) >> 32) >= thresh for e in range(num_edges)],
                        dtype=torch.bool)   # (a batch without edges still gets a bool mask)


def hidden_keep_reference(seed, num_graphs, p):
    """Host twin of the hidden dropout before ``lin2`` (the kernels' own draw when no ``hidden_keep`` is injected):
    bool keep mask [num_graphs, 128]; unit ``o`` of graph ``g`` is an ``edge_keep`` draw of index ``g*128 + o`` on the
    seed ``seed ^ 0x5bd1e995a5a5a5a5``.  Kept units are scaled by 1 / (1 - p)."""
    M = (1 << 64) - 1
    thresh = _keep_threshold(p)
    s = (seed ^ 0x5bd1e995a5a5a5a5) & M
    keep = [(splitmix64((s + i) & M) >> 32) >= thresh for i in range(num_graphs * 128)]
    return torch.tensor(keep, dtype=torch.bool).view(num_graphs, 128)


def l2_cluster(n_cap, B, sms):
    """CTAs per subgraph of the L2 plan (csrc/rgcn_l2.cu).  A CTA owns a contiguous range of destination nodes and
    works through it in 64-node tiles; the cluster shares one subgraph's layers through L2 with one cluster barrier
    per layer.  Rule: the most CTAs (8, 4, 2, 1) that keep the grid within four CTAs per SM and still give every CTA
    at least one tile of the largest subgraph.  Measured at batch 50 only, on an H100 80GB HBM3 (700 W), train step
    subgraphs/s with 1 / 2 / 4 / 8 CTAs (scripts/large_subgraph_rate.py): ml_100k* h = 1 without a node cap (n_cap
    1236) 3.3 k / 5.6 k / 8.3 k / 13.1 k; h = 2 at mnph 200 (n_cap 802) 3.2 k / 5.9 k / 8.1 k / 10.2 k; R = 71 at n_cap
    564: 5.3 k / 9.9 k / 17.6 k / 17.5 k.  More CTAs per subgraph never lost, even past one wave (400 CTAs on 132
    SMs).  The four-per-SM bound (other batch sizes) and the one-tile bound (smaller n_cap) are unmeasured choices."""
    for c in (8, 4, 2):
        if B * c <= 4 * sms and n_cap >= 64 * c:
            return c
    return 1


def select_plan(cmodel, n_cap, B, sms, want="auto", max_edges=None):
    """kernel plan of ``cmodel`` for batches of ``B`` subgraphs of up to ``n_cap`` nodes on a device with ``sms`` SMs
    (host only: plan queries through igmc_model_plan).  ``want`` forces one plan value; ``max_edges`` (longest
    per-subgraph directed edge list seen) sizes the list buffers of the relation-space plans through
    ``cmodel.list_hint``.  Raises RuntimeError when no plan accepts the shape."""
    lib = _lib.load()
    R = cmodel.num_relations
    if want != "auto":
        cands = [int(want)]
    elif n_cap > 256 and R <= 12:
        # large subgraphs (ml_100k*: up to 402 nodes): four CTAs per subgraph even when that is more than one wave
        # of the SMs - node features of the whole subgraph take 100 KB of every CTA's shared memory, and only with
        # a quarter of the nodes per CTA do the edge lists still fit next to them.
        cands = [4, 3, 2, 1, 0]
    else:
        cands = [cl for cl in (4, 2, 1) if B * cl <= sms or cl == 1] + [0]
    if want == "auto":
        # node features in L2 instead of shared memory: subgraphs too large for every plan above
        cands.append(_lib.plan_l2(l2_cluster(n_cap, B, sms)))
    for cl in cands:
        if max_edges and _lib.is_rs(cl):
            cmodel.list_hint = int(1.25 * max_edges / int(cl)) + 256
        f = lib.igmc_model_plan(C.byref(cmodel), n_cap, int(cl), 0)
        b = lib.igmc_model_plan(C.byref(cmodel), n_cap, int(cl), 1)
        if f > 0 and b > 0:
            return int(cl)
    raise RuntimeError("igmc_b200: no kernel plan fits subgraphs of up to %d nodes with %d relations (the L2 plan "
                       "takes up to %d nodes per subgraph); lower --max-nodes-per-hop"
                       % (n_cap, R, _lib.L2_MAX_NODES))


class _RGCNParams(nn.Module):
    """Sizes, parameters and ``repr`` of an RGCNConv parameter holder.  The arithmetic lives in the fused kernels of
    the owning ``IGMC``.  ``NAMES``: the subclass's names of its [NB,in,out], [R,NB], [in,out] and [out] parameters, in
    the order they are registered (the order of ``parameters()``, which optimizer state_dicts are indexed by)."""

    NAMES = ()

    def __init__(self, in_channels, out_channels, num_relations, num_bases):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.num_relations, self.num_bases = num_relations, num_bases
        shapes = ((num_bases, in_channels, out_channels), (num_relations, num_bases), (in_channels, out_channels),
                  (out_channels,))
        for name, shape in zip(self.NAMES, shapes):
            setattr(self, name, nn.Parameter(torch.empty(*shape)))
        self.reset_parameters()

    def att_basis(self):
        """(coefficients [R,NB], bases [NB,in,out]) of W_r = sum_b att[r,b] basis[b]"""
        return getattr(self, self.NAMES[1]), getattr(self, self.NAMES[0])

    def __repr__(self):
        return "RGCNConv(%d, %d, num_relations=%d, num_bases=%d)" % (
            self.in_channels, self.out_channels, self.num_relations, self.num_bases)


class RGCNConv(_RGCNParams):
    """Parameter holder with PyG 1.4.2 ``RGCNConv`` names/shapes/init (SURVEY.md A.1)."""

    NAMES = ("basis", "att", "root", "bias")

    def reset_parameters(self):
        bound = 1.0 / math.sqrt(self.num_bases * self.in_channels)   # PyG inits.uniform(size, tensor)
        with torch.no_grad():
            for p in (self.basis, self.att, self.root, self.bias):
                p.uniform_(-bound, bound)


class RGCNConv2(_RGCNParams):
    """Parameter holder with the names/shapes/init of PyG >= 1.6 ``RGCNConv(in, out, num_relations, num_bases)``:
    ``weight [NB,in,out]``, ``comp [R,NB]``, ``root [in,out]``, ``bias [out]``; glorot(weight, comp, root), zeros(bias)
    (PyG 2.x ``reset_parameters``).  W_r = sum_b comp[r,b] weight[b] - the 1.4.2 layer's ``att @ basis`` - but the
    aggregation is a mean PER RELATION (``IGMC(..., rgcn="pyg-2")``; DESIGN.md §2)."""

    NAMES = ("weight", "comp", "root", "bias")

    def reset_parameters(self):
        with torch.no_grad():
            for p in (self.weight, self.comp, self.root):   # PyG inits.glorot: U(+-sqrt(6 / (size(-2) + size(-1))))
                bound = math.sqrt(6.0 / (p.size(-2) + p.size(-1)))
                p.uniform_(-bound, bound)
            self.bias.zero_()


# rgcn= keyword of IGMC / DGCNN_RS: which RGCNConv the model is (names, init and aggregation go together)
RGCN_LAYERS = {"pyg-1.4": RGCNConv, "pyg-2": RGCNConv2}


def _rgcn_layer(rgcn):
    if not isinstance(rgcn, str) or rgcn not in RGCN_LAYERS:
        raise ValueError("rgcn must be one of %s, not %r" % (sorted(RGCN_LAYERS), rgcn))
    return RGCN_LAYERS[rgcn]


class _IGMCFunction(torch.autograd.Function):
    """autograd bridge: forward/backward kernels behind ``IGMC.forward``."""

    @staticmethod
    def forward(ctx, model, batch, training, drop, *params):
        out, saved = model._launch_forward(batch, training, drop, y=None)
        ctx.model, ctx.batch, ctx.saved, ctx.drop = model, batch, saved, drop
        return out.clone()

    @staticmethod
    def backward(ctx, grad_out):
        model = ctx.model
        if not ctx.saved["train"]:
            raise RuntimeError("igmc_b200: backward through an eval-mode forward (zsave not kept); "
                               "call model.train() or use torch.no_grad()")
        model._launch_backward(ctx.batch, ctx.drop, ctx.saved,
                               (grad_out.float() * float(model.multiply_by)).contiguous())
        model._launch_grad_reduce(ctx.batch, ctx.saved, loss_scale=0.0, arr=0.0, with_loss=False)
        grads = [model._pview(model.flat_grad, e).clone() for e in model._layout]
        return (None, None, None, None) + tuple(grads)


class IGMC(nn.Module):
    REGRESSION_ONLY = "igmc_b200.IGMC implements the regression head Main.py uses (Main.py:396)"

    def __init__(self, dataset, gconv=RGCNConv, latent_dim=[32, 32, 32, 32], num_relations=5, num_bases=2,
                 regression=False, adj_dropout=0.2, force_undirected=False, side_features=False,
                 n_side_features=0, multiply_by=1, rgcn="pyg-1.4"):
        super().__init__()
        self._init_convs(dataset, latent_dim, num_relations, num_bases, regression, adj_dropout, force_undirected,
                         side_features, multiply_by, rgcn)
        self.lin1 = nn.Linear(2 * sum(latent_dim), 128)
        self.lin2 = nn.Linear(128, 1)
        self._init_bucket()

    @staticmethod
    def _check_latent_dim(latent_dim):
        if any(int(d) != HID for d in latent_dim) or not (1 <= len(latent_dim) <= _lib.MAX_LAYERS):
            raise NotImplementedError("latent_dim entries must be 32 (Main.py:391 hard-codes [32,32,32,32])")

    def _init_convs(self, dataset, latent_dim, num_relations, num_bases, regression, adj_dropout, force_undirected,
                    side_features, multiply_by, rgcn):
        """the constructor part IGMC and DGCNN_RS share: argument checks, node feature width and the conv stack"""
        conv_cls = _rgcn_layer(rgcn)
        self.rgcn = rgcn
        if not regression:
            raise NotImplementedError(self.REGRESSION_ONLY)
        if force_undirected:
            raise NotImplementedError("force_undirected edge dropout is not on the hot path")
        if side_features:
            raise NotImplementedError("side features are outside the hot path (SURVEY.md §2)")
        self._check_latent_dim(latent_dim)
        if num_bases not in (2, 4):
            raise NotImplementedError("num_bases must be 2 or 4")
        self.regression, self.adj_dropout, self.force_undirected = regression, adj_dropout, force_undirected
        self.side_features, self.multiply_by = side_features, multiply_by
        num_features = dataset if isinstance(dataset, int) else dataset.num_features
        self.num_features = int(num_features)
        if self.num_features > HID:
            raise NotImplementedError("node feature width > 32")
        self.num_relations, self.num_bases = int(num_relations), int(num_bases)
        dims = [self.num_features] + [int(d) for d in latent_dim]
        self.convs = nn.ModuleList([conv_cls(dims[l], dims[l + 1], num_relations, num_bases)
                                    for l in range(len(latent_dim))])

    def _init_bucket(self):
        self.drop_seed = 0x1234ABCD
        self._step = 0
        self._flatten()

    def _readout(self):
        """(bucket name prefix, module) of the layers after the convs, in bucket order"""
        return (("lin1", self.lin1), ("lin2", self.lin2))

    # ---- flat parameter bucket ---------------------------------------------------------------------
    def _named_order(self):
        for l, c in enumerate(self.convs):
            att, basis = c.att_basis()    # (comp, weight) of a PyG >= 1.6 layer: the same slots of the bucket
            yield ("att", l, att)
            yield ("basis", l, basis)
            yield ("root", l, c.root)
            yield ("bias", l, c.bias)
        for name, mod in self._readout():
            yield (name + "_w", 0, mod.weight)
            yield (name + "_b", 0, mod.bias)

    def _slot(self, kind, l, p):
        """(floats reserved in the bucket, padded shape or None) of one parameter."""
        return p.numel(), None

    @staticmethod
    def _pview(buf, e):
        """view of layout entry ``e`` = (offset, slot size, shape[, padded shape]) inside a flat buffer."""
        o, n, s = e[:3]
        if len(e) == 3:
            return buf[o:o + n].view(s)
        return buf[o:o + n].view(e[3])[..., :s[-1]]   # padded along the last (output channel) dimension

    def _flatten(self):
        """(re)create flat_params / flat_grad on the parameters' device and alias every parameter."""
        items = list(self._named_order())
        dev = items[0][2].device
        off, layout, m, offs = 0, [], _lib.Model(), {}
        m.num_layers, m.num_relations, m.num_bases, m.in_dim0 = len(self.convs), self.num_relations, \
            self.num_bases, self.num_features
        m.conv_param_count = -1
        for kind, l, p in items:
            n, pad = self._slot(kind, l, p)
            layout.append((off, n, tuple(p.shape)) if pad is None else (off, n, tuple(p.shape), tuple(pad)))
            if kind == "att":
                m.off_att[l] = off
            elif kind == "basis":
                m.off_basis[l] = off
            elif kind == "root":
                m.off_root[l] = off
            elif kind == "bias":
                m.off_bias[l] = off
            else:
                if m.conv_param_count < 0:
                    m.conv_param_count = off
                offs[kind] = off
                if hasattr(m, "off_" + kind):
                    setattr(m, "off_" + kind, off)
            off = _align4(off + n)
        m.param_count = off
        m.multiply_by = float(self.multiply_by)
        flat = torch.zeros(off, dtype=torch.float32, device=dev)
        grad = torch.zeros(off, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for e, (_, _, p) in zip(layout, items):
                v = self._pview(flat, e)
                v.copy_(p.data.float())
                p.data = v
                p.grad = None
        self.flat_params, self.flat_grad = flat, grad
        self._layout, self._cmodel, self._offs = layout, m, offs
        self._prepped = False
        self._ws = {}
        self._plans = {}
        self._wprep = None
        self._update_grid_fits = None

    def alias_grads(self):
        """point every ``p.grad`` at its slice of ``flat_grad`` (for stock torch optimizers)."""
        for e, (_, _, p) in zip(self._layout, self._named_order()):
            p.grad = self._pview(self.flat_grad, e)

    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        self._flatten()
        return out

    def load_state_dict(self, state_dict, *a, **kw):
        # the two RGCNConv layers compute different functions of equally shaped parameters: refuse the other layer's
        # checkpoint by its key names even when strict=False would load the rest of it
        own, other = (("att", "basis"), ("comp", "weight")) if self.rgcn == "pyg-1.4" else \
            (("comp", "weight"), ("att", "basis"))
        foreign = [k for k in state_dict if k.startswith("convs.") and k.rsplit(".", 1)[-1] in other]
        if foreign:
            raise RuntimeError("igmc_b200: %s belongs to the other RGCNConv layer (this model has rgcn=%r: convs.*.%s / "
                               "convs.*.%s); build the model with the matching rgcn= keyword" % ((foreign[0], self.rgcn) + own))
        self._prepped = False         # prepared weights (igmc_prep_weights) belong to the old parameters
        return super().load_state_dict(state_dict, *a, **kw)

    def reset_parameters(self):
        for c in self.convs:
            c.reset_parameters()
        for _, mod in self._readout():
            mod.reset_parameters()

    # ---- kernel launches ---------------------------------------------------------------------------------
    kernel_plan = "auto"   # "auto" | 0 (generic kernels) | 1 | 2 | 3 | 4 (relation-space kernels, CTAs per subgraph)
    #                        | 17 | 18 | 20 | 24 (L2 plan with 1 / 2 / 4 / 8 CTAs per subgraph, _lib.plan_l2)
    hidden_dropout_p = 0.5   # F.dropout(x, p=0.5) before lin2 (models.py:212)

    def _plan(self, batch):
        """kernel plan for this batch (``select_plan``): the relation-space kernels when the relation count allows,
        each subgraph spread over as many CTAs (1/2/4) as keeps the grid within one wave of the SMs; the generic
        kernels otherwise; the L2 plan when no shared-memory plan fits the subgraphs."""
        p = batch._priv
        key = (p["n_cap"], batch.num_graphs)
        c = self._plans.get(key)
        if c is not None:
            return c
        n_cap, B = p["n_cap"], batch.num_graphs
        want = self.kernel_plan
        env = os.environ.get("IGMC_PLAN")
        if want == "auto" and env:
            want = int(env)
        if self.num_relations <= 12 and n_cap > 256 and self._cmodel.list_hint == 0:
            # large subgraphs: size the shared-memory list buffers from the data (longest per-graph edge list of
            # this first batch, one host sync per model; the lists of one CTA hold its share of the directed edges)
            ep = p["edge_ptr"][:B + 1].cpu()
            self._max_edges = int((ep[1:] - ep[:-1]).max())
        sms = torch.cuda.get_device_properties(self.flat_params.device).multi_processor_count
        cl = select_plan(self._cmodel, n_cap, B, sms, want, self.__dict__.get("_max_edges"))
        self._plans[key] = cl
        return cl

    def _workspace(self, batch, train):
        p = batch._priv
        cl = self._plan(batch)
        key = (p["node_cap"], batch.num_graphs, bool(train), cl)
        ws = self._ws.get(key)
        if ws is None:
            dev, L, NB, B, ncap = self.flat_params.device, len(self.convs), self.num_bases, batch.num_graphs, \
                p["node_cap"]
            f32 = dict(dtype=torch.float32, device=dev)
            ws = dict(states=torch.empty(ncap, HID * L, **f32), inv_deg=torch.empty(ncap, **f32),
                      feat=torch.empty(B, 2 * HID * L, **f32), hid=torch.empty(B, 128, **f32),
                      hid_gscale=torch.empty(B, 128, **f32), pred=torch.empty(B, **f32),
                      target=torch.empty(B, 2, dtype=torch.int32, device=dev),
                      dpred=torch.zeros(B, **f32), sqerr=torch.zeros(B, **f32), loss=torch.zeros(1, **f32),
                      reg_ws=torch.zeros(_lib.REDUCE_WS_FLOATS, **f32), cluster=cl)
            if self.rgcn == "pyg-2":   # mean per relation: 1/|N_r(v)| table, filled by the forward
                ws["rel_inv_deg"] = torch.empty(ncap, self.num_relations, **f32)
            if train:
                if _lib.is_rs(cl):   # cluster plans: layer-0 aggregate only; raw partial rows (chain rule in igmc_grad_reduce)
                    zs = torch.empty(ncap, self.num_relations * _align4(self.num_features), **f32)
                    width = _lib.load().igmc_raw_grad_count(C.byref(self._cmodel))
                else:
                    zs = torch.empty(L, ncap, NB * HID, **f32)
                    width = self._cmodel.conv_param_count
                ws.update(zsave=zs, dstate=torch.empty(L, ncap, HID, **f32),
                          gpart=torch.zeros(B * _lib.ctas_per_graph(cl), width, **f32),
                          dhid=torch.empty(B, 128, **f32))
                if _lib.l2_csize(cl):   # d pre / d h of the backward (node features are not in shared memory)
                    ws["l2_scratch"] = torch.empty(2, ncap, HID, **f32)
            # never evicted: captured CUDA graphs hold raw pointers into these buffers (a handful of
            # (capacity, batch size, mode) keys per run; a few MB each)
            self._ws[key] = ws
        return ws

    # ---- pre-staged edge lists (igmc_stage_lists): built once per batch, off the model kernels' critical path ----
    def stage_batch(self, batch, training=True, drop=None, slot=0):
        """Build the list images of ``batch`` for the forward (and, when training, backward) kernel of its plan and
        attach them to the batch.  ``drop`` must be the dropout descriptor the step will use (same seed source).
        No-op for the generic and L2 plans."""
        self._check_types(batch)
        cl = self._plan(batch)
        if not _lib.is_rs(cl):
            batch._stage = None
            return None
        lib = _lib.load()
        p = batch._priv
        # (an image is laid out for n_cap, which an extractor that follows graph updates may lower inside buffers of the
        # same node_cap, and for the list capacity of list_hint, which a later plan for larger subgraphs may set)
        key = (p["node_cap"], p["n_cap"], batch.num_graphs, bool(training), cl, int(slot), self._cmodel.list_hint)
        cache = self.__dict__.setdefault("_stage_ws", {})
        st = cache.get(key)
        if st is None:
            dev = self.flat_params.device
            st = {}
            for name, bw in (("fwd", 0), ("bwd", 1)):
                if bw and not training:
                    continue
                img = _lib.Stage()
                _lib.check(lib.igmc_stage_plan(C.byref(self._cmodel), p["n_cap"], cl, bw, C.byref(img)),
                           "igmc_stage_plan")
                rows = batch.num_graphs * cl
                t = dict(tab=torch.zeros(rows, img.tab_ints, dtype=torch.int32, device=dev),
                         ent=torch.zeros(rows, img.lcap, dtype=torch.int32, device=dev))
                img.tab, img.ent = t["tab"].data_ptr(), t["ent"].data_ptr()
                if not bw:
                    t["inv_deg"] = torch.ones(p["node_cap"], dtype=torch.float32, device=dev)
                    img.inv_deg = t["inv_deg"].data_ptr()
                st[name] = (img, t)
            cache[key] = st
        if drop is None:
            drop = self.make_dropout(training)
        d, keep = drop
        adj_c, _ = batch.adjacency()
        _lib.check(lib.igmc_stage_lists(C.byref(self._cmodel), p["node_ptr"].data_ptr(), p["edge_ptr"].data_ptr(),
                                        C.byref(adj_c), batch.num_graphs, p["n_cap"], C.byref(d), int(training),
                                        C.byref(st["fwd"][0]), C.byref(st["bwd"][0]) if training else None,
                                        batch._err.data_ptr(), _stream_ptr()), "igmc_stage_lists")
        batch._stage = st
        return st

    @staticmethod
    def _stage_arg(batch, name):
        st = getattr(batch, "_stage", None)
        if not st or name not in st:
            return None
        return C.byref(st[name][0])

    def _saved_struct(self, ws, ncap):
        rs = _lib.is_rs(ws["cluster"])
        return _lib.Saved(ws["states"].data_ptr(), _lib.ptr(ws.get("zsave")), ws["inv_deg"].data_ptr(),
                          ws["feat"].data_ptr(), ws["hid"].data_ptr(), ws["hid_gscale"].data_ptr(),
                          ws["pred"].data_ptr(), ws["target"].data_ptr(), ncap, _lib.ptr(ws.get("dstate")),
                          _lib.ptr(self._wprep_buf()) if rs else None,
                          _lib.ptr(getattr(self, "_prof_buf", None)),
                          _lib.ptr(self._gate) if (rs and self.__dict__.pop("_gate_armed", False)) else None,
                          _lib.ptr(ws.get("l2_scratch")), _lib.ptr(ws.get("rel_inv_deg")))

    def _prep_weights_unless_prepped(self):
        """W_r / W_r^T of the current parameters (one tiny launch per step), unless ``prep_weights(mark=True)`` or the
        update kernel has just written them"""
        if not self.__dict__.pop("_prepped", False):
            self.prep_weights()

    def prep_weights(self, mark=False):
        """launch igmc_prep_weights on the current stream; ``mark`` lets the next forward skip its own launch (the
        train engine issues it early so that the extraction branch of the step can be ordered after it)."""
        _lib.check(_lib.load().igmc_prep_weights(C.byref(self._cmodel), self.flat_params.data_ptr(),
                                                 self._wprep_buf().data_ptr(), _stream_ptr()), "igmc_prep_weights")
        if mark:
            self._prepped = True

    def gate_wait(self, batch, timeout_us=300):
        """enqueue (on the CURRENT stream) a one-warp kernel that returns when every CTA of the next cluster-plan
        forward of ``batch``'s shape is resident: work queued behind it runs BESIDE that forward instead of in front
        of it (igmc_gate_wait).  The forward must be launched after this call (the gate pointer is armed here)."""
        cl = self._plan(batch)
        if not _lib.is_rs(cl):
            return
        if self.__dict__.get("_gate") is None:
            self._gate = torch.zeros(2, dtype=torch.int32, device=self.flat_params.device)
        _lib.check(_lib.load().igmc_gate_wait(self._gate.data_ptr(), batch.num_graphs * cl, int(timeout_us),
                                              _stream_ptr()), "igmc_gate_wait")
        self._gate_armed = True      # the next forward launch (and only that one) counts its CTAs into the gate

    def _wprep_buf(self):
        if self._wprep is None or self._wprep.device != self.flat_params.device:
            # two slabs per layer of wprep_slab(R) floats each (csrc/lists.cuh)
            n = len(self.convs) * 2 * HID * ((self.num_relations + 1) * HID + 4)
            self._wprep = torch.zeros(n, dtype=torch.float32, device=self.flat_params.device)
        return self._wprep

    def make_dropout(self, training, edge_keep=None, hidden_keep=None, seed=None, seed_dev=None):
        """dropout descriptor of one step (+ the tensors it references, to keep them alive)."""
        d = _lib.Dropout()
        d.adj_dropout = float(self.adj_dropout) if training else 0.0
        d.hidden_dropout = float(self.hidden_dropout_p) if training else 0.0
        if seed is None:
            seed = splitmix64(self.drop_seed + self._step)
        d.seed = int(seed) & ((1 << 64) - 1)
        keep = []
        if seed_dev is not None:
            d.seed_dev = seed_dev.data_ptr()
            keep.append(seed_dev)
        if edge_keep is not None:
            ek = torch.as_tensor(edge_keep).to(self.flat_params.device).to(torch.uint8).contiguous()
            d.edge_keep = ek.data_ptr()
            keep.append(ek)
        if hidden_keep is not None:
            hk = torch.as_tensor(hidden_keep).to(self.flat_params.device).to(torch.uint8).contiguous()
            d.hidden_keep = hk.data_ptr()
            keep.append(hk)
        return d, keep

    def _launch_forward(self, batch, training, drop, y=None, loss_scale=0.0):
        lib = _lib.load()
        p = batch._priv
        adj_c, _ = batch.adjacency()
        ws = self._workspace(batch, training)
        S = self._saved_struct(ws, p["node_cap"])
        d, keep = drop
        if _lib.is_rs(ws["cluster"]):
            self._prep_weights_unless_prepped()
        _lib.check(lib.igmc_forward(C.byref(self._cmodel), self.flat_params.data_ptr(), p["node_label"].data_ptr(),
                                    p["node_ptr"].data_ptr(), p["edge_ptr"].data_ptr(), C.byref(adj_c),
                                    batch.num_graphs, p["n_cap"], C.byref(d), int(training), C.byref(S),
                                    _lib.ptr(y), float(loss_scale), ws["dpred"].data_ptr() if y is not None else None,
                                    ws["sqerr"].data_ptr() if y is not None else None, ws["cluster"],
                                    self._stage_arg(batch, "fwd"), batch._err.data_ptr(), _stream_ptr()),
                   "igmc_forward")
        return ws["pred"], dict(ws=ws, S=S, train=bool(training))

    def _launch_backward(self, batch, drop, saved, dpred):
        lib = _lib.load()
        p = batch._priv
        adj_c, _ = batch.adjacency()
        ws = saved["ws"]
        d, keep = drop
        saved["dpred_used"] = dpred
        _lib.check(lib.igmc_backward(C.byref(self._cmodel), self.flat_params.data_ptr(), p["node_label"].data_ptr(),
                                     p["node_ptr"].data_ptr(), p["edge_ptr"].data_ptr(), C.byref(adj_c),
                                     batch.num_graphs, p["n_cap"], C.byref(d), C.byref(saved["S"]),
                                     dpred.data_ptr(), ws["gpart"].data_ptr(), ws["dhid"].data_ptr(), ws["cluster"],
                                     self._stage_arg(batch, "bwd"), batch._err.data_ptr(), _stream_ptr()),
                   "igmc_backward")

    def _launch_grad_reduce(self, batch, saved, loss_scale, arr, with_loss=True):
        lib = _lib.load()
        ws = saved["ws"]
        _lib.check(lib.igmc_grad_reduce(C.byref(self._cmodel), self.flat_params.data_ptr(), batch.num_graphs,
                                        batch.num_graphs * _lib.ctas_per_graph(ws["cluster"]),
                                        ws["gpart"].data_ptr(), 1 if _lib.is_rs(ws["cluster"]) else 0,
                                        ws["dhid"].data_ptr(), ws["feat"].data_ptr(),
                                        ws["hid"].data_ptr(), saved["dpred_used"].data_ptr(),
                                        ws["sqerr"].data_ptr() if with_loss else None, float(loss_scale),
                                        float(arr), 1.0, self.flat_grad.data_ptr(),
                                        ws["loss"].data_ptr() if with_loss else None, ws["reg_ws"].data_ptr(),
                                        _stream_ptr()), "igmc_grad_reduce")

    # ---- public API ------------------------------------------------------------------------------------------
    def _check_types(self, batch):
        """IndexError unless every edge type of a foreign batch lies in [0, num_relations): the kernels index the
        relation tables with it (PyG's RGCNConv fails in index_select).  Foreign batches and batches assembled from a
        StaticStore carry the range; extracted batches are checked by the extractor (IGMC_ERR_LABEL)."""
        tr = batch._priv.get("type_range")
        if tr is not None and (tr[0] < 0 or tr[1] >= self.num_relations):
            bad = tr[0] if tr[0] < 0 else tr[1]
            raise IndexError("edge type %d outside the model's %d relations (types must lie in [0, %d))"
                             % (bad, self.num_relations, self.num_relations))

    def _as_batch(self, data):
        if isinstance(data, Batch):
            return data
        if getattr(data, "batch", None) is None:
            raise ValueError("IGMC.forward expects a collated Batch")
        return Batch.from_arrays(data.x, data.edge_index, data.edge_type, data.batch, data.y,
                                 getattr(data, "num_graphs", None), self.flat_params.device)

    def forward(self, data, edge_keep=None, hidden_keep=None):
        batch = self._as_batch(data)
        self._check_types(batch)
        drop = self.make_dropout(self.training, edge_keep, hidden_keep)
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if need_grad:
            self._step += 1
            params = [p for (_, _, p) in self._named_order()]
            return _IGMCFunction.apply(self, batch, self.training, drop, *params)
        out, _ = self._launch_forward(batch, False if not self.training else True, drop)
        return out.clone()

    def forward_backward(self, batch, global_num_graphs=None, edge_keep=None, hidden_keep=None, seed_dev=None):
        """prep + forward + loss + backward of one training step WITHOUT the gradient assembly: leaves the raw partial
        rows / readout factors in the workspace for ``FusedAdam.reduce_update`` (or ``_launch_grad_reduce``)."""
        return self._train_launches(batch, global_num_graphs, edge_keep, hidden_keep, seed_dev, one_launch=True)[0]

    def _train_launches(self, batch, global_num_graphs, edge_keep, hidden_keep, seed_dev, one_launch):
        """the step's forward + loss + backward launches; ``one_launch`` allows igmc_forward_backward where the plan
        has it.  Returns (saved, G)."""
        self._check_types(batch)
        self._step += 1
        drop = self.make_dropout(True, edge_keep, hidden_keep, seed_dev=seed_dev)
        G = batch.num_graphs if global_num_graphs is None else int(global_num_graphs)
        if one_launch and self._cmodel.readout == 0 and _lib.is_rs(self._plan(batch)) \
                and os.environ.get("IGMC_FUSED_FB", "1") != "0":
            return self._launch_train(batch, drop, batch.y, 1.0 / G), G
        out, saved = self._launch_forward(batch, True, drop, y=batch.y, loss_scale=1.0 / G)
        self._launch_backward(batch, drop, saved, saved["ws"]["dpred"])
        return saved, G

    def _launch_train(self, batch, drop, y, loss_scale):
        """forward + loss + backward as ONE launch (igmc_forward_backward): cluster plans, IGMC readout."""
        lib = _lib.load()
        p = batch._priv
        adj_c, _ = batch.adjacency()
        ws = self._workspace(batch, True)
        S = self._saved_struct(ws, p["node_cap"])
        d, keep = drop
        self._prep_weights_unless_prepped()
        _lib.check(lib.igmc_forward_backward(C.byref(self._cmodel), self.flat_params.data_ptr(),
                                             p["node_label"].data_ptr(), p["node_ptr"].data_ptr(),
                                             p["edge_ptr"].data_ptr(), C.byref(adj_c), batch.num_graphs, p["n_cap"],
                                             C.byref(d), C.byref(S), y.data_ptr(), float(loss_scale),
                                             ws["dpred"].data_ptr(), ws["sqerr"].data_ptr(), ws["gpart"].data_ptr(),
                                             ws["dhid"].data_ptr(), ws["cluster"], self._stage_arg(batch, "fwd"),
                                             self._stage_arg(batch, "bwd"), batch._err.data_ptr(), _stream_ptr()),
                   "igmc_forward_backward")
        return dict(ws=ws, S=S, train=True, dpred_used=ws["dpred"])

    def fused_update_ok(self, batch):
        """the one-kernel reduce -> all-reduce -> Adam path needs raw partial rows (cluster plans) and the IGMC
        readout (an external readout writes its own gradient slice), and a grid the device runs at once: the kernel's
        grid barriers wait for every block (one per layer input row, so more than 4 layers do not fit on an H100)."""
        if self._cmodel.readout != 0 or not _lib.is_rs(self._plan(batch)):
            return False
        fits = self.__dict__.get("_update_grid_fits")
        if fits is None:
            blocks, resident = C.c_int(), C.c_int()
            _lib.check(_lib.load().igmc_reduce_update_grid(C.byref(self._cmodel), C.byref(blocks), C.byref(resident)),
                       "igmc_reduce_update_grid")
            fits = self._update_grid_fits = blocks.value <= resident.value
        return fits

    def fused_step(self, batch, ARR=0.0, global_num_graphs=None, edge_keep=None, hidden_keep=None,
                   seed_dev=None):
        """forward + MSE (+ARR) + backward + gradient assembly, no autograd, no host sync.

        Equivalent to the body of the reference's ``train`` loop up to ``loss.backward()``
        (train_eval.py:158-175).  ``flat_grad`` then holds d loss / d params where the MSE mean is taken
        over ``global_num_graphs`` (defaults to this batch; under data parallelism pass B*world so that an
        NCCL SUM of flat_grad is the gradient of the global-batch mean).  Returns the device scalar
        ``sum_g (out_g-y_g)^2 / global_num_graphs + ARR*reg``.
        """
        saved, G = self._train_launches(batch, global_num_graphs, edge_keep, hidden_keep, seed_dev, one_launch=False)
        self._launch_grad_reduce(batch, saved, loss_scale=1.0 / G, arr=ARR, with_loss=True)
        return saved["ws"]["loss"]

    def __repr__(self):
        return self.__class__.__name__


class DGCNN_RS(IGMC):
    """Drop-in for the reference's ``DGCNN_RS`` (models.py:123-167; constructor chain DGCNN.__init__ models.py:65-85):
    R-GCN layers with ``latent_dim=[32,32,32,1]``, SortPooling over the last channel, two 1-D convolutions and the
    dense head, on the same fused kernels as ``IGMC`` plus ``csrc/sortpool.cu`` for the readout.

    The conv kernels run 32-wide layers, so a layer with fewer output channels (the last one) is stored padded in the
    flat bucket: ``convs[-1].basis/root/bias`` are strided views of a 32-wide slot whose other columns are zero and stay
    zero (their gradients are exactly zero).  ``state_dict`` keys and shapes are the reference's.

    ``k < 1`` is the reference's percentile rule over ALL subgraphs (models.py:69-73); the node counts come from
    ``dataset.node_counts()`` (large GPU batches) instead of a Python loop over ``dataset``.
    """

    C1, C2, KW2 = 16, 32, 5   # conv1d_channels and the second kernel width (models.py:75-79)
    REGRESSION_ONLY = "igmc_b200.DGCNN_RS implements the regression head (x[:, 0], models.py:165)"

    def __init__(self, dataset, gconv=RGCNConv, latent_dim=[32, 32, 32, 1], k=30, num_relations=5, num_bases=2,
                 regression=False, adj_dropout=0.2, force_undirected=False, rgcn="pyg-1.4"):
        nn.Module.__init__(self)
        latent_dim = [int(d) for d in latent_dim]
        self._init_convs(dataset, latent_dim, num_relations, num_bases, regression, adj_dropout, force_undirected,
                         False, 1, rgcn)
        if k < 1:   # transform percentile to number (models.py:69-73)
            if isinstance(dataset, int):
                raise ValueError("a percentile k needs the dataset")
            if hasattr(dataset, "node_counts"):      # all subgraphs, extracted in large GPU batches
                node_nums = sorted(int(v) for v in dataset.node_counts())
            else:
                node_nums = sorted(int(g.num_nodes) for g in dataset)
            k = node_nums[int(math.ceil(k * len(node_nums))) - 1]
            k = max(10, k)
        self.k = int(k)
        self.latent_dim = latent_dim
        self.total_latent_dim = sum(latent_dim)
        self.conv1d_params1 = nn.Conv1d(1, self.C1, self.total_latent_dim, self.total_latent_dim)
        self.maxpool1d = nn.MaxPool1d(2, 2)
        self.conv1d_params2 = nn.Conv1d(self.C1, self.C2, self.KW2, 1)
        dense_dim = int((self.k - 2) / 2 + 1)
        self.dense_dim = (dense_dim - self.KW2 + 1) * self.C2
        if self.dense_dim <= 0:
            raise ValueError("k = %d is too small for the 1-D convolutions" % self.k)
        self.lin1 = nn.Linear(self.dense_dim, 128)
        self.lin2 = nn.Linear(128, 1)
        self._init_bucket()

    @staticmethod
    def _check_latent_dim(latent_dim):
        if not (1 <= len(latent_dim) <= _lib.MAX_LAYERS) or any(d != HID for d in latent_dim[:-1]) \
                or not (1 <= latent_dim[-1] <= HID):
            raise NotImplementedError("latent_dim must be [32, ..., 32, d] with 1 <= d <= 32")

    def _readout(self):
        return (("conv1", self.conv1d_params1), ("conv2", self.conv1d_params2), ("lin1", self.lin1),
                ("lin2", self.lin2))

    def _slot(self, kind, l, p):
        if kind in ("basis", "root", "bias") and p.shape[-1] != HID:
            pad = tuple(p.shape[:-1]) + (HID,)
            return int(torch.Size(pad).numel()), pad
        return p.numel(), None

    def _flatten(self):
        super()._flatten()
        self._cmodel.readout = 1
        o, sp = self._offs, _lib.SortPool()
        sp.k, sp.width, sp.state_stride = self.k, self.total_latent_dim, HID * len(self.convs)
        sp.c1, sp.c2, sp.kw2 = self.C1, self.C2, self.KW2
        sp.t1 = self.k // 2
        sp.t2 = sp.t1 - self.KW2 + 1
        sp.dense_dim = self.dense_dim
        assert sp.dense_dim == sp.c2 * sp.t2
        sp.off_conv1_w, sp.off_conv1_b, sp.off_conv2_w, sp.off_conv2_b = o["conv1_w"], o["conv1_b"], o["conv2_w"], \
            o["conv2_b"]
        sp.off_lin1_w, sp.off_lin1_b, sp.off_lin2_w, sp.off_lin2_b = o["lin1_w"], o["lin1_b"], o["lin2_w"], o["lin2_b"]
        sp.param_begin, sp.param_end = self._cmodel.conv_param_count, self._cmodel.param_count
        self._csort = sp

    def _workspace(self, batch, train):
        ws = super()._workspace(batch, train)
        if "sp" not in ws:
            lib = _lib.load()
            p, sp, B = batch._priv, self._csort, batch.num_graphs
            for bw in (0, 1):
                if lib.igmc_sortpool_plan(C.byref(sp), p["n_cap"], bw) <= 0:
                    raise RuntimeError("igmc_b200: the SortPooling readout (k = %d) does not fit in shared memory" % self.k)
            dev = self.flat_params.device
            f32, i32 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int32, device=dev)
            gp = sp.c1 * sp.width + sp.c1 + sp.c2 * sp.c1 * sp.kw2 + sp.c2
            d = dict(rank=torch.zeros(p["node_cap"], **i32), perm=torch.zeros(B, sp.k, **i32),
                     act1=torch.empty(B, sp.c1, sp.k, **f32), pool=torch.empty(B, sp.c1, sp.t1, **f32),
                     flat=torch.empty(B, sp.dense_dim, **f32), hid=torch.empty(B, 128, **f32),
                     hid_gscale=torch.empty(B, 128, **f32), pred=torch.empty(B, **f32),
                     dhid=torch.empty(B, 128, **f32), gpart=torch.zeros(B, gp, **f32))
            d["S"] = _lib.SortPoolSaved(*[d[k].data_ptr() for k in ("rank", "perm", "act1", "pool", "flat", "hid",
                                                                    "hid_gscale", "pred", "dhid", "gpart")])
            ws["sp"] = d
        return ws

    def _launch_forward(self, batch, training, drop, y=None, loss_scale=0.0):
        lib = _lib.load()
        _, saved = super()._launch_forward(batch, training, drop, y=None)    # concat_states only (readout = 1)
        ws, p = saved["ws"], batch._priv
        d, keep = drop
        _lib.check(lib.igmc_sortpool_forward(C.byref(self._csort), self.flat_params.data_ptr(),
                                             ws["states"].data_ptr(), p["node_ptr"].data_ptr(), batch.num_graphs,
                                             p["n_cap"], C.byref(d), int(training), C.byref(ws["sp"]["S"]),
                                             _lib.ptr(y), float(loss_scale),
                                             ws["dpred"].data_ptr() if y is not None else None,
                                             ws["sqerr"].data_ptr() if y is not None else None,
                                             batch._err.data_ptr(), _stream_ptr()), "igmc_sortpool_forward")
        return ws["sp"]["pred"], saved

    def _launch_backward(self, batch, drop, saved, dpred):
        lib = _lib.load()
        ws, p = saved["ws"], batch._priv
        _lib.check(lib.igmc_sortpool_backward(C.byref(self._csort), self.flat_params.data_ptr(),
                                              ws["states"].data_ptr(), p["node_ptr"].data_ptr(), batch.num_graphs,
                                              p["n_cap"], C.byref(ws["sp"]["S"]), dpred.data_ptr(),
                                              ws["dstate"].data_ptr(), 1.0, self.flat_grad.data_ptr(),
                                              batch._err.data_ptr(), _stream_ptr()), "igmc_sortpool_backward")
        super()._launch_backward(batch, drop, saved, dpred)


class FusedAdam(torch.optim.Optimizer):
    """``torch.optim.Adam`` semantics (train_eval.py:54) as ONE kernel over the flat bucket.

    ``state_dict()`` has the stock Adam structure (per-parameter ``step/exp_avg/exp_avg_sq`` that are
    views of the flat moments), so optimizer checkpoints interchange with the reference's
    (Main.py:45, train_eval.py:60-62)."""

    def __init__(self, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        self.model = model
        # parameter ORDER = model.parameters(), i.e. what the reference's Adam(model.parameters()) (train_eval.py:54)
        # sees (per conv: basis, att, root, bias): optimizer state_dicts are keyed by position in this list.  The
        # flat bucket has its own order (model._layout); `_entry` maps a parameter to its slice.
        params = list(model.parameters())
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False))
        dev = model.flat_params.device
        n = model.flat_params.numel()
        self.exp_avg = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev)
        self.step_count = torch.zeros(2, dtype=torch.int64, device=dev)   # [step | completion ticket of the kernel]
        self._entry = {id(p): e for e, (_, _, p) in zip(model._layout, model._named_order())}
        for p in params:
            e = self._entry[id(p)]
            self.state[p] = dict(step=self.step_count[0], exp_avg=model._pview(self.exp_avg, e),
                                 exp_avg_sq=model._pview(self.exp_avg_sq, e))

    def state_dict(self):
        """stock ``torch.optim.Adam`` layout with INDEPENDENT per-parameter tensors: every ``step`` is its own float32
        scalar (torch's Adam increments each one separately - shared storage would be bumped once per parameter)
        and the moments are contiguous clones, so the file loads into ``torch.optim.Adam`` of the reference
        (Main.py:45, train_eval.py:60-62) as well as back into ``FusedAdam``."""
        sd = super().state_dict()
        step = float(self.step_count[0].item())
        out_state = {}
        for k, st in sd["state"].items():
            out_state[k] = dict(step=torch.tensor(step, dtype=torch.float32),
                                exp_avg=st["exp_avg"].detach().clone().contiguous(),
                                exp_avg_sq=st["exp_avg_sq"].detach().clone().contiguous())
        return dict(state=out_state, param_groups=sd["param_groups"])

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        params = list(self.model.parameters())
        with torch.no_grad():
            for p in params:
                e = self._entry[id(p)]
                st = self.state[p]
                ea, es = self.model._pview(self.exp_avg, e), self.model._pview(self.exp_avg_sq, e)
                ea.copy_(st["exp_avg"])
                es.copy_(st["exp_avg_sq"])
                self.step_count[0] = int(st["step"])
                self.state[p] = dict(step=self.step_count[0], exp_avg=ea, exp_avg_sq=es)

    @torch.no_grad()
    def step(self, grad_mul=1.0, lr_dev=None, loss_in=None, loss_acc=None, loss_weight=0.0):
        lib = _lib.load()
        self.model._prepped = False   # parameters change: the prepared weights are stale
        g = self.param_groups[0]
        m = self.model
        _lib.check(lib.igmc_adam_step(m.flat_params.data_ptr(), m.flat_grad.data_ptr(), self.exp_avg.data_ptr(),
                                      self.exp_avg_sq.data_ptr(), self.step_count.data_ptr(),
                                      m.flat_params.numel(), float(g["lr"]), _lib.ptr(lr_dev),
                                      float(g["betas"][0]),
                                      float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"]),
                                      float(grad_mul), _lib.ptr(loss_in), _lib.ptr(loss_acc) if loss_in is not None else None,
                                      float(loss_weight), _stream_ptr()), "igmc_adam_step")

    @torch.no_grad()
    def reduce_update(self, exchange, ws, B, rows, loss_scale, arr, lr_dev=None, loss_acc=None, loss_weight=0.0,
                      grad_copy=None, loss_ring=None):
        """gradient assembly (+ARR) -> one-shot all-reduce over the ranks of ``exchange`` -> Adam, ONE kernel
        (igmc_reduce_update).  ``ws`` is the model workspace ``forward_backward`` filled (``B`` graphs, ``rows`` raw
        partial rows; both 0 for a rank that holds no graph of a short tail batch)."""
        lib = _lib.load()
        g = self.param_groups[0]
        m = self.model
        _lib.check(lib.igmc_reduce_update(C.byref(m._cmodel), m.flat_params.data_ptr(), int(B), int(rows),
                                          ws["gpart"].data_ptr(), ws["dhid"].data_ptr(), ws["feat"].data_ptr(),
                                          ws["hid"].data_ptr(), ws["dpred"].data_ptr(), ws["sqerr"].data_ptr(),
                                          float(loss_scale), float(arr), C.byref(exchange.c),
                                          self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
                                          self.step_count.data_ptr(), float(g["lr"]), _lib.ptr(lr_dev),
                                          float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]),
                                          float(g["weight_decay"]), 1.0, ws["loss"].data_ptr(), _lib.ptr(loss_acc),
                                          float(loss_weight), ws["reg_ws"].data_ptr(), _lib.ptr(grad_copy),
                                          _lib.ptr(loss_ring), int(loss_ring.numel()) if loss_ring is not None else 0,
                                          m._wprep_buf().data_ptr(), _stream_ptr()), "igmc_reduce_update")
        m._prepped = True     # the update kernel re-prepared W_r / W_r^T from the new parameters (next forward skips it)
        return ws["loss"]

    def zero_grad(self, set_to_none=False):
        pass  # flat_grad is fully overwritten by every fused_step
