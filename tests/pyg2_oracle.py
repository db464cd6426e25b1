"""Test oracle of the PyG >= 1.6 ``RGCNConv`` (``IGMC(..., rgcn="pyg-2")``), built on oracle/pyg_restated.py without
changing it.

The layer: parameters ``weight [B,in,out]`` (the 1.4.2 ``basis``), ``comp [R,B]`` (``att``), ``root [in,out]``,
``bias [out]``; init glorot(weight, comp, root) = U(+-sqrt(6 / (size(-2) + size(-1)))), zeros(bias); aggregation
``aggr='mean'`` taken PER RELATION:

    x'_i = x_i root + bias + sum_r 1/|N_r(i)| sum_{j in N_r(i)} x_j W_r,   W_r = sum_b comp[r,b] weight[b]

Those facts are recalled from PyG's sources and documentation; no PyG build or checkpoint here pins them.  The models
subclass ``IGMCRef`` / ``DGCNN_RSRef``, so tests/helpers.py (``oracle_train_step``, ``assert_step_matches``,
``check_step``) and ``pyg_restated.arr_regulariser`` / ``train_loss`` / ``set_formulation`` work on them unchanged."""
import math

import torch
import torch.nn as nn

from oracle import pyg_restated


def mean_per_relation(msg, dst, edge_type, n, R):
    """sum over relations of the mean of the messages of each (destination, relation) segment: [n, out]"""
    seg = dst * R + edge_type
    cnt = torch.zeros(n * R, dtype=msg.dtype, device=msg.device).index_add_(0, seg, torch.ones_like(seg, dtype=msg.dtype))
    return torch.zeros(n, msg.shape[1], dtype=msg.dtype, device=msg.device).index_add_(0, dst, msg / cnt[seg].unsqueeze(1))


class RGCNConvRelMeanRef(pyg_restated.RGCNConvRef):
    """``RGCNConvRef`` that also takes ``aggr="mean_per_relation"`` (PyG 1.4.2 names and init), in both message
    formulations ("bmm": per-edge weight gather + bmm; "transform": x W_r first, then a row gather)."""

    def forward(self, x, edge_index, edge_type):
        if self.aggr != "mean_per_relation":
            return super().forward(x, edge_index, edge_type)
        src, dst = edge_index[0], edge_index[1]
        w = torch.matmul(self.att, self.basis.view(self.num_bases, -1))
        w = w.view(self.num_relations, self.in_channels, self.out_channels)
        if self.formulation == "transform":
            msg = torch.einsum("ni,rio->nro", x, w)[src, edge_type]
        else:
            msg = torch.bmm(x[src].unsqueeze(1), torch.index_select(w, 0, edge_type)).squeeze(1)
        return mean_per_relation(msg, dst, edge_type, x.shape[0], self.num_relations) + x @ self.root + self.bias


class RGCNConv2Ref(RGCNConvRelMeanRef):
    """PyG >= 1.6 ``RGCNConv(in, out, num_relations, num_bases)``: ``comp`` / ``weight`` names, glorot / zeros init,
    mean per relation."""

    def __init__(self, in_channels, out_channels, num_relations, num_bases, aggr="mean_per_relation"):
        nn.Module.__init__(self)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.num_relations, self.num_bases = num_relations, num_bases
        self.aggr = aggr
        self.weight = nn.Parameter(torch.empty(num_bases, in_channels, out_channels))
        self.comp = nn.Parameter(torch.empty(num_relations, num_bases))
        self.root = nn.Parameter(torch.empty(in_channels, out_channels))
        self.bias = nn.Parameter(torch.empty(out_channels))
        self.reset_parameters()

    # the message code (and pyg_restated.arr_regulariser) read ``att`` / ``basis``: the same tensors by the new names
    @property
    def att(self):
        return self.comp

    @property
    def basis(self):
        return self.weight

    def reset_parameters(self):
        for p in (self.weight, self.comp, self.root):
            bound = math.sqrt(6.0 / (p.size(-2) + p.size(-1)))
            p.data.uniform_(-bound, bound)
        self.bias.data.zero_()


def _pyg2_convs(model, dims, num_relations, num_bases):
    # (assigning to the existing ``convs`` entry keeps its place in the state_dict order)
    model.convs = nn.ModuleList([RGCNConv2Ref(dims[l], dims[l + 1], num_relations, num_bases)
                                 for l in range(len(dims) - 1)])


class IGMC2Ref(pyg_restated.IGMCRef):
    """``IGMCRef`` with the PyG >= 1.6 layer (state_dict keys ``convs.{l}.weight/comp/root/bias``, lin1, lin2)."""

    def __init__(self, num_features=4, latent_dim=(32, 32, 32, 32), num_relations=5, num_bases=4, adj_dropout=0.2,
                 multiply_by=1):
        super().__init__(num_features, latent_dim, num_relations, num_bases, adj_dropout, multiply_by)
        _pyg2_convs(self, [num_features] + list(latent_dim), num_relations, num_bases)


class DGCNN_RS2Ref(pyg_restated.DGCNN_RSRef):
    """``DGCNN_RSRef`` with the PyG >= 1.6 layer."""

    def __init__(self, num_features=4, latent_dim=(32, 32, 32, 1), k=30, num_relations=5, num_bases=2,
                 adj_dropout=0.2):
        super().__init__(num_features, latent_dim, k, num_relations, num_bases, adj_dropout)
        _pyg2_convs(self, [num_features] + list(latent_dim), num_relations, num_bases)


def igmc_ref(rgcn, *a, **kw):
    """the restated IGMC of layer ``rgcn`` ("pyg-1.4": pyg_restated.IGMCRef, "pyg-2": IGMC2Ref)"""
    return (pyg_restated.IGMCRef if rgcn == "pyg-1.4" else IGMC2Ref)(*a, **kw)


def dgcnn_rs_ref(rgcn, *a, **kw):
    return (pyg_restated.DGCNN_RSRef if rgcn == "pyg-1.4" else DGCNN_RS2Ref)(*a, **kw)
