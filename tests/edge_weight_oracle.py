"""fp64 restatement of the model with a weight on every directed edge (the definition behind ``attribute_pairs``), built
on oracle/pyg_restated.py and tests/pyg2_oracle.py without changing them.

Directed edge e carries weight w_e.  It multiplies the edge's message, and the mean normalisers count the weights:
``aggr="mean_all"`` (PyG 1.4.2) divides by deg(v) = sum of w over v's in-edges, ``aggr="mean_per_relation"`` (PyG
>= 1.6) each relation's sum by |N_r(v)| = sum of w over v's in-edges of type r.  A normaliser of 0 (no in-edge, or all
weights 0) leaves the aggregate 0, as scatter_mean does.  w = 1 is the restated model; a 0/1 w is dropout_adj with
that draw.  ``centred_edge_grad`` is the closed form the CUDA kernel evaluates."""
import torch
import torch.nn.functional as F

from oracle import pyg_restated


def _weights(conv):
    return torch.matmul(conv.att, conv.basis.view(conv.num_bases, -1)).view(conv.num_relations, conv.in_channels,
                                                                             conv.out_channels)


def _segments(conv, dst, et):
    """segment id of every directed edge: its destination, or (destination, relation) for the per-relation mean"""
    return dst * conv.num_relations + et if conv.aggr == "mean_per_relation" else dst


def _conv_pre(conv, x, edge_index, edge_type, w):
    """pre-activation of one weighted layer"""
    src, dst = edge_index[0], edge_index[1]
    n = x.shape[0]
    msg = torch.einsum("ni,rio->nro", x, _weights(conv))[src, edge_type] * w[:, None]
    seg = _segments(conv, dst, edge_type)
    nseg = n * conv.num_relations if conv.aggr == "mean_per_relation" else n
    den = torch.zeros(nseg, dtype=x.dtype, device=x.device).index_add(0, seg, w)
    den = torch.where(den > 0, den, torch.ones_like(den))
    agg = torch.zeros(n, msg.shape[1], dtype=x.dtype, device=x.device).index_add(0, dst, msg / den[seg][:, None])
    return agg + x @ conv.root + conv.bias


def _sort_pool(cs, batch, k, num_graphs, perm):
    """SortPooling of pyg_restated.global_sort_pool, or, with ``perm`` [B, k] (node index or -1, the kernel's order),
    the rows that order names"""
    if perm is None:
        return pyg_restated.global_sort_pool(cs, batch, k, num_graphs)
    perm = torch.as_tensor(perm, device=cs.device).long()
    rows = torch.where(perm[..., None] >= 0, cs[perm.clamp(min=0)], torch.zeros((), dtype=cs.dtype, device=cs.device))
    return rows.reshape(perm.shape[0], -1)


def weighted_forward(ref, x, edge_index, edge_type, w, batch=None, num_graphs=None, perm=None, trace=None):
    """eval-mode scores [B] of the restated IGMC (IGMCRef / IGMC2Ref) or DGCNN_RS (DGCNN_RSRef / DGCNN_RS2Ref) ``ref``
    with edge weights ``w`` [E].  ``trace``: a list that receives (h_{l-1}, pre_l) of every layer."""
    h, states = x, []
    for conv in ref.convs:
        pre = _conv_pre(conv, h, edge_index, edge_type, w)
        if trace is not None:
            trace.append((h, pre))
        h = torch.tanh(pre)
        states.append(h)
    cs = torch.cat(states, 1)
    if isinstance(ref, pyg_restated.DGCNN_RSRef):
        z = _sort_pool(cs, batch, ref.k, num_graphs, perm).unsqueeze(1)
        z = F.relu(ref.conv1d_params1(z))
        z = ref.maxpool1d(z)
        z = F.relu(ref.conv1d_params2(z))
        z = F.relu(ref.lin1(z.view(len(z), -1)))
        return ref.lin2(z)[:, 0]
    users, items = x[:, 0] == 1, x[:, 1] == 1
    z = F.relu(ref.lin1(torch.cat([cs[users], cs[items]], 1)))
    return ref.lin2(z)[:, 0] * ref.multiply_by


def autograd_edge_grad(ref, x, edge_index, edge_type, **kw):
    """d (sum of the scores) / d w_e at w = 1, per directed edge [E], by autograd"""
    w = torch.ones(edge_index.shape[1], dtype=x.dtype, device=x.device, requires_grad=True)
    weighted_forward(ref, x, edge_index, edge_type, w, **kw).sum().backward()
    return w.grad.detach()


def centred_edge_grad(ref, x, edge_index, edge_type, **kw):
    """the same gradient in closed form: for every layer l and directed edge j -> v of type r, with s = <h_{l-1}[j] W_r,
    d pre_l[v]> (d pre_l by autograd), (s - mean of s over v's segment) / |segment|, summed over the layers"""
    w = torch.ones(edge_index.shape[1], dtype=x.dtype, device=x.device)
    trace = []
    with torch.enable_grad():
        out = weighted_forward(ref, x, edge_index, edge_type, w, trace=trace, **kw)
        dpre = torch.autograd.grad(out.sum(), [pre for _, pre in trace])
    src, dst = edge_index[0], edge_index[1]
    g = torch.zeros_like(w)
    for conv, (h, _), dp in zip(ref.convs, trace, dpre):
        with torch.no_grad():
            s = (torch.einsum("ni,rio->nro", h, _weights(conv))[src, edge_type] * dp[dst]).sum(1)
            seg = _segments(conv, dst, edge_type)
            nseg = int(seg.max()) + 1 if len(seg) else 0
            cnt = torch.zeros(nseg, dtype=s.dtype, device=s.device).index_add(0, seg, torch.ones_like(s))
            tot = torch.zeros(nseg, dtype=s.dtype, device=s.device).index_add(0, seg, s)
            g += (s - tot[seg] / cnt[seg]) / cnt[seg]
    return g


def rating_grad(g, m):
    """per rating j < m of a [u|v ; v|u] subgraph: the sum of its two directed edges' gradients"""
    return g[:m] + g[m:2 * m]
