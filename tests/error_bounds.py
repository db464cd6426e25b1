"""Per-element fp32 error bounds of the model kernels, one layer at a time.

Every quantity a kernel writes (a layer's states, the predictions, ``d hid`` and the assembled parameter gradient) is
recomputed in fp64 from the kernel's OWN inputs to that step: layer l from the kernel's saved ``h_{l-1}``, the readout
from the kernel's concatenated states, the backward from the kernel's ``dpred`` with ``tanh' = 1 - h^2`` of the
kernel's ``h``.  Every branch (ReLU masks, hidden dropout scales, MaxPool argmax, the SortPooling order) is taken from
what the kernel saved, so a value within rounding of a kink cannot put the two sides on different branches;
``branch_mismatches`` checks separately that every branch away from its kink is the one the fp64 value takes.  The
per-layer arithmetic is the restated conv (oracle/pyg_restated.py ``RGCNConvRef``; tests/pyg2_oracle.py for the mean
per relation of ``rgcn="pyg-2"``) in its memory-light "transform" formulation.

The magnitude pass runs the same code on ``|x|``, ``|h|``, ``|att|``, ``|basis|`` (not ``|W_r|``: the kernels round W_r
themselves), ``|root|``, ``|bias|``, the absolute readout weights and ``|dpred|``, with the same masks and the positive
mean weights.  Its output ``M`` is, per element, the sum of the absolute values of the terms behind that element, so a
kernel that sums those terms in fp32 in any order is off by at most a small multiple of ``u * M`` (``u = 2^-24``):

    |got - ref| <= KAPPA[quantity] * u * M,     and got == 0 exactly where M == 0 (padding columns, empty rows).

A state ``h = tanh(pre)`` is bounded by ``(1 - h^2) M_pre + |h|``: the pre-activation's bound through tanh' plus the
rounding of tanhf itself."""
import torch
import torch.nn.functional as F

U = 2.0 ** -24

# The smallest power of two at least 4x the largest err / (u M) measured over every case of
# tests/test_gpu_error_bounds.py on an H100 80GB HBM3 (700 W): states 10.3 (plan 0 and the L2 plan, fp32 sums in
# sequence), predictions 0.097, d hid 0.99 (two roundings of one product), gradients 5.0 (ml_1m* batch 50).  A lost
# 3xTF32 cross term or an operand truncated to TF32 is off by ~2^-11 of its products: hundreds to thousands of u M.
# The prediction bound is below one rounding of u M.  It holds because a prediction is a heavily cancelling sum over
# 128 hidden units and the lin1 sums behind them, so |pred| is far below M.  A prediction whose |pred| came close to
# M could exceed 0.5 u M with correct fp32 arithmetic; a reordering of those sums that trips it is not by itself a
# kernel bug.  The num_bases = 2 cases, on the same H100 and power limit, stay inside these constants: states 7.9 (R = 71
# on the L2 plan), predictions 0.139 (ml_1m* batch 50, one-launch train kernel: 3.6x below 0.5, kept), d hid 0.98,
# gradients 4.8.
# edge (igmc_edge_grad per directed edge, tests/test_gpu_edge_grad_bounds.py): largest 0.24, DGCNN_RS NB 2 k 30 seeded
# by the kernel's own dstate; IGMC cases 0.0001 to 0.15.  dstate (igmc_sortpool_backward seeded with 1): largest 0.51.
# Both are far below one u M because M carries the magnitude pass's d pre, which bounds the kernel's own d pre error
# and is far above |d pre|.  For the same reason a TF32-truncated h moves the edge ratio by only ~1 to 5 (numpy
# emulation in tests/test_error_bounds_oracle.py): the edge bound catches a lost 1/|segment|, a wrong segment or a
# missing layer by 500x and more, but not reliably a TF32 slip in h (the EG pass has no tensor-core path today).
# The regime cases (tests/test_gpu_regime_bounds.py: relation counts 1..11, 1 to 8 layers on every plan family,
# degenerate batches, staging limits, readout variants) and the train engine's steps (tests/test_gpu_engine_bounds.py),
# same H100 and power limit, stay inside these constants: states 9.1 (L 5, plan 0), predictions 0.41 (the engine's
# third step after a resume at step 5000), d hid 0.99, gradients 11.0 (one 202-node pair on plan 4).
# adam (k_adam and the fused update, per element of m, v and p; M in adam_terms): largest 3.3 (v, first step after
# the resume), m 1.9, p 1.7; numpy fp32 emulation 1.9.  An off-by-one step in the bias corrections (steps 1 to 3), weight
# decay left out or eps inside the square root is off by 2 000 to 16 000 000 u M.
# wprep (prepared W_r / W_r^T slabs after a fused update; M = sum_b |att| |basis|): largest 2.8, emulation 1.9; a
# TF32-rounded basis is off by ~10 000, a dropped basis by ~10^7.  Root columns are copies (exact) and padding is 0.
KAPPA = dict(states=64, pred=0.5, dhid=4, grad=32, edge=1, dstate=4, adam=16, wprep=16)


class Graph:
    """one collated batch (an oracle ``extract_batch`` dict) in fp64, edge dropout applied by ``edge_keep``"""

    def __init__(self, ob, edge_keep=None):
        self.x = torch.as_tensor(ob["x"]).double()
        ei = torch.as_tensor(ob["edge_index"]).long()
        et = torch.as_tensor(ob["edge_type"]).long()
        if edge_keep is not None:
            keep = torch.as_tensor(edge_keep).bool()
            ei, et = ei[:, keep], et[keep]
        self.edge_index, self.edge_type = ei, et
        self.users, self.items = self.x[:, 0] == 1, self.x[:, 1] == 1
        self.num_graphs = int(ob["num_graphs"])
        counts = torch.bincount(torch.as_tensor(ob["batch"]).long(), minlength=self.num_graphs)
        self.node_ptr = torch.cat([torch.zeros(1, dtype=torch.long), torch.cumsum(counts, 0)])


def conv_names(params):
    """state_dict suffixes of the [R,NB], [NB,in,out], [in,out], [out] parameters of a conv layer"""
    return ("att", "basis", "root", "bias") if any(k.endswith(".att") for k in params) else \
        ("comp", "weight", "root", "bias")


def _conv(att, basis, root, bias, aggr):
    """the restated conv with the given tensors in place of its parameters (autograd flows into them)"""
    from tests import pyg2_oracle
    NB, fin, fout = basis.shape
    with torch.random.fork_rng(devices=[]):      # construction draws an init; keep the caller's RNG stream
        c = pyg2_oracle.RGCNConvRelMeanRef(fin, fout, att.shape[0], NB, aggr)
    for name, t in (("att", att), ("basis", basis), ("root", root), ("bias", bias)):
        delattr(c, name)
        setattr(c, name, t)
    c.formulation = "transform"
    return c


def layer_pre(h, p4, g, aggr):
    """pre-activation of one conv layer: mean aggregate of h W_r + h root + bias"""
    return _conv(*p4, aggr)(h, g.edge_index, g.edge_type)


def head(cs, P, g, saved, dgcnn, parts=None):
    """readout of the concatenated states ``cs`` up to the lin2 output (before ``multiply_by``), on the kernel's
    branches: IGMC target rows -> lin1 -> ReLU / dropout (``gscale``) -> lin2; DGCNN_RS SortPooling in the kernel's
    order (``perm``) -> conv1 -> ReLU (``act1 > 0``) -> MaxPool (argmax of ``act1``) -> conv2 -> ReLU (``flat > 0``) ->
    lin1 -> ReLU / dropout -> lin2.  ``parts`` (a dict) receives the arguments of those branches: the pre-activations
    "conv1", "conv2" and "lin1" """
    parts = {} if parts is None else parts
    if not dgcnn:
        z = torch.cat([cs[g.users], cs[g.items]], 1)
    else:
        perm, act1, flat = saved["perm"], saved["act1"], saved["flat"]
        B, k = perm.shape
        W = cs.shape[1]
        rows = cs[perm.clamp(min=0)] * (perm >= 0).unsqueeze(-1).to(cs.dtype)      # padding rows are zero
        a1 = F.conv1d(rows.reshape(B, 1, k * W), P["conv1d_params1.weight"], P["conv1d_params1.bias"], stride=W)
        parts["conv1"] = a1
        a1 = a1 * (act1 > 0).to(cs.dtype)
        t1 = k // 2
        arg = (act1[..., 1:2 * t1:2] > act1[..., 0:2 * t1:2]).long()           # first maximum wins
        pool = a1.gather(2, 2 * torch.arange(t1).view(1, 1, t1) + arg)
        a2 = F.conv1d(pool, P["conv1d_params2.weight"], P["conv1d_params2.bias"])
        parts["conv2"] = a2
        z = (a2 * (flat.view(a2.shape) > 0).to(cs.dtype)).reshape(B, -1)
    parts["lin1"] = z @ P["lin1.weight"].t() + P["lin1.bias"]
    hid = parts["lin1"] * saved["gscale"]
    return hid @ P["lin2.weight"][0] + P["lin2.bias"][0]


def _readout_keys(params):
    return [k for k in params if not k.startswith("convs.")]


def _prep(params, saved, mag):
    A = torch.abs if mag else (lambda t: t)
    P = {k: A(v) for k, v in params.items()}
    states = [A(h) for h in saved["states"]]
    return A, P, states


def forward(params, g, saved, aggr, dgcnn, mag=False):
    """(per-layer pre-activations from the kernel's own inputs, readout output before multiply_by)"""
    A, P, states = _prep(params, saved, mag)
    names = conv_names(params)
    with torch.no_grad():
        pres = [layer_pre(g.x if l == 0 else states[l - 1], [P["convs.%d.%s" % (l, n)] for n in names], g, aggr)
                for l in range(len(states))]
        out = head(torch.cat(states, 1), P, g, saved, dgcnn)
    return pres, out


def _arr_dW(W, arr, mag):
    """d (arr * sum_r ||W_{r+1} - W_r||^2) / d W; the magnitude pass adds where the value subtracts"""
    s = 1.0 if mag else -1.0
    D = torch.zeros_like(W)
    D[1:] += W[1:] + s * W[:-1]
    D[:-1] += W[:-1] + s * W[1:]
    return 2.0 * arr * D


def _readout_vjp(P, states, g, saved, dgcnn, dpred, keys):
    """(d concat_states, [d P[k] for k in keys]) of the readout output weighted by ``dpred``, on the kernel's branches"""
    cs = torch.cat(states, 1).requires_grad_(True)
    gr = torch.autograd.grad(head(cs, P, g, saved, dgcnn), [cs] + [P[k] for k in keys], dpred)
    return gr[0], list(gr[1:])


def readout_dstate(params, g, saved, dgcnn, mag=False):
    """d (readout output . dpred) / d concat_states [N, total width]: what igmc_sortpool_backward writes to ``dstate``
    (DGCNN_RS, seeded with ``dpred``)"""
    A, P, states = _prep(params, saved, mag)
    with torch.enable_grad():
        return _readout_vjp(P, states, g, saved, dgcnn, A(saved["dpred"]), [])[0]


def backward(params, g, saved, aggr, dgcnn, arr, mag=False, dpres=None, dstate=None):
    """(d hid [B,128], parameter gradients by state_dict name) of the loss whose lin2-output gradient is the kernel's
    ``dpred``, plus the ARR term: per-layer vector-Jacobian products from the readout down to layer 0.  ``dpres``: a
    list that receives d pre_l of every layer, in layer order.  ``dstate``: d concat_states [N, total width] to start
    from in place of the readout's VJP (the kernel's ``S.dstate`` of an external readout); the readout's gradients are
    then left out and d hid is None"""
    A, P0, states = _prep(params, saved, mag)
    P = {k: v.detach().clone().requires_grad_(True) for k, v in P0.items()}
    names = conv_names(params)
    L = len(states)
    rk = _readout_keys(params)
    if dstate is None:
        dcs, gr = _readout_vjp(P, states, g, saved, dgcnn, A(saved["dpred"]), rk)
        grads = dict(zip(rk, gr))
    else:
        dcs, grads = A(dstate), {}
    dh = list(torch.split(dcs, [h.shape[1] for h in states], 1))
    for l in reversed(range(L)):
        h = saved["states"][l]
        dpre = dh[l] * (1.0 - h * h)
        if dpres is not None:
            dpres.insert(0, dpre)
        keys = ["convs.%d.%s" % (l, n) for n in names]
        hin = g.x if l == 0 else states[l - 1].clone().requires_grad_(True)
        pre = layer_pre(hin, [P[k] for k in keys], g, aggr)
        gr = torch.autograd.grad(pre, [P[k] for k in keys] + ([hin] if l else []), dpre)
        grads.update(zip(keys, gr[:4]))
        if l:
            dh[l - 1] = dh[l - 1] + gr[4]
        if arr:
            att, basis = P[keys[0]], P[keys[1]]
            W = torch.einsum("rb,bio->rio", att, basis)
            ga, gb = torch.autograd.grad(W, [att, basis], _arr_dW(W.detach(), arr, mag))
            grads[keys[0]] = grads[keys[0]] + ga
            grads[keys[1]] = grads[keys[1]] + gb
    if dstate is not None:
        return None, grads
    dhid = A(saved["dpred"]).unsqueeze(1) * A(params["lin2.weight"])[0] * saved["gscale"]
    return dhid, grads


def edge_terms(params, g, saved, aggr, dgcnn, mag=False):
    """d (sum of the scores) / d w_e at w = 1 of every directed edge e = j -> v of type r [E] (the edge weights of
    tests/edge_weight_oracle.py): the closed form of ``centred_edge_grad`` from the kernel's own inputs, summed over
    the layers l of

        (s_e - mean of s over e's segment) / |segment|,     s_e = <h_{l-1}[j] W_r, d pre_l[v]>,

    the segment v's in-edges (mean_all) or v's in-edges of type r (mean_per_relation).  d pre_l comes from
    ``backward`` seeded with the kernel's ``dpred`` (IGMC: d score / d lin2 output, ``multiply_by``) or, for DGCNN_RS,
    with its ``dstate`` (``saved["dstate"]``, true widths) at the concat states.  The magnitude pass sums
    (|s|_e + mean of |s| over the segment) / |segment|, |s| from |h|, |att|, |basis| and the magnitude pass's d pre:
    an error the kernel carries in its own d pre is covered by M too"""
    dpres = []
    backward(params, g, saved, aggr, dgcnn, 0.0, mag, dpres, saved["dstate"] if dgcnn else None)
    A, P, states = _prep(params, saved, mag)
    att, basis = conv_names(params)[:2]
    src, dst = g.edge_index
    et = g.edge_type
    R = P["convs.0." + att].shape[0]
    per_rel = aggr == "mean_per_relation"
    seg = dst * R + et if per_rel else dst
    nseg = g.x.shape[0] * (R if per_rel else 1)
    cnt = torch.zeros(nseg, dtype=torch.float64).index_add_(0, seg, torch.ones(len(seg), dtype=torch.float64))[seg]
    out = torch.zeros(len(seg), dtype=torch.float64)
    with torch.no_grad():
        for l, dp in enumerate(dpres):
            W = torch.einsum("rb,bio->rio", P["convs.%d.%s" % (l, att)], P["convs.%d.%s" % (l, basis)])
            h = A(g.x) if l == 0 else states[l - 1]
            s = (torch.einsum("ni,rio->nro", h, W)[src, et] * dp[dst]).sum(1)
            mean = torch.zeros(nseg, dtype=torch.float64).index_add_(0, seg, s)[seg] / cnt
            out += ((s + mean) if mag else (s - mean)) / cnt
    return out


def branch_mismatches(params, g, saved, dgcnn, hidden_keep=None):
    """the number of branches the kernel took against the fp64 value of their argument, counted only where that value
    is farther than KAPPA["states"] u M from the kink (closer than that, either side is correct): the lin1 ReLU
    (``gscale > 0`` iff pre-activation > 0 and the unit is kept by ``hidden_keep``), and for DGCNN_RS the conv1 ReLU
    (``act1``), the MaxPool side, the conv2 ReLU (``flat``) and the SortPooling order, which must be exactly the stable
    descending order of the kernel's own last-channel keys"""
    _, P, states = _prep(params, saved, False)
    _, MP, mstates = _prep(params, saved, True)
    parts, mparts = {}, {}
    with torch.no_grad():
        head(torch.cat(states, 1), P, g, saved, dgcnn, parts)
        head(torch.cat(mstates, 1), MP, g, saved, dgcnn, mparts)

    def wrong(kernel_side, ref, M, forced=None):
        """kernel_side: the branch taken (bool); forced: elements whose side is known without ref (dropped units)"""
        sure = ref.abs() > KAPPA["states"] * U * M
        want = ref > 0
        if forced is not None:
            sure, want = sure | forced, want & ~forced
        return int((kernel_side != want)[sure].sum())

    pre1 = parts["lin1"]
    dropped = torch.zeros_like(pre1, dtype=torch.bool) if hidden_keep is None else ~torch.as_tensor(hidden_keep).bool()
    bad = wrong(saved["gscale"] > 0, pre1, mparts["lin1"], dropped)
    if dgcnn:
        act1, a1, ma1 = saved["act1"], parts["conv1"], mparts["conv1"]
        bad += wrong(act1 > 0, a1, ma1)
        t1 = act1.shape[-1] // 2
        z = a1.clamp(min=0)
        odd, even = slice(1, 2 * t1, 2), slice(0, 2 * t1, 2)
        bad += wrong(act1[..., odd] > act1[..., even], z[..., odd] - z[..., even], ma1[..., odd] + ma1[..., even])
        bad += wrong(saved["flat"].view(parts["conv2"].shape) > 0, parts["conv2"], mparts["conv2"])
        key = torch.cat(saved["states"], 1)[:, -1]
        perm = saved["perm"]
        for gi, (lo, hi) in enumerate(zip(g.node_ptr[:-1].tolist(), g.node_ptr[1:].tolist())):
            order = lo + torch.sort(-key[lo:hi], stable=True).indices[:perm.shape[1]]
            want = torch.full_like(perm[gi], -1)
            want[:len(order)] = order
            bad += int((perm[gi] != want).sum())
    return bad


# ---- device side ----------------------------------------------------------------------------------------------------
def device_saved(m, ws, num_nodes, train):
    """the kernel's saved tensors of the last forward (and backward) of ``m`` on workspace ``ws``, on the host in fp64:
    per-layer states at their true widths, hidden dropout scales, dpred, and DGCNN_RS's SortPooling order and ReLU
    outputs"""
    st = ws["states"][:num_nodes].double().cpu()
    widths = [c.out_channels for c in m.convs]
    src = ws["sp"] if "sp" in ws else ws
    saved = dict(states=[st[:, 32 * l:32 * l + w] for l, w in enumerate(widths)], states_full=st,
                 gscale=src["hid_gscale"].double().cpu(), pred=src["pred"].double().cpu())
    if "sp" in ws:
        sp = ws["sp"]
        saved.update(perm=sp["perm"].long().cpu(), act1=sp["act1"].double().cpu(), flat=sp["flat"].double().cpu())
    if train:
        saved.update(dpred=ws["dpred"].double().cpu(), dhid=src["dhid"].double().cpu())
    return saved


def ratio(got, ref, M):
    """largest |got - ref| / (u M) over the elements with M > 0, and the number of elements with M == 0 where got is
    not exactly zero; also the flat index of the worst element.  A NaN or infinity anywhere (in got, or in ref or M
    from non-finite kernel inputs) gives an infinite ratio: it can never pass, and it hides no other element"""
    got, ref, M = got.reshape(-1).double(), ref.reshape(-1).double(), M.reshape(-1).double()
    zero = M == 0
    nonzero_pad = int((got[zero] != 0).sum())
    r = (got - ref).abs() / (U * M.clamp(min=1e-300))
    r[zero] = 0.0
    r[~(torch.isfinite(r) & torch.isfinite(got))] = float("inf")
    worst = int(r.argmax()) if r.numel() else -1
    return (float(r.max()) if r.numel() else 0.0), nonzero_pad, worst


def _pad32(t, w):
    return F.pad(t, (0, w - t.shape[1]))


def check_device(m, ob, ws, train, edge_keep=None, arr=0.0, hidden_keep=None, params=None):
    """every quantity of the last forward (eval) or train step of ``m`` on the oracle batch ``ob`` against its fp64
    recomputation; returns {quantity: (largest err / (u M), elements that must be zero but are not, worst index)} and
    under "branches" the count of ``branch_mismatches`` (``edge_keep`` / ``hidden_keep``: the step's dropout draws).
    ``params``: the state_dict the step ran with (default ``m``'s current one; pass a snapshot when an optimizer
    update has changed the parameters since)"""
    if params is None:
        params = m.state_dict()
    params = {k: v.detach().double().cpu().contiguous() for k, v in params.items()}
    dgcnn = "sp" in ws
    aggr = "mean_per_relation" if m.rgcn == "pyg-2" else "mean_all"
    N = ob["x"].shape[0]
    g = Graph(ob, edge_keep if train else None)
    saved = device_saved(m, ws, N, train)
    pres, out = forward(params, g, saved, aggr, dgcnn)
    mpres, mout = forward(params, g, saved, aggr, dgcnn, mag=True)
    res = dict(branches=branch_mismatches(params, g, saved, dgcnn, hidden_keep if train else None))
    for l, (pre, mpre) in enumerate(zip(pres, mpres)):
        got = saved["states_full"][:, 32 * l:32 * l + 32]
        h = saved["states"][l]
        res["states%d" % l] = ratio(got, _pad32(torch.tanh(pre), 32), _pad32((1 - h * h) * mpre + h.abs(), 32))
    mult = float(m.multiply_by)
    res["pred"] = ratio(saved["pred"], out * mult, mout * abs(mult))
    if train:
        dhid, grads = backward(params, g, saved, aggr, dgcnn, arr)
        mdhid, mgrads = backward(params, g, saved, aggr, dgcnn, arr, mag=True)
        res["dhid"] = ratio(saved["dhid"], dhid, mdhid)
        names = {id(p): n for n, p in m.named_parameters()}
        fg = m.flat_grad.double().cpu()
        got, ref, M = [], [], []
        for e, (_, _, p) in zip(m._layout, m._named_order()):
            o, n, s = e[:3]
            full = e[3] if len(e) == 4 else s
            name = names[id(p)]
            r, mm = torch.zeros(full, dtype=torch.float64), torch.zeros(full, dtype=torch.float64)
            r[..., :s[-1]] = grads[name].reshape(s)
            mm[..., :s[-1]] = mgrads[name].reshape(s)
            got.append(fg[o:o + n])
            ref.append(r.reshape(-1))
            M.append(mm.reshape(-1))
        res["grad"] = ratio(torch.cat(got), torch.cat(ref), torch.cat(M))
    return res


def kappa_of(key):
    """the KAPPA entry that bounds result ``key`` (states0..7 -> states, adam_m / adam_v / adam_p -> adam,
    wprep_root -> wprep)"""
    return KAPPA[next((k for k in ("states", "adam", "wprep") if key.startswith(k)), key)]


def violations(res):
    """the entries of a ``check_device`` result that fail: a ratio not within its KAPPA (NaN included), an element that
    must be zero and is not, or a branch mismatch"""
    bad = [("branches", res.get("branches", 0))] if res.get("branches", 0) else []
    for key, val in res.items():
        if key == "branches":
            continue
        r, pad, worst = val
        if not r <= kappa_of(key) or pad:
            bad.append((key, r, pad, worst))
    return bad


# ---- optimizer and prepared weights ---------------------------------------------------------------------------------
def f32(x):
    """a hyperparameter as the kernels receive it (a float argument), in fp64"""
    return float(torch.tensor(float(x), dtype=torch.float32))


def adam_terms(p, m, v, g, step, lr, b1, b2, eps, wd, grad_mul=1.0):
    """one torch-Adam update (k_adam and phase 3 of k_reduce_allreduce_adam: eps outside the square root, L2 weight
    decay added to the gradient) in fp64 from the state before the step (``p``, ``m``, ``v``), the gradient it applied
    (``g``, before ``grad_mul``) and the step number it ran as (``step``, counted from 1), with the bias corrections
    1 - beta^step in fp64.  Hyperparameters are taken at fp32, as the kernel receives them.

    Returns {"adam_m" | "adam_v" | "adam_p": (reference, M)}.  M sums the magnitudes of the terms: for the moments
    b1 |m| + (1 - b1) |g'| and b2 v + (1 - b2) |g'|^2 with |g'| = |g grad_mul| + |wd p|; for the parameter |p| + |dp|
    plus the first-order effect of the moments' own bounds on dp = lr/bc1 * m / (sqrt(v / bc2) + eps):
    lr/bc1 * M_m / den + |dp| M_v / (2 v)."""
    p, m, v, g = [t.double() for t in (p, m, v, g)]
    lr, b1, b2, eps, wd, grad_mul = [f32(x) for x in (lr, b1, b2, eps, wd, grad_mul)]
    gg = g * grad_mul + wd * p
    Mg = (g * grad_mul).abs() + abs(wd) * p.abs()
    m1 = b1 * m + (1 - b1) * gg
    v1 = b2 * v + (1 - b2) * gg * gg
    Mm = b1 * m.abs() + (1 - b1) * Mg
    Mv = b2 * v.abs() + (1 - b2) * Mg * Mg
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    den = torch.sqrt(v1) / bc2 ** 0.5 + eps
    dp = (lr / bc1) * m1 / den
    Mp = p.abs() + dp.abs() + (lr / bc1) * Mm / den + dp.abs() * torch.where(v1 > 0, Mv / (2 * v1.clamp(min=1e-300)),
                                                                             torch.zeros_like(v1))
    return {"adam_m": (m1, Mm), "adam_v": (v1, Mv), "adam_p": (p - dp, Mp)}


def adam_check(got, terms):
    """{key: ratio(...)} of the device's updated (exp_avg, exp_avg_sq, params) against ``adam_terms``"""
    return {key: ratio(g, *terms[key]) for key, g in zip(("adam_m", "adam_v", "adam_p"), got)}


def wprep_terms(params, L, R, in0):
    """the prepared weight slabs (igmc_prep_weights, phase 4 of k_reduce_allreduce_adam) of ``params`` (a state_dict)
    in fp64: slab (l, dir) holds 32 rows of KS = K1p + a8(inp) + 4 floats, inp = a4(in), K1 = R inp, K1p = a8(K1);
    dir 0 row n: W_r[q][n] at r inp + q, root[q][n] at K1p + q; dir 1 (layers >= 1) row k: W_r[k][q] at r inp + q,
    root[k][q] at K1p + q; every other float of a row is 0.  W_r = sum_b att[r,b] basis[b].

    Returns (reference, M, copied, written) as flat tensors over the whole buffer: M = sum_b |att[r,b]| |basis[b]|,
    ``copied`` marks the root entries (copied, so exact), ``written`` every float some row covers (slab (0, 1) and
    the tail of the layer-0 slabs are not written)."""
    a4 = lambda x: (x + 3) & ~3      # noqa: E731
    a8 = lambda x: (x + 7) & ~7      # noqa: E731
    att_n, basis_n = conv_names(params)[:2]
    slab = 32 * ((R + 1) * 32 + 4)
    ref = torch.zeros(L * 2 * slab, dtype=torch.float64)
    M, copied, written = torch.zeros_like(ref), torch.zeros_like(ref, dtype=torch.bool), torch.zeros_like(ref, dtype=torch.bool)
    for l in range(L):
        at = params["convs.%d.%s" % (l, att_n)].double()
        bs = params["convs.%d.%s" % (l, basis_n)].double()
        rt = params["convs.%d.root" % l].double()
        bs, rt = F.pad(bs, (0, 32 - bs.shape[2])), F.pad(rt, (0, 32 - rt.shape[1]))    # a narrow last layer
        fin = bs.shape[1]
        inp = a4(fin)
        K1p = a8(R * inp)
        KS = K1p + a8(inp) + 4
        W = torch.einsum("rb,bio->rio", at, bs)                 # [R, in, 32]
        MW = torch.einsum("rb,bio->rio", at.abs(), bs.abs())
        for d in (0, 1) if l else (0,):
            rows = torch.zeros(32, KS, dtype=torch.float64)
            mrows, crows = torch.zeros_like(rows), torch.zeros_like(rows, dtype=torch.bool)
            # [32 rows, R, in]: dir 0 row n, column (r, q) = W_r[q][n]; dir 1 row k, column (r, q) = W_r[k][q]
            order = (2, 0, 1) if d == 0 else (1, 0, 2)
            rows[:, :R * inp].view(32, R, inp)[:, :, :fin] = W.permute(*order)
            mrows[:, :R * inp].view(32, R, inp)[:, :, :fin] = MW.permute(*order)
            rows[:, K1p:K1p + fin] = rt.t() if d == 0 else rt
            crows[:, K1p:K1p + fin] = True
            o = (l * 2 + d) * slab
            ref[o:o + 32 * KS] = rows.reshape(-1)
            M[o:o + 32 * KS] = mrows.reshape(-1)
            copied[o:o + 32 * KS] = crows.reshape(-1)
            written[o:o + 32 * KS] = True
    return ref, M, copied, written


def wprep_check(got, terms):
    """{"wprep": ratio of the W_r entries and padding, "wprep_root": (0, root entries not copied exactly, -1)}"""
    ref, M, copied, written = terms
    got = got.reshape(-1).double().cpu()
    sel = written & ~copied
    miss = int((got[copied] != ref[copied]).sum())
    return {"wprep": ratio(got[sel], ref[sel], M[sel]), "wprep_root": (0.0, miss, -1)}
