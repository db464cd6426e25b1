"""Shared loaders for tests/golden, the train-step parity check and the kernel-regime shapes of the test suite."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = ("u_nodes", "v_nodes", "u", "v", "r", "node_labels")


def load_random_cases():
    """Yield dict(tag, A (scipy csr), pairs, cv, h, ratio, mnph, cases=[canonical dicts])."""
    from igmc_b200.data import build_adj
    z = np.load(os.path.join(GOLDEN, "random_cases.npz"))
    out = []
    for tag in z["tags"]:
        tag = str(tag)
        nu, nv, R, h, mnph = [int(x) for x in z[tag + "__shape"]]
        A = build_adj(z[tag + "__coo_u"], z[tag + "__coo_v"], z[tag + "__coo_l"], nu, nv)
        n = z[tag + "__pairs"].shape[1]
        cases = []
        for c in range(n):
            d = {}
            for k in KEYS:
                off = z["%s__%s_off" % (tag, k)]
                d[k] = z["%s__%s" % (tag, k)][off[c]:off[c + 1]]
            d["y"] = float(z[tag + "__y"][c])
            cases.append(d)
        out.append(dict(tag=tag, A=A, pairs=z[tag + "__pairs"], cv=z[tag + "__cv"], h=h,
                        ratio=float(z[tag + "__ratio"]), mnph=None if mnph < 0 else mnph,
                        R=R, cases=cases))
    return out


def injected_sampler(case):
    """sampler(cands, k, side, hop) returning the reference's recorded draw for a golden case."""
    n_u = len(case["u_nodes"])
    labels = case["node_labels"]
    ud, vd = labels[:n_u] // 2, (labels[n_u:] - 1) // 2

    def smp(cands, k, side, hop):
        nodes, dist = (case["u_nodes"], ud) if side == 0 else (case["v_nodes"], vd)
        sel = nodes[dist == hop]
        assert len(sel) == k and set(sel.tolist()) <= set(np.asarray(cands).tolist())
        return sel
    return smp


def oracle_collated(group, sampler_from_cases=True, seed=0):
    """numpy-oracle collate of every pair of a golden group (h must be 1)."""
    from oracle import extract_np
    g = extract_np.RatingCSR(group["A"])
    pu, pv, pl = group["pairs"]
    smp = None
    if sampler_from_cases:
        samplers = [injected_sampler(c) for c in group["cases"]]
        smp = lambda k, cands, kk, side, hop: samplers[k](cands, kk, side, hop)  # noqa: E731
    return extract_np.extract_batch(g, pu, pv, pl, group["cv"].astype(np.float32), group["h"], group["ratio"],
                                    group["mnph"], sampler=smp, seed=seed)


def inject_arrays(cases, cap):
    """golden canonical node lists -> padded [B,cap] int32 arrays for SubgraphExtractor.extract(inject=...)."""
    B = len(cases)
    nu = np.zeros((B, cap), np.int32)
    nv = np.zeros((B, cap), np.int32)
    cu = np.zeros(B, np.int32)
    cvv = np.zeros(B, np.int32)
    for k, c in enumerate(cases):
        cu[k], cvv[k] = len(c["u_nodes"]), len(c["v_nodes"])
        nu[k, :cu[k]] = c["u_nodes"]
        nv[k, :cvv[k]] = c["v_nodes"]
    return nu, nv, cu, cvv


def batch_equal(b, ob):
    """compare an igmc_b200 Batch with an oracle collated dict, bit-exact on every integer field."""
    import torch
    out = {}
    out["x"] = np.array_equal(b.x.cpu().numpy(), ob["x"])
    out["edge_index"] = np.array_equal(b.edge_index.cpu().numpy(), ob["edge_index"])
    out["edge_type"] = np.array_equal(b.edge_type.cpu().numpy(), ob["edge_type"])
    out["batch"] = np.array_equal(b.batch.cpu().numpy(), ob["batch"])
    out["y"] = np.array_equal(b.y.cpu().numpy(), ob["y"].astype(np.float32))
    out["node_label"] = np.array_equal(b.node_label.cpu().numpy().astype(np.int64), ob["node_labels"])
    return out


# ---- staging regimes of the relation-space kernels (csrc/rgcn_rs.cu) and the shapes that pin them -------------------
# Constants restated from csrc/rgcn_rs.cu: edges per segment, extra staging rows per chunk, chunks that may use extra
# rows, destination nodes per warp group (the granularity of a CTA's node range), list-image header ints.
SEG, XR, XCH, GN, IMG_HDR = 32, 16, 8, 4, 4

# name -> shape of one regime test in tests/test_gpu_regimes.py.  ``own``: the own-node count of the CTA that enters
# the regime in that test's batch (its subgraphs are built so that some CTA reaches it; the GPU test asserts that).
REGIMES = {
    # backward chunks with index >= XCH get no extra segment rows (stage_lists: allowed = ci < XCH ? ... : 0)
    "bwd_chunks_past_xch": dict(R=12, in0=4, n_cap=202, plan=1, own=200),
    # layer-0 weight gradient in several tile passes (backward_body, layer-0 branch: t0 > 0)
    "layer0_tile_passes_in4": dict(R=12, in0=4, n_cap=202, plan=1, own=200),
    "layer0_tile_passes_in8": dict(R=12, in0=8, n_cap=202, plan=1, own=180),
    # backward lists read from global memory (Ls.lst == nullptr) while the forward's lists are staged: in-entries of
    # the two CTAs of a 101 x 101 fully rated block (every CTA between ``entries`` bounds after 20 % edge dropout)
    "fwd_staged_bwd_global": dict(R=5, in0=4, n_cap=202, plan=2, entries=(7400, 10600)),
    # eval-mode forward lists read from global memory: without dropout every in-entry of a pair inside that block counts
    # (101 x 101 - 1 ratings, both directions), all on the one CTA of plan 1 - beyond the forward's list capacity
    "fwd_global_eval": dict(R=5, in0=4, n_cap=202, plan=1, entries=20400),
    # the same at mnph 200 after a sparse first batch set list_hint: a pair inside a fully rated 201 x 201 block has
    # 90-104 own nodes with ~201 in-entries each on every CTA of plan 4, above the largest list capacity any hint buys
    "fwd_global_eval_hinted": dict(R=5, in0=4, n_cap=402, plan=4, entries=18000),
    # CTAs of a cluster that own no node (forward / backward n_own == 0 branches): a 2-node subgraph at plan 4
    "ctas_without_nodes": dict(R=5, in0=4, n_cap=202, plan=4, n=2),
}


def a4(x):
    return (x + 3) & ~3


def a8(x):
    return (x + 7) & ~7


def own_cap_of(n_cap, cluster):
    """most nodes one CTA of a ``cluster``-CTA plan owns (own_cap_of in csrc/rgcn_rs.cu)"""
    per = (n_cap + cluster - 1) // cluster
    return (per + GN - 1) // GN * GN


def own_counts(n, cluster):
    """own-node count of every CTA of a cluster for an ``n``-node subgraph (own_range in csrc/rgcn_rs.cu)"""
    per = own_cap_of(n, cluster)
    return [min(n, (r + 1) * per) - min(n, r * per) for r in range(cluster)]


def layer0_tile_rows(R, in0, bwd_chunk):
    """node rows of one layer-0 weight-gradient tile pass (``trows`` in backward_body): the pass reuses the staging
    rows (chunk + XR rows of R*32+4 floats) as a tile of KRp + 8 floats per node."""
    inp = a4(in0)
    KRp = a8(R * inp) + a8(inp)
    return ((bwd_chunk + XR) * (R * 32 + 4) // (KRp + 8)) & ~7


def image_tables(tab_row, n_cap, cluster):
    """(list lengths, extra-segment counts) of the own nodes of one list image row (``tab[blk]`` after
    ``IGMC.stage_batch``): the header is followed by lptr[own_cap+4], segbase[own_cap+4], ex[own_cap+4]."""
    import numpy as np
    t = np.asarray(tab_row)
    n_own, oc = int(t[3]), own_cap_of(n_cap, cluster)
    lptr = t[IMG_HDR:IMG_HDR + n_own + 1]
    ex = t[IMG_HDR + 2 * (oc + 4):IMG_HDR + 2 * (oc + 4) + n_own]
    return np.diff(lptr), ex >> 16


def oracle_train_step(ref, ob, ARR, edge_keep, hidden_keep):
    """fp64 autograd of one train step of the restated oracle ``ref`` (IGMCRef or DGCNN_RSRef, train mode) on the
    collated oracle batch ``ob``: fills the parameters' ``.grad`` and returns (loss, predictions)."""
    import torch
    from oracle import pyg_restated
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    ref.zero_grad()
    if isinstance(ref, pyg_restated.DGCNN_RSRef):
        out = ref(tb["x"], tb["edge_index"], tb["edge_type"], tb["batch"], edge_keep, hidden_keep, tb["num_graphs"])
        loss = torch.nn.functional.mse_loss(out, tb["y"].view(-1))
        if ARR != 0:
            loss = loss + ARR * pyg_restated.arr_regulariser(ref)
    else:
        loss, out = pyg_restated.train_loss(ref, tb, ARR, edge_keep, hidden_keep)
    loss.backward()
    return loss.detach(), out.detach()


def assert_step_matches(m, ref, pred, loss, grad, loss_ref, out_ref, tag="step"):
    """a train step of ``m`` (device predictions ``pred``, loss ``loss``, flat gradient ``grad`` in ``m``'s layout)
    against the oracle's (``loss_ref``, ``out_ref`` and ``ref``'s parameter ``.grad``): predictions within 1e-4 RMSE, the
    loss within 1e-4 relative and every parameter gradient within 2e-4 of the largest entry of that tensor's reference
    gradient (DGCNN_RS: 3e-4 of it + 2e-6 of the largest entry of any tensor, the bar of tests/test_gpu_full_batch.py:
    its first-layer att gradients cancel to ~1e-3 of the largest).  Returns (prediction RMSE, worst gradient error in
    units of the relative bar's scale)."""
    import torch
    from oracle import pyg_restated
    rmse = float(torch.sqrt(torch.mean((pred.double().cpu() - out_ref.detach()) ** 2)))
    assert rmse <= 1e-4, (tag, rmse)
    assert abs(float(loss) - float(loss_ref)) <= 1e-4 * max(1.0, abs(float(loss_ref))), (tag, float(loss),
                                                                                         float(loss_ref))
    names = {id(p): n for n, p in m.named_parameters()}
    sd_ref = dict(ref.named_parameters())
    table = []
    for e, (_, _, p) in zip(m._layout, m._named_order()):
        gref = sd_ref[names[id(p)]].grad
        table.append((names[id(p)], float((m._pview(grad, e).double().cpu() - gref).abs().max()),
                      float(gref.abs().max())))
    worst = 0.0
    if isinstance(ref, pyg_restated.DGCNN_RSRef):
        gmax = max(t[2] for t in table)
        for name, err, scale in table:
            assert err <= 3e-4 * scale + 2e-6 * gmax, (tag, name, err, scale, gmax)
            worst = max(worst, err / (scale + gmax / 150.0))
    else:
        for name, err, scale in table:
            rel = err / (scale + 1e-12)
            assert rel <= 2e-4, (tag, name, rel)
            worst = max(worst, rel)
    print("%s: prediction RMSE %.2e, worst relative gradient error %.2e" % (tag, rmse, worst))
    return rmse, worst


def check_step(m, ref, b, ob, ARR, adj_dropout, hk, step=30, edge_keep=None):
    """One ``fused_step`` of ``m`` on batch ``b`` against fp64 autograd of the restated oracle ``ref`` on the collated
    oracle batch ``ob`` (bars: ``assert_step_matches``).  The edge dropout is the kernels' own hash draw of step
    ``step + 1`` unless ``edge_keep`` injects one; so is the hidden dropout when ``hk`` is None (the oracle then gets
    the host twin's mask).  Returns (prediction RMSE, worst relative gradient error)."""
    from igmc_b200.models import edge_keep_reference, hidden_keep_reference, splitmix64
    E, B = ob["edge_index"].shape[1], ob["num_graphs"]
    m._step = step
    seed = splitmix64(m.drop_seed + step + 1)          # fused_step draws after its _step += 1
    ek = edge_keep
    if ek is None and adj_dropout > 0:
        ek = edge_keep_reference(seed, E, adj_dropout)
    hk_ref = hk if hk is not None else hidden_keep_reference(seed, B, m.hidden_dropout_p)
    loss_ref, out_ref = oracle_train_step(ref, ob, ARR, ek, hk_ref)
    loss = m.fused_step(b, ARR=ARR, hidden_keep=hk, edge_keep=edge_keep)
    b.check()
    assert m._step == step + 1
    ws = next(iter(v for k, v in m._ws.items() if k[2] and k[1] == B))
    pred = ws["sp"]["pred"] if "sp" in ws else ws["pred"]
    return assert_step_matches(m, ref, pred, loss, m.flat_grad, loss_ref, out_ref, "check_step")


def load_flixster_cases():
    """(dataset dict, pairs [3,n], list of canonical dicts) of tests/golden/flixster_cases.npz: outputs of the
    reference's own subgraph_extraction_labeling on 64 pairs of the REAL flixster split (h=1, no sampling)."""
    from igmc_b200.data import load_flixster
    ds = load_flixster()
    z = np.load(os.path.join(GOLDEN, "flixster_cases.npz"))
    cases = []
    for c in range(z["pairs"].shape[1]):
        d = {k: z[k][z[k + "_off"][c]:z[k + "_off"][c + 1]] for k in KEYS}
        d["y"] = float(z["y"][c])
        cases.append(d)
    return ds, z["pairs"], cases
