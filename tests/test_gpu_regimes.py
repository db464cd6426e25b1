"""Train-step parity in every regime the relation-space kernels (csrc/rgcn_rs.cu) and the generic kernels
(csrc/rgcn.cu) branch on: multi-hop input widths, relation counts, staging limits, degenerate subgraphs, layer counts,
``multiply_by`` and the optimizer.

Every case runs one train step (the kernels' own hash dropout draws unless a case injects them) on a batch the CUDA
extractor built and that is first checked bit-exact against oracle/extract_np, then compares predictions, loss and
every parameter gradient with fp64 autograd of oracle/pyg_restated ("transform" formulation): ratings within 1e-4
RMSE, gradients within 2e-4 of the tensor's largest reference entry (tests/helpers.py check_step).  The staging
cases assert from the list images that they entered their regime; tests/test_regime_plans.py checks the same shapes
against the plans without a GPU."""
import functools

import numpy as np
import pytest
import torch

from igmc_b200.data import build_adj, make_synthetic_dataset, synth_ratings
from oracle import extract_np, pyg_restated
from tests.helpers import REGIMES, SEG, XCH, batch_equal, check_step, image_tables, layer0_tile_rows

pytestmark = pytest.mark.gpu


# ---- data ----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _ml_100k():
    return make_synthetic_dataset("ml_100k", seed=0)


def _dense(nu, nv, density, R, seed, u0=0, v0=0):
    """every (u, v) rated with probability ``density``, R uniform rating levels"""
    rng = np.random.default_rng(seed)
    u, v = np.nonzero(rng.random((nu, nv)) < density)
    return u + u0, v + v0, rng.integers(0, R, len(u))


def _matrix(parts, nu, nv):
    u, v, lab = [np.concatenate(p) for p in zip(*parts)]
    return build_adj(u, v, lab, nu, nv), (u, v, lab)


def _extracted(A, pairs, R, h, mnph, seed=3):
    """the CUDA extractor's batch of ``pairs`` (u, v, label) and the oracle's, asserted bit-exact"""
    from igmc_b200.util_functions import MyDynamicDataset
    pu, pv, pl = [np.asarray(x, np.int64) for x in pairs]
    cv = np.arange(1, R + 1, dtype=np.float32)
    d = MyDynamicDataset(None, A, (pu, pv), pl, h, 1.0, mnph, None, None, cv, seed=seed)
    idx = np.arange(len(pu))
    b = d.extract_batch(idx)
    ob = extract_np.extract_batch(extract_np.RatingCSR(A), pu, pv, pl, cv, h, 1.0, mnph, seed=seed, pair_ids=idx)
    res = batch_equal(b, ob)
    assert all(res.values()), res
    return b, ob


def _models(in0, R, NB=4, L=4, adj_dropout=0.2, plan="auto", multiply_by=1, dgcnn_k=None):
    from igmc_b200.models import DGCNN_RS, IGMC
    torch.manual_seed(0)
    if dgcnn_k is None:
        ref = pyg_restated.IGMCRef(in0, (32,) * L, R, NB, adj_dropout, multiply_by)
        m = IGMC(in0, latent_dim=[32] * L, num_relations=R, num_bases=NB, regression=True, adj_dropout=adj_dropout,
                 multiply_by=multiply_by)
    else:
        ref = pyg_restated.DGCNN_RSRef(in0, (32, 32, 32, 1), dgcnn_k, R, NB, adj_dropout)
        m = DGCNN_RS(in0, latent_dim=[32, 32, 32, 1], k=dgcnn_k, num_relations=R, num_bases=NB, regression=True,
                     adj_dropout=adj_dropout)
    ref = pyg_restated.set_formulation(ref.double().train(), "transform")
    m = m.cuda().train()
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    m.kernel_plan = plan
    return ref, m


def _hk(B, seed=2):
    return torch.rand(B, 128, generator=torch.Generator().manual_seed(seed)) > 0.5


def _images(m, b, step=30):
    """list images (host copies of the tables) the kernels of the step after ``m._step = step`` work on"""
    m._step = step + 1                  # fused_step draws its dropout with the seed of step + 1
    st = m.stage_batch(b, True, m.make_dropout(True))
    m._step = step
    return {k: t["tab"].cpu().numpy() for k, (img, t) in st.items()}, {k: img for k, (img, t) in st.items()}


def _restaged_step_bit_identical(m, b, hk, step=30):
    """the step just checked (self-staged lists) repeated on the list images of igmc_stage_lists: same gradient"""
    g0 = m.flat_grad.clone()
    _images(m, b, step)
    m.fused_step(b, ARR=0.001, hidden_keep=hk)
    b.check()
    b._stage = None
    assert torch.equal(m.flat_grad, g0)


def _paths_bit_identical(m, b, hk, monkeypatch, step=30):
    """two launches (igmc_forward + igmc_backward), one launch (igmc_forward_backward) self-staged and one launch on
    staged list images: bit-identical predictions, raw gradient rows, readout factors and assembled gradient"""
    got = []
    for fused, staged in (("0", False), ("1", False), ("1", True)):
        monkeypatch.setenv("IGMC_FUSED_FB", fused)
        b._stage = None
        if staged:
            _images(m, b, step)
        m._step = step
        m.flat_grad.zero_()
        saved = m.forward_backward(b, hidden_keep=hk)
        ws = saved["ws"]
        gpart = ws["gpart"].clone()
        m._launch_grad_reduce(b, saved, loss_scale=1.0 / b.num_graphs, arr=0.001)
        b.check()
        got.append((ws["pred"].clone(), gpart, ws["dhid"].clone(), m.flat_grad.clone()))
    b._stage = None
    for a, c in zip(got, got[1:]):
        for x, y in zip(a, c):
            assert torch.equal(x, y)


# ---- 1. input width x plan -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,mnph", [(2, 40), (3, 25)])
@pytest.mark.parametrize("plan", [0, 1, 2, 4])
def test_multi_hop_train_step(h, mnph, plan, monkeypatch):
    """layer-0 input width 6 (h = 2) and 8 (h = 3): the saved aggregate zsave is R * a4(in0) wide, the layer-0
    weight-gradient tile KRp, the one-hot columns start at K1p (backward_body layer-0 branch); plan 0 runs the generic
    kernels of csrc/rgcn.cu at that width"""
    ds = _ml_100k()
    tu, tv, tl = ds["train"]
    idx = np.array([0, 1, 2, 3])
    b, ob = _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, h, mnph)
    in0 = 2 * h + 2
    assert ob["x"].shape[1] == in0
    ref, m = _models(in0, 5, plan=plan)
    hk = _hk(len(idx))
    check_step(m, ref, b, ob, 0.001, 0.2, hk)
    assert m._plan(b) == plan
    if h == 2 and plan > 0:
        _paths_bit_identical(m, b, hk, monkeypatch)


# ---- 2. relation count ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,NB,plan", [(1, 2, 1), (1, 4, 2), (2, 4, 4), (2, 2, 2), (7, 4, 1), (7, 2, 2), (8, 4, 2),
                                       (8, 2, 4), (11, 4, 4), (11, 2, 2), (12, 4, 1), (12, 2, 2), (13, 4, "auto")])
def test_relation_count_train_step(R, NB, plan):
    """relation-space path for every R <= 12 (weight-gradient tiles in a second pass over the nodes from R = 8 on,
    num_bases > R at R = 1, 2), and R = 13 on the generic plan that "auto" must pick"""
    u, v, lab = synth_ratings(120, 90, 2500, num_classes=R, seed=3)
    A = build_adj(u, v, lab, 120, 90)
    B = 8
    b, ob = _extracted(A, (u[:B], v[:B], lab[:B]), R, 1, 30)
    ref, m = _models(4, R, NB=NB, plan=plan)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(B))
    assert m._plan(b) == (0 if R > 12 else plan)


# ---- 3. staging regimes --------------------------------------------------------------------------------------------
def test_bwd_chunks_past_xch_and_layer0_tile_passes():
    """R = 12, plan 1, n_cap 202, ~200-node subgraphs (dense 150 x 150 matrix, mnph 100):
    * backward chunks with index >= XCH get no extra segment rows, so a node's whole list (> SEG entries) is one
      long segment (stage_lists: ``allowed = ci < XCH ? ... : 0``);
    * the layer-0 weight gradient runs in several tile passes of ``trows`` node rows (backward_body layer-0 branch,
      ``t0 > 0``) and the weight-gradient column tiles in a second pass (R > 7)"""
    r = REGIMES["bwd_chunks_past_xch"]
    R = r["R"]
    A, (u, v, lab) = _matrix([_dense(150, 150, 0.75, R, 1)], 150, 150)
    pick = np.random.default_rng(0).choice(len(u), 4, replace=False)
    b, ob = _extracted(A, (u[pick], v[pick], lab[pick]), R, 1, 100)
    assert b._priv["n_cap"] == r["n_cap"]
    ref, m = _models(4, R, plan=r["plan"])
    hk = _hk(4)
    tabs, imgs = _images(m, b)
    bwd, chunk = tabs["bwd"], imgs["bwd"].chunk
    entered = False
    for row in bwd:
        lens, nex = image_tables(row, r["n_cap"], r["plan"])
        late = np.arange(len(lens)) >= XCH * chunk
        entered |= bool(np.any(late & (lens > SEG) & (nex == 0)))
    assert entered, "no backward node past chunk XCH with a list longer than one segment"
    assert int(bwd[:, 3].max()) >= r["own"]
    assert int(bwd[:, 3].max()) > layer0_tile_rows(R, 4, chunk)
    b._stage = None
    check_step(m, ref, b, ob, 0.001, 0.2, hk)
    _restaged_step_bit_identical(m, b, hk)


def test_layer0_tile_passes_at_input_width_8():
    """R = 12, plan 1, h = 3 (in0 = 8) on a dense 100 x 100 matrix: n_cap 202, ~200-node subgraphs, so the layer-0
    weight-gradient tile (KRp = 104 columns) holds fewer node rows than a CTA owns (backward_body layer-0 branch,
    several ``t0`` passes) while the one-hot input columns start at K1p = 96"""
    r = REGIMES["layer0_tile_passes_in8"]
    R = r["R"]
    A, (u, v, lab) = _matrix([_dense(100, 100, 0.5, R, 2)], 100, 100)
    pick = np.random.default_rng(1).choice(len(u), 3, replace=False)
    b, ob = _extracted(A, (u[pick], v[pick], lab[pick]), R, 3, 100)
    assert b._priv["n_cap"] == r["n_cap"] and ob["x"].shape[1] == r["in0"]
    ref, m = _models(r["in0"], R, plan=r["plan"])
    hk = _hk(3)
    tabs, imgs = _images(m, b)
    own = int(tabs["bwd"][:, 3].max())
    assert own >= r["own"] and own > layer0_tile_rows(R, r["in0"], imgs["bwd"].chunk)
    b._stage = None
    check_step(m, ref, b, ob, 0.001, 0.2, hk)
    _restaged_step_bit_identical(m, b, hk)


def _dense_block_matrix(R=5):
    """a fully rated 101 x 101 block (users 0..100 x items 0..100) whose users rate nothing else and whose items
    nobody else rates, next to a sparse 200 x 200 background"""
    blk = _dense(101, 101, 1.1, R, 3)
    bu, bv, bl = synth_ratings(200, 200, 3000, num_classes=R, seed=4)
    return _matrix([blk, (bu + 101, bv + 101, bl)], 301, 301)


def test_fwd_staged_bwd_global_lists():
    """R = 5, plan 2, mnph 100 (n_cap 202): a pair inside the dense block has a 202-node subgraph with ~10 200
    in-entries per CTA - within the forward's list capacity, beyond the backward's, so in the same step the forward
    gathers from staged lists and the backward from global memory with per-edge hash dropout (``Ls.lst == nullptr``)"""
    r = REGIMES["fwd_staged_bwd_global"]
    A, (u, v, lab) = _dense_block_matrix(r["R"])
    blk = np.nonzero((u < 101) & (v < 101))[0]
    bg = np.nonzero(u >= 101)[0]
    pick = np.array([blk[17], bg[0], blk[5000], bg[1]])
    b, ob = _extracted(A, (u[pick], v[pick], lab[pick]), r["R"], 1, 100)
    assert b._priv["n_cap"] == r["n_cap"]
    ref, m = _models(4, r["R"], plan=r["plan"])
    hk = _hk(4)
    tabs, _ = _images(m, b)
    f, w = tabs["fwd"], tabs["bwd"]
    assert np.any((f[:, 2] == 1) & (w[:, 2] == 0)), "no CTA with staged forward and global backward lists"
    lo, hi = r["entries"]
    assert np.all(w[w[:, 2] == 0, 0] >= lo) and np.all(f[:, 0] <= hi)
    b._stage = None
    check_step(m, ref, b, ob, 0.001, 0.2, hk)
    _restaged_step_bit_identical(m, b, hk)


# ---- 4. degenerate subgraphs ---------------------------------------------------------------------------------------
def _degenerate_matrix(R=5):
    """dense 200 x 200 background (202-node subgraphs at mnph 100), 6 isolated rated pairs (user 200+i rated only item
    200+i and nobody else rated it) and 4 users / items that rated / were rated by nobody (cold start)"""
    bg = _dense(200, 200, 0.6, R, 5)
    iso = (200 + np.arange(6), 200 + np.arange(6), np.arange(6) % R)
    A, (u, v, lab) = _matrix([bg, iso], 210, 210)
    cold = np.arange(206, 210)
    pairs = dict(iso=[(200 + i, 200 + i, i % R) for i in range(6)],
                 bg=[(int(u[k]), int(v[k]), int(lab[k])) for k in (0, 3001, 7777)],
                 cold=[(cold[0], cold[0], 2), (cold[1], int(v[10]), 4), (int(u[20]), cold[2], 0)])
    return A, pairs


def _mixed_pairs(pairs):
    p = pairs
    return [p["iso"][0], p["bg"][0], p["cold"][0], p["bg"][1], p["cold"][1], p["iso"][1], p["cold"][2]]


@pytest.mark.parametrize("plan,which", [(1, "mixed"), (2, "mixed"), (4, "mixed"), (2, "one_isolated"),
                                        (4, "one_normal")])
def test_degenerate_subgraphs(plan, which):
    """2-node subgraphs with zero edges (an isolated rated pair once its target edge is removed, a cold-start pair),
    target nodes without any in-edge (cold user or item next to a normal one) and 202-node subgraphs in one batch;
    B = 1.  Plans 2 and 4 run CTAs that own no node (forward / backward ``n_own == 0`` branches)"""
    A, pairs = _degenerate_matrix()
    sel = {"mixed": _mixed_pairs(pairs), "one_isolated": [pairs["iso"][2]], "one_normal": [pairs["bg"][2]]}[which]
    b, ob = _extracted(A, tuple(np.array(c) for c in zip(*sel)), 5, 1, 100)
    sizes = np.diff(b._priv["node_ptr"].cpu().numpy())
    if which == "mixed":
        assert sizes.min() == 2 and sizes.max() == 202 and ob["edge_index"].shape[1] > 0
    ref, m = _models(4, 5, plan=plan)
    hk = _hk(len(sel))
    tabs, _ = _images(m, b)
    if which == "mixed" and plan > 1:
        assert np.any(tabs["fwd"][:, 3] == 0) and np.any(tabs["bwd"][:, 3] == 0), "no CTA without own nodes"
    b._stage = None
    check_step(m, ref, b, ob, 0.001, 0.2, hk)
    _restaged_step_bit_identical(m, b, hk)


def test_dropout_removes_every_in_edge():
    """foreign batch (separate out-lists) with an injected edge_keep that drops every in-edge of a target item and of
    a few other nodes: their mean aggregate falls back to 1/max(0, 1) and must be exactly the root term"""
    from igmc_b200.util_functions import Batch
    A, pairs = _degenerate_matrix()
    _, ob = _extracted(A, tuple(np.array(c) for c in zip(*_mixed_pairs(pairs))), 5, 1, 100)
    b = Batch.from_arrays(ob["x"], ob["edge_index"], ob["edge_type"], ob["batch"], ob["y"], ob["num_graphs"])
    nptr = np.concatenate([[0], np.cumsum(np.bincount(ob["batch"], minlength=ob["num_graphs"]))])
    n_u1 = int((ob["x"][nptr[1]:nptr[2], 0::2].sum(1) > 0).sum())     # user nodes of graph 1 (labels 0, 2, ...)
    chosen = np.array([nptr[1] + n_u1, nptr[1] + 3, nptr[3] + 7, nptr[3] + n_u1 + 5])
    dst = ob["edge_index"][1]
    assert all(np.any(dst == c) for c in chosen)
    ek = torch.from_numpy((np.random.default_rng(6).random(len(dst)) > 0.2) & ~np.isin(dst, chosen))
    ref, m = _models(4, 5, plan=2)
    rmse, worst = check_step(m, ref, b, ob, 0.001, 0.2, _hk(ob["num_graphs"]), edge_keep=ek)
    ws = next(iter(v for k, v in m._ws.items() if k[2]))
    assert torch.equal(ws["inv_deg"][torch.from_numpy(chosen).cuda()].cpu(), torch.ones(len(chosen)))


def test_dgcnn_rs_on_degenerate_batch():
    """DGCNN_RS with k = 30 on the mixed batch: SortPooling pads the 2-node subgraphs"""
    from igmc_b200.models import edge_keep_reference, splitmix64
    A, pairs = _degenerate_matrix()
    b, ob = _extracted(A, tuple(np.array(c) for c in zip(*_mixed_pairs(pairs))), 5, 1, 100)
    ref, m = _models(4, 5, dgcnn_k=30)
    B, E = ob["num_graphs"], ob["edge_index"].shape[1]
    hk = _hk(B)
    m._step = 30
    ek = edge_keep_reference(splitmix64(m.drop_seed + 31), E, 0.2)
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    out_ref = ref(tb["x"], tb["edge_index"], tb["edge_type"], tb["batch"], ek, hk, tb["num_graphs"])
    loss_ref = torch.nn.functional.mse_loss(out_ref, tb["y"].view(-1)) + 0.001 * pyg_restated.arr_regulariser(ref)
    loss_ref.backward()
    loss = m.fused_step(b, ARR=0.001, hidden_keep=hk)
    b.check()
    ws = next(iter(v for k, v in m._ws.items() if k[2]))
    rmse = float(torch.sqrt(torch.mean((ws["sp"]["pred"].double().cpu() - out_ref.detach()) ** 2)))
    assert rmse <= 1e-4, rmse
    assert abs(float(loss) - float(loss_ref)) <= 1e-4 * max(1.0, abs(float(loss_ref)))
    names = {id(p): nme for nme, p in m.named_parameters()}
    sd_ref = dict(ref.named_parameters())
    table = []
    for e, (_, _, p) in zip(m._layout, m._named_order()):
        gref = sd_ref[names[id(p)]].grad
        table.append((names[id(p)], float((m._pview(m.flat_grad, e).double().cpu() - gref).abs().max()),
                      float(gref.abs().max())))
    gmax = max(t[2] for t in table)
    for name, err, scale in table:
        # the DGCNN_RS bar of tests/test_gpu_full_batch.py (first-layer att gradients cancel to ~1e-3 of the largest)
        assert err <= 3e-4 * scale + 2e-6 * gmax, (name, err, scale, gmax)


# ---- 5. layer count and multiply_by --------------------------------------------------------------------------------
def _small_batch(B=8, R=5):
    u, v, lab = synth_ratings(120, 90, 2500, num_classes=R, seed=3)
    return _extracted(build_adj(u, v, lab, 120, 90), (u[:B], v[:B], lab[:B]), R, 1, 30)


@pytest.mark.parametrize("L", [1, 2, 3, 8])
@pytest.mark.parametrize("plan", [0, 2])
def test_layer_count_train_step(L, plan):
    """IGMC with 1..MAX_LAYERS = 8 layers (the readout concatenates 32 L channels per target node)"""
    b, ob = _small_batch()
    ref, m = _models(4, 5, L=L, plan=plan)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(8))


def test_multiply_by_train_step():
    """multiply_by = 2 scales the prediction and therefore every gradient: fused_step and the autograd path"""
    from igmc_b200.models import edge_keep_reference, splitmix64
    b, ob = _small_batch()
    ref, m = _models(4, 5, multiply_by=2, plan=2)
    hk = _hk(8)
    check_step(m, ref, b, ob, 0.001, 0.2, hk)
    # autograd path (IGMC.forward + loss.backward, no ARR) with the same draws
    ek = edge_keep_reference(splitmix64(m.drop_seed + 31), ob["edge_index"].shape[1], 0.2)
    ref.zero_grad()
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    loss_ref, out_ref = pyg_restated.train_loss(ref, tb, 0.0, ek, hk)
    loss_ref.backward()
    m.zero_grad()
    out = m(b, edge_keep=ek, hidden_keep=hk)
    torch.nn.functional.mse_loss(out, b.y).backward()
    assert float(torch.sqrt(torch.mean((out.detach().double().cpu() - out_ref.detach()) ** 2))) <= 1e-4
    sd_ref = dict(ref.named_parameters())
    for name, p in m.named_parameters():
        gref = sd_ref[name].grad
        assert float((p.grad.double().cpu() - gref).abs().max()) <= 2e-4 * float(gref.abs().max()), name


# ---- 6. optimizer --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused_update", [True, False])
def test_adam_steps_match_torch_adam(fused_update, monkeypatch):
    """TrainEngine.step_pipe with the fused update kernel (igmc_reduce_update) and with FusedAdam.step (igmc_adam_step)
    against torch.optim.Adam in fp64 applied to the kernels' own gradients, step by step: Adam resumed from a state
    dict at step 5000, weight_decay 1e-2, and an lr lowered between two CUDA-graph replays (sync_lr)"""
    from igmc_b200.models import IGMC, FusedAdam
    from igmc_b200.train_eval import TrainEngine
    from igmc_b200.util_functions import MyDynamicDataset
    ds = make_synthetic_dataset("tiny", seed=0)
    tu, tv, tl = ds["train"]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, 10, None, None, ds["class_values"])
    torch.manual_seed(0)
    m = IGMC(d, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True, adj_dropout=0.2).cuda()
    opt = FusedAdam(m, lr=1e-3, weight_decay=1e-2)
    sd = opt.state_dict()
    gen = torch.Generator().manual_seed(7)
    for st in sd["state"].values():
        ea = torch.randn(st["exp_avg"].shape, generator=gen) * 1e-3
        st.update(step=torch.tensor(5000.0), exp_avg=ea, exp_avg_sq=(1.5 * ea) ** 2 + 1e-8)
    opt.load_state_dict(sd)
    params = list(m.parameters())
    ref_p = [p.detach().double().cpu().clone().requires_grad_(True) for p in params]
    ref_opt = torch.optim.Adam(ref_p, lr=1e-3, weight_decay=1e-2)
    ref_opt.load_state_dict(sd)
    start = [p.detach().cpu().clone() for p in params]
    if fused_update:   # the update kernel also writes the assembled gradient it applied into flat_grad
        monkeypatch.setattr(opt, "reduce_update", functools.partial(FusedAdam.reduce_update, opt, grad_copy=m.flat_grad))
    eng = TrainEngine(d, m, opt, 8, ARR=0.001)
    eng.fused_update = fused_update
    eng.prime(np.arange(0, 8), epoch=1)
    steps = 8
    for s in range(steps):
        if s == 5:
            for grp in opt.param_groups + ref_opt.param_groups:
                grp["lr"] = 2e-4
            eng.sync_lr()
        eng.step_pipe(np.arange((s + 1) * 8, (s + 2) * 8) if s < steps - 1 else None, epoch=1)
        torch.cuda.synchronize()
        for p, rp in zip(params, ref_p):
            rp.grad = m._pview(m.flat_grad, opt._entry[id(p)]).double().cpu().clone()
        ref_opt.step()
        err = max(float((p.detach().double().cpu() - rp.detach()).abs().max()) for p, rp in zip(params, ref_p))
        assert err <= 1e-6, (s, err)
    eng.check()
    assert (eng.exchange is not None) == fused_update and len(eng.graphs) > 0
    assert int(opt.step_count[0]) == 5000 + steps
    moved = max(float((p.detach().cpu() - p0).abs().max()) for p, p0 in zip(params, start))
    assert moved > 1e-3
    eng.close()
