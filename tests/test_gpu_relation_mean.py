"""Training and evaluation with the PyG >= 1.6 RGCNConv (``rgcn="pyg-2"``: one mean per destination and relation) on
every kernel plan, against fp64 autograd of the restated layer (tests/pyg2_oracle.py).

Bars are the suite's (tests/helpers.py assert_step_matches): predictions within 1e-4 RMSE, every gradient within 2e-4
of its tensor's largest reference entry (DGCNN_RS: its own bar), Adam after 3 steps within 5e-5 of torch's."""
import functools

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200.data import build_adj, make_synthetic_dataset
from igmc_b200.models import edge_keep_reference, hidden_keep_reference, splitmix64
from oracle import extract_np, pyg_restated
from tests import pyg2_oracle
from tests.helpers import assert_step_matches, check_step, oracle_train_step
from tests.test_gpu_model import _gpu_batch, _oracle_batch
from tests.test_gpu_production_path import _check_eval, _dataset_and_oracle, _oracle_eval
from tests.test_gpu_regimes import _extracted, _hk, _ml_100k

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _ml_1m():
    return make_synthetic_dataset("ml_1m", seed=0)


def _models(in0, R, NB=4, L=4, adj_dropout=0.2, plan="auto", dgcnn_k=None, rgcn="pyg-2"):
    """(fp64 oracle, device model) of the same parameters, both with the layer ``rgcn``"""
    from igmc_b200.models import DGCNN_RS, IGMC
    torch.manual_seed(0)
    if dgcnn_k is None:
        ref = pyg2_oracle.igmc_ref(rgcn, in0, (32,) * L, R, NB, adj_dropout)
        m = IGMC(in0, latent_dim=[32] * L, num_relations=R, num_bases=NB, regression=True, adj_dropout=adj_dropout,
                 rgcn=rgcn)
    else:
        ref = pyg2_oracle.dgcnn_rs_ref(rgcn, in0, (32, 32, 32, 1), dgcnn_k, R, NB, adj_dropout)
        m = DGCNN_RS(in0, latent_dim=[32, 32, 32, 1], k=dgcnn_k, num_relations=R, num_bases=NB, regression=True,
                     adj_dropout=adj_dropout, rgcn=rgcn)
    with torch.no_grad():   # PyG 2 zero-inits the bias: give it values so that its gradient path is exercised too
        for c in ref.convs:
            c.bias.uniform_(-0.3, 0.3)
    ref = pyg_restated.set_formulation(ref.double().train(), "transform")
    m = m.cuda().train()
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    m.kernel_plan = plan
    return ref, m


def _staged_step_bit_identical(m, b, hk, step=30):
    """the step just checked, repeated on the list images of igmc_stage_lists: the same gradient bit for bit"""
    g0 = m.flat_grad.clone()
    m._step = step + 1
    m.stage_batch(b, True, m.make_dropout(True))
    m._step = step
    m.fused_step(b, ARR=0.001, hidden_keep=hk)
    b.check()
    b._stage = None
    assert torch.equal(m.flat_grad, g0)


# ---- full batches of the BASELINE configs ---------------------------------------------------------------------------
@pytest.mark.parametrize("name,mnph,B,plan", [("ml_100k", 200, 50, "auto"), ("ml_1m", 100, 50, 2),
                                              ("ml_1m", 100, 50, 3), ("ml_1m_r02", 100, 256, 1)])
def test_full_batch_train_step(name, mnph, B, plan):
    """ml_100k* batch 50 with the kernels' own edge and hidden dropout; ml_1m* batch 50 on 2 and 3 CTAs; ml_1m* ratio
    0.2 at batch 256 on one CTA per subgraph; then the same step on staged list images"""
    from igmc_b200.util_functions import MyDynamicDataset
    ds = make_synthetic_dataset(name, seed=0)
    tu, tv, tl = ds["train"]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, mnph, None, None, ds["class_values"], seed=11)
    idx = np.random.default_rng(5).choice(len(tu), B, replace=False)
    b = d.extract_batch(idx)
    ob = extract_np.extract_batch(extract_np.RatingCSR(ds["adj_train"]), tu[idx], tv[idx], tl[idx], ds["class_values"],
                                  1, 1.0, mnph, seed=11, pair_ids=idx)
    assert np.array_equal(b.edge_index.cpu().numpy(), ob["edge_index"])
    ref, m = _models(4, 5, adj_dropout=ds["adj_dropout"], plan=plan)
    hk = None if name == "ml_100k" else _hk(B)
    check_step(m, ref, b, ob, 0.001, ds["adj_dropout"], hk)
    assert _lib.is_rs(m._plan(b)) and (plan == "auto" or m._plan(b) == plan)
    if hk is not None:
        _staged_step_bit_identical(m, b, hk)


def test_full_batch_flixster_static():
    """REAL flixster split (R = 10) through the static MyDataset store, batch 50, edge dropout 0.2"""
    from igmc_b200.util_functions import MyDataset
    ds = make_synthetic_dataset("flixster", seed=0)
    tu, tv, tl = ds["train"]
    n = 400
    d = MyDataset(None, ds["adj_train"], (tu[:n], tv[:n]), tl[:n], 1, 1.0, ds["max_nodes_per_hop"], None, None,
                  ds["class_values"])
    idx = np.random.default_rng(1).choice(n, 50, replace=False)
    b = d.extract_batch(idx)
    ob = extract_np.extract_batch(extract_np.RatingCSR(ds["adj_train"]), tu[idx], tv[idx], tl[idx], ds["class_values"],
                                  1, 1.0, ds["max_nodes_per_hop"], pair_ids=idx)
    assert np.array_equal(b.edge_index.cpu().numpy(), ob["edge_index"])
    ref, m = _models(4, ds["num_relations"])
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(50, 3))
    assert _lib.is_rs(m._plan(b))


@pytest.mark.parametrize("plan", ["auto", 0, _lib.plan_l2(2)])
def test_dgcnn_rs_ml_1m(plan, monkeypatch):
    """DGCNN_RS (k = 30) on an ml_1m* batch of 50: the same conv kernels with the external readout.

    SortPooling orders nodes by their last channel; where two keys lie within fp32 rounding of each other the kernels
    (fp32) and the oracle (fp64) may order them differently, and the gradient is discontinuous there.  As in
    tests/test_gpu_large_subgraphs.py, the kernels' order is first checked against the oracle's keys (it may differ from
    the oracle's own sort only between keys closer than 1e-5) and the oracle's gradient is then taken in that order."""
    from tests.test_gpu_large_subgraphs import _pool_in_order
    ds = _ml_1m()
    tu, tv, tl = ds["train"]
    idx = np.arange(50)
    b, ob = _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, 1, 100)
    B, k = 50, 30
    ref, m = _models(4, 5, adj_dropout=0.0, dgcnn_k=k, plan=plan)
    hk = _hk(B)
    m._step = 30
    m.fused_step(b, ARR=0.001, hidden_keep=hk)          # the step check_step runs: the kernels' pooling order
    b.check()
    ws = next(v for key, v in m._ws.items() if key[2] and key[1] == B)
    perm = ws["sp"]["perm"][:B * k].view(B, k).cpu()
    keys = {}
    orig = pyg_restated.global_sort_pool

    def capture(x, batch, kk, num_graphs=None):
        keys["x"] = x.detach()[:, -1].cpu().numpy()
        return orig(x, batch, kk, num_graphs)
    monkeypatch.setattr(pyg_restated, "global_sort_pool", capture)
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    with torch.no_grad():
        ref(tb["x"], tb["edge_index"], tb["edge_type"], tb["batch"], None, hk, tb["num_graphs"])
    key = keys["x"]
    start = np.concatenate([[0], np.cumsum(np.bincount(ob["batch"], minlength=B))])
    flips, worst = 0, 0.0
    for g in range(B):
        n = start[g + 1] - start[g]
        own = start[g] + np.argsort(-key[start[g]:start[g + 1]], kind="stable")[:k]
        got = perm[g].numpy()
        assert (got[:min(n, k)] >= 0).all() and (got[min(n, k):] < 0).all()
        for t in range(min(n, k)):
            if got[t] != own[t]:
                flips += 1
                worst = max(worst, abs(float(key[got[t]]) - float(key[own[t]])))
    assert worst <= 1e-5, worst
    print("dgcnn_rs plan %s: %d pooled positions ordered differently from the fp64 sort, keys within %.1e"
          % (plan, flips, worst))
    monkeypatch.setattr(pyg_restated, "global_sort_pool", _pool_in_order(perm))
    check_step(m, ref, b, ob, 0.001, 0.0, hk)


# ---- every plan -----------------------------------------------------------------------------------------------------
def _ml_1m_batch(B, mnph=100):
    ds = _ml_1m()
    tu, tv, tl = ds["train"]
    idx = np.arange(200, 200 + B)
    return _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, 1, mnph)


@pytest.mark.parametrize("plan", [1, 2, 4, 0, _lib.plan_l2(1), _lib.plan_l2(4)])
def test_every_plan(plan):
    b, ob = _ml_1m_batch(16)
    ref, m = _models(4, 5, NB=2 if plan in (2, 0) else 4, plan=plan)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(16))
    assert m._plan(b) == plan


@pytest.mark.parametrize("R", [13, 71])
def test_generic_plan_many_relations(R):
    """R = 13 and R = 71: beyond the relation-space kernels; plan 0 by the "auto" rule"""
    nu, nv = 150, 150
    rng = np.random.default_rng(R)
    u, v = np.nonzero(rng.random((nu, nv)) < 0.08)
    A = build_adj(u, v, rng.integers(0, R, len(u)), nu, nv)
    sel = np.arange(0, len(u), len(u) // 8)[:8]
    b, ob = _extracted(A, (u[sel], v[sel], np.asarray(A[u[sel], v[sel]]).ravel() - 1), R, 1, 40)
    ref, m = _models(4, R)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(8))
    assert m._plan(b) == 0


def test_l2_plan_auto_uncapped():
    """ml_100k* h = 1 without a node cap (a subgraph of more than 700 nodes): the L2 plan by the "auto" rule, with the
    kernels' own dropout draws"""
    ds = _ml_100k()
    tu, tv, tl = ds["train"]
    A = ds["adj_train"]
    score = np.diff(A.indptr)[tu] + np.asarray(A.getnnz(0)).ravel()[tv]
    idx = np.concatenate([np.argsort(-score, kind="stable")[:1], np.arange(100, 111)])
    b, ob = _extracted(A, (tu[idx], tv[idx], tl[idx]), 5, 1, None)
    assert np.bincount(ob["batch"]).max() > 700
    ref, m = _models(4, 5)
    check_step(m, ref, b, ob, 0.001, 0.2, None)
    assert _lib.l2_csize(m._plan(b)) > 0


# ---- regimes --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("plan", [2, 0, _lib.plan_l2(2)])
def test_relation_dropped_at_a_node(plan):
    """every in-edge of one relation at a target node dropped (its term vanishes, the other relations keep their own
    means); nodes whose in-edges all have one relation are in the batch too"""
    b, ob = _ml_1m_batch(12)
    ei, et = ob["edge_index"], ob["edge_type"]
    tgt = int(np.nonzero(ob["x"][:, 0] == 1)[0][0])           # target user of graph 0
    types = et[ei[1] == tgt]
    r = int(np.bincount(types).argmax())
    assert len(set(types.tolist())) > 1
    ek = torch.rand(ei.shape[1], generator=torch.Generator().manual_seed(4)) > 0.2
    ek[torch.from_numpy((ei[1] == tgt) & (et == r))] = False
    one_rel = [v for v in range(ob["x"].shape[0]) if len(set(et[ei[1] == v].tolist())) == 1]
    assert len(one_rel) > 10
    ref, m = _models(4, 5, plan=plan)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(12), edge_keep=ek)
    assert m._plan(b) == plan


def _sparse_cases():
    """ml_1m* plus a user and an item that rated only each other (a 2-node subgraph without edges) and a user with a
    single rating (a cold-start subgraph: no other user-side node), next to an ordinary pair"""
    ds = _ml_1m()
    A0 = ds["adj_train"].tocoo()
    nu, nv = A0.shape
    tu, tv, tl = ds["train"]
    A = build_adj(np.append(A0.row, [nu, nu + 1]), np.append(A0.col, [nv, int(tv[3])]), np.append(A0.data - 1, [2, 4]),
                  nu + 2, nv + 1)
    pairs = (np.array([nu, nu + 1, tu[7]]), np.array([nv, tv[3], tv[7]]), np.array([2, 4, tl[7]]))
    b, ob = _extracted(A, pairs, 5, 1, 100)
    n = np.bincount(ob["batch"], minlength=3)
    assert n[0] == 2 and n[1] > 2
    return b, ob


@pytest.mark.parametrize("plan", [4, 1, 0, _lib.plan_l2(8)])
def test_zero_edge_and_cold_start_subgraphs(plan):
    """plan 4 and the 8-CTA L2 plan leave CTAs of the 2-node subgraph without nodes"""
    b, ob = _sparse_cases()
    ref, m = _models(4, 5, plan=plan)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(3))
    assert m._plan(b) == plan


@pytest.mark.parametrize("plan", [1, 2, 0])
def test_single_subgraph_batch(plan):
    b, ob = _ml_1m_batch(1)
    ref, m = _models(4, 5, plan=plan)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(1))


@pytest.mark.parametrize("plan", [2, 0, _lib.plan_l2(2)])
def test_single_relation_modes_agree(plan):
    """with R = 1 the two layers are the same function: the same parameters give predictions and gradients within 1e-6"""
    A, links, cv, ob = _oracle_batch(R=1)
    out = []
    for rgcn in ("pyg-1.4", "pyg-2"):
        ref, m = _models(4, 1, plan=plan, rgcn=rgcn)
        if rgcn == "pyg-2":   # the pyg-1.4 model's parameters under the new names
            sd = {k.replace(".att", ".comp").replace(".basis", ".weight"): v for k, v in out[0][2].items()}
            m.load_state_dict(sd)
        b = _gpu_batch(ob)
        m._step = 30
        m.fused_step(b, ARR=0.001, hidden_keep=_hk(ob["num_graphs"]))
        b.check()
        ws = next(v for k, v in m._ws.items() if k[2])
        out.append((ws["pred"].clone(), m.flat_grad.clone(), m.state_dict()))
    assert float((out[0][0] - out[1][0]).abs().max()) <= 1e-6
    assert float((out[0][1] - out[1][1]).abs().max()) <= 1e-6 * float(out[0][1].abs().max())


# ---- optimizer, engine, evaluation, checkpoints ---------------------------------------------------------------------
def test_adam_matches_torch():
    from igmc_b200.models import FusedAdam
    A, links, cv, ob = _oracle_batch()
    ref, m = _models(4, 5, adj_dropout=0.0)
    opt_ref = torch.optim.Adam(ref.parameters(), lr=1e-3)
    opt = FusedAdam(m, lr=1e-3)
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    b = _gpu_batch(ob)
    for it in range(3):
        hk = _hk(ob["num_graphs"], it)
        opt_ref.zero_grad()
        loss_ref, _ = pyg_restated.train_loss(ref, tb, 0.001, None, hk)
        loss_ref.backward()
        opt_ref.step()
        m.fused_step(b, ARR=0.001, hidden_keep=hk)
        opt.step()
    want = dict(ref.named_parameters())
    for name, p in m.named_parameters():
        assert float((p.detach().double().cpu() - want[name].detach()).abs().max()) <= 5e-5, name


def _engine_run(use_graph, check_oracle):
    """two epochs of 200 ml_1m* pairs (mnph 100, batch 50) through TrainEngine.step_pipe; returns the parameters"""
    from igmc_b200.models import FusedAdam
    from igmc_b200.train_eval import TrainEngine, shard_batches
    from igmc_b200.util_functions import MyDynamicDataset
    ds = _ml_1m()
    n, cv, B = 200, ds["class_values"], 50
    tu, tv, tl = [a[:n] for a in ds["train"]]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, 100, None, None, cv)
    ref, m = _models(4, 5)
    launched = []
    one = m._launch_train
    m._launch_train = lambda *a: launched.append(1) or one(*a)
    opt = FusedAdam(m, lr=1e-3)
    # the update kernel also writes the assembled gradient it applied into flat_grad
    opt.reduce_update = functools.partial(FusedAdam.reduce_update, opt, grad_copy=m.flat_grad)
    eng = TrainEngine(d, m, opt, B, ARR=0.001, use_graph=use_graph, sample_seed=5)
    g = extract_np.RatingCSR(ds["adj_train"])
    gen = torch.Generator().manual_seed(3)
    try:
        for ep in (1, 2):
            batches = shard_batches(torch.randperm(n, generator=gen).numpy(), B, 0, 1)
            eng.prime(batches[0][0], ep, batches[0][1])
            for k, (idx, G) in enumerate(batches):
                sd = {key: v.detach().double().cpu().clone() for key, v in m.state_dict().items()}
                nxt = batches[k + 1] if k + 1 < len(batches) else None
                eng.step_pipe(nxt[0] if nxt else None, ep, nxt[1] if nxt else None)
                torch.cuda.synchronize()
                eng.check()
                if not check_oracle or k not in (0, len(batches) - 1):
                    continue
                seed = eng.drop_seed(eng.steps)
                ob = extract_np.extract_batch(g, tu[idx], tv[idx], tl[idx], cv, 1, 1.0, 100,
                                              seed=splitmix64(eng.sample_seed + ep), pair_ids=idx)
                ref.load_state_dict(sd)
                loss_ref, out_ref = oracle_train_step(
                    ref, ob, 0.001, edge_keep_reference(seed, ob["edge_index"].shape[1], 0.2),
                    hidden_keep_reference(seed, len(idx), 0.5))
                ws = next(v for key, v in m._ws.items() if key[2] and key[1] == len(idx))
                assert_step_matches(m, ref, ws["pred"], eng.last_loss, m.flat_grad, loss_ref, out_ref,
                                    "engine epoch %d step %d" % (ep, eng.steps))
        # R <= 12: the one-launch train kernel and the fused reduce / exchange / Adam kernel
        assert eng.exchange is not None and len(launched) > 0
        assert _lib.is_rs(next(iter(m._plans.values())))
        if use_graph:
            assert len(eng.graphs) > 0
    finally:
        eng.close()
    return m.flat_params.clone()


def test_engine_fast_path_graphs_and_determinism():
    """the pipelined engine on the fast path, against the oracle; CUDA graphs on and off give bit-identical
    parameters, and so does a second run"""
    p_graph = _engine_run(True, True)
    p_eager = _engine_run(False, False)
    p_again = _engine_run(True, False)
    assert torch.equal(p_graph, p_eager) and torch.equal(p_graph, p_again)


def test_eval_ensemble_and_checkpoint_round_trip():
    """150 ml_100k* test pairs at mnph 200 (402-node subgraphs, plan 4), batch 32: per-pair predictions, eval_rmse,
    eval_loss, test_once; a two-checkpoint ensemble; a state_dict round trip in the new names"""
    import math
    import os
    import tempfile
    from igmc_b200.models import IGMC
    from igmc_b200.train_eval import eval_rmse_ensemble
    ds = _ml_100k()
    eu, ev, el = [a[:150] for a in ds["test"]]
    d, ob = _dataset_and_oracle(ds["adj_train"], (eu, ev, el), ds["class_values"], 1, 200)
    ref, m = _models(4, 5)
    ref.eval()
    pred_ref, y = _oracle_eval(ref, ob)
    _check_eval(m, d, pred_ref, y, (32,), "pyg-2 eval")
    ref2, m2 = _models(4, 5)
    with torch.no_grad():
        for p in ref2.parameters():
            p.mul_(0.9)
    m2.load_state_dict({k: v.float() for k, v in ref2.state_dict().items()})
    pred_ref2, _ = _oracle_eval(ref2.eval(), ob)
    with tempfile.TemporaryDirectory() as tmp:
        cks = []
        for k, mm in enumerate((m, m2)):
            cks.append(os.path.join(tmp, "model_checkpoint%d.pth" % k))
            torch.save(mm.state_dict(), cks[-1])
        got = eval_rmse_ensemble(m, cks, d, None, batch_size=32)
        # round trip: a fresh pyg-2 model loads the file and predicts the same bits; the default layer refuses it
        m3 = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True, rgcn="pyg-2").cuda().eval()
        sd = torch.load(cks[1])
        assert "convs.0.comp" in sd and "convs.0.weight" in sd
        m3.load_state_dict(sd)
        with pytest.raises(RuntimeError):
            IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).load_state_dict(sd)
    want = math.sqrt(float((((pred_ref + pred_ref2) / 2 - y) ** 2).mean()))
    assert abs(got - want) <= 1e-4, (got, want)
    m2.eval()
    b = d.extract_batch(np.arange(32))
    with torch.no_grad():
        assert torch.equal(m2(b), m3(b))
