"""Enclosing subgraphs too large for every shared-memory kernel plan, trained and evaluated on the L2 plan
(csrc/rgcn_l2.cu: node features in global memory / L2, a cluster of CTAs per subgraph).

Every batch comes from the CUDA extractor and is first checked bit-exact against oracle/extract_np; train steps are
then compared with fp64 autograd of oracle/pyg_restated with the suite's bars (tests/helpers.py assert_step_matches):
ratings within 1e-4 RMSE, gradients within 2e-4 of the tensor's largest reference entry."""
import functools

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200.data import build_adj, make_synthetic_dataset
from igmc_b200.models import edge_keep_reference, hidden_keep_reference, splitmix64
from oracle import extract_np, pyg_restated
from tests.helpers import assert_step_matches, check_step, oracle_train_step
from tests.test_gpu_production_path import _check_eval, _dataset_and_oracle, _oracle_eval
from tests.test_gpu_regimes import _extracted, _hk, _ml_100k, _models

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _ml_1m():
    return make_synthetic_dataset("ml_1m", seed=0)


def _sizes(ob):
    return np.bincount(ob["batch"], minlength=ob["num_graphs"])


def _is_l2(m, b):
    return _lib.l2_csize(m._plan(b)) > 0


def _largest_pairs(A, pairs, k):
    """indices of the ``k`` training pairs with the largest one-hop enclosing subgraphs (row + column degree)"""
    tu, tv, _ = pairs
    score = np.diff(A.indptr)[tu] + np.asarray(A.getnnz(0)).ravel()[tv]
    return np.argsort(-score, kind="stable")[:k]


@functools.lru_cache(maxsize=None)
def _case1():
    """ml_100k*, h = 1, no max-nodes-per-hop, B = 16, one subgraph of more than 700 nodes"""
    ds = _ml_100k()
    tu, tv, tl = ds["train"]
    idx = np.concatenate([_largest_pairs(ds["adj_train"], ds["train"], 1), np.arange(100, 115)])
    b, ob = _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, 1, None)
    assert _sizes(ob).max() > 700 and ob["num_graphs"] == 16
    return b, ob


# ---- 1-5. train steps ----------------------------------------------------------------------------------------------
def test_ml_100k_uncapped_own_dropout():
    """own edge and hidden dropout draws; the L2 plan is picked by the "auto" rule; two runs are bit-identical"""
    b, ob = _case1()
    ref, m = _models(4, 5)
    check_step(m, ref, b, ob, 0.001, 0.2, None)
    assert _is_l2(m, b)
    g0 = m.flat_grad.clone()
    m._step = 30
    m.fused_step(b, ARR=0.001)
    b.check()
    assert torch.equal(m.flat_grad, g0)


@pytest.mark.parametrize("h,mnph", [(2, 200), (3, 100)])
def test_multi_hop_large(h, mnph):
    """input widths 6 and 8 with the subgraph sizes of the hop-count ablation"""
    ds = _ml_100k()
    tu, tv, tl = ds["train"]
    idx = np.array([0, 1, 2, 3])
    b, ob = _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, h, mnph)
    assert ob["x"].shape[1] == 2 * h + 2 and _sizes(ob).max() > 446
    ref, m = _models(2 * h + 2, 5)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(4))
    assert _is_l2(m, b)


def _many_relations_batch():
    """(R, batch, oracle batch): four pairs of a 600 x 600 matrix with R = 71 rating levels, n_cap 564"""
    R, nu, nv = 71, 600, 600
    rng = np.random.default_rng(4)
    u, v = np.nonzero(rng.random((nu, nv)) < 0.3)
    keep = ~((u == 0) & (v >= 281))               # user 0 rates exactly items 0..280: the longest list, 281
    u, v = u[keep], v[keep]
    u, v = np.concatenate([u, np.zeros(281, np.int64)]), np.concatenate([v, np.arange(281)])
    uv = np.unique(u * nv + v)
    u, v = uv // nv, uv % nv
    A = build_adj(u, v, rng.integers(0, R, len(u)), nu, nv)
    assert max(np.diff(A.indptr).max(), A.getnnz(0).max()) == 281
    pairs = (A.nonzero()[0][:4], A.nonzero()[1][:4], np.asarray(A[A.nonzero()[0][:4], A.nonzero()[1][:4]]).ravel() - 1)
    b, ob = _extracted(A, pairs, R, 1, None)
    assert b._priv["n_cap"] == 564
    return R, b, ob


@pytest.mark.parametrize("NB", [2, 4])
def test_many_relations(NB):
    """R = 71 (YahooMusic's rating levels) at n_cap 564: beyond the generic plan's 422 nodes"""
    R, b, ob = _many_relations_batch()
    ref, m = _models(4, R, NB=NB)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(4))
    assert _is_l2(m, b)


def test_giant_subgraph_next_to_empty_one():
    """one uncapped ml_1m* subgraph of more than 4000 nodes, a 2-node subgraph without edges, and a third"""
    ds = _ml_1m()
    A0 = ds["adj_train"].tocoo()
    nu, nv = A0.shape
    # one more user and item that rated only each other: their enclosing subgraph is the two targets, no edge
    A = build_adj(np.append(A0.row, nu), np.append(A0.col, nv), np.append(A0.data - 1, 2), nu + 1, nv + 1)
    tu, tv, tl = ds["train"]
    big = _largest_pairs(ds["adj_train"], ds["train"], 1)[0]
    pairs = (np.array([tu[big], nu, tu[7]]), np.array([tv[big], nv, tv[7]]), np.array([tl[big], 2, tl[7]]))
    b, ob = _extracted(A, pairs, 5, 1, None)
    n = _sizes(ob)
    assert n[0] > 4000 and n[1] == 2
    ref, m = _models(4, 5)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(3))
    assert _is_l2(m, b) and _lib.l2_csize(m._plan(b)) == 8


def test_forced_l2_at_baseline_batch():
    """the benchmark's batch (ml_1m*, mnph 100, B = 50) on the forced L2 plan: matches the oracle and plan 0"""
    ds = _ml_1m()
    tu, tv, tl = ds["train"]
    idx = np.arange(50)
    b, ob = _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, 1, 100)
    hk = _hk(50)
    grads, preds = [], []
    for plan in (_lib.plan_l2(2), 0):
        ref, m = _models(4, 5, plan=plan)
        check_step(m, ref, b, ob, 0.001, 0.2, hk)
        assert m._plan(b) == plan
        grads.append(m.flat_grad.clone())
        preds.append(next(v for k, v in m._ws.items() if k[2])["pred"].clone())
    rmse = float(torch.sqrt(torch.mean((preds[0].double() - preds[1].double()) ** 2)))
    assert rmse <= 1e-4
    for e in m._layout:
        a, c = m._pview(grads[0], e), m._pview(grads[1], e)
        assert float((a - c).abs().max()) <= 2e-4 * float(c.abs().max()) + 1e-12


# ---- 6. foreign batch through autograd ----------------------------------------------------------------------------
def test_foreign_batch_autograd():
    """a PyG-collated batch (separate in- and out-lists) through model(data) + loss.backward(), with an injected edge
    dropout that keeps the two directions of an edge differently"""
    from igmc_b200.util_functions import Batch
    _, ob = _case1()
    fb = Batch.from_arrays(ob["x"], ob["edge_index"], ob["edge_type"], ob["batch"], ob["y"], ob["num_graphs"])
    E, B = ob["edge_index"].shape[1], ob["num_graphs"]
    ek = torch.rand(E, generator=torch.Generator().manual_seed(5)) > 0.3
    half = E // 2
    assert bool((ek[:half] != ek[half:2 * half]).any())
    hk = _hk(B)
    ref, m = _models(4, 5)
    loss_ref, out_ref = oracle_train_step(ref, ob, 0.0, ek, hk)
    out = m(fb, edge_keep=ek, hidden_keep=hk)
    assert _is_l2(m, fb) and fb._priv["symmetric"] == 0
    loss = torch.nn.functional.mse_loss(out, fb.y)
    loss.backward()
    fb.check()
    grad = torch.zeros_like(m.flat_grad)
    for e, (_, _, p) in zip(m._layout, m._named_order()):
        m._pview(grad, e).copy_(p.grad)
    assert_step_matches(m, ref, out.detach(), loss.detach(), grad, loss_ref, out_ref, "foreign autograd")


# ---- 7. DGCNN_RS --------------------------------------------------------------------------------------------------
def test_dgcnn_rs_l2_plan_train_step():
    """the external readout's d concat_states (S.dstate) through the L2 backward, full bars: DGCNN_RS (k = 30) on the
    forced L2 plan at the benchmark's subgraph sizes (ml_1m*, mnph 100, 16 pairs)"""
    ds = _ml_1m()
    tu, tv, tl = ds["train"]
    idx = np.arange(16)
    b, ob = _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, 1, 100)
    ref, m = _models(4, 5, dgcnn_k=30, plan=_lib.plan_l2(4))
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(16))
    assert m._plan(b) == _lib.plan_l2(4)


def _pool_in_order(perm):
    """``global_sort_pool`` that keeps the rows ``perm`` [B, k] names (batch-global node ids, -1 = padding) in that
    order instead of sorting: the oracle's gradient for a given pooling order"""
    def pool(x, batch, k, num_graphs=None):
        P = perm.to(x.device).long()
        out = torch.zeros(P.shape[0], k, x.shape[1], dtype=x.dtype, device=x.device)
        valid = P >= 0
        out[valid] = x[P[valid]]
        return out.reshape(P.shape[0], k * x.shape[1])
    return pool


def _percentile_k(q=0.6):
    """k of the reference's percentile rule (models.py:69-73) over the uncapped ml_100k* subgraphs of 64 pairs"""
    from igmc_b200.models import DGCNN_RS
    from igmc_b200.util_functions import MyDynamicDataset
    ds = _ml_100k()
    tu, tv, tl = [a[:64] for a in ds["train"]]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, None, None, None, ds["class_values"], seed=3)
    m = DGCNN_RS(d, latent_dim=[32, 32, 32, 1], k=q, num_relations=5, num_bases=4, regression=True)
    counts = sorted(int(v) for v in d.node_counts())
    assert m.k == max(10, counts[int(np.ceil(q * len(counts))) - 1])
    return m.k


@pytest.mark.parametrize("k", ["30", "percentile"])
def test_dgcnn_rs_large(k, monkeypatch):
    """DGCNN_RS on case 1's batch (a subgraph of more than 700 nodes), on the L2 plan the rule picks, full bars.

    SortPooling orders nodes by their last channel; where two keys lie within fp32 rounding of each other the kernels
    (fp32) and the oracle (fp64) may order them differently, and the gradient is discontinuous there (a node moves to
    another Conv1d position).  So the kernels' order is first checked against the oracle's keys - it may differ from
    the oracle's own sort only between keys closer than 1e-5 - and the oracle's gradient is then taken in that order."""
    k = 30 if k == "30" else _percentile_k()
    b, ob = _case1()
    B = ob["num_graphs"]
    ref, m = _models(4, 5, dgcnn_k=k)
    hk = _hk(B)
    m._step = 30
    m.fused_step(b, ARR=0.001, hidden_keep=hk)          # the step check_step runs: the kernels' pooling order
    b.check()
    assert _is_l2(m, b)
    ws = next(v for key, v in m._ws.items() if key[2] and key[1] == B)
    perm = ws["sp"]["perm"][:B * k].view(B, k).cpu()
    # the oracle's fp64 sort keys of the same step (same edge dropout draws)
    keys = {}
    orig = pyg_restated.global_sort_pool

    def capture(x, batch, kk, num_graphs=None):
        keys["x"] = x.detach()[:, -1].cpu().numpy()
        return orig(x, batch, kk, num_graphs)
    monkeypatch.setattr(pyg_restated, "global_sort_pool", capture)
    E = ob["edge_index"].shape[1]
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    with torch.no_grad():
        ref(tb["x"], tb["edge_index"], tb["edge_type"], tb["batch"], edge_keep_reference(splitmix64(m.drop_seed + 31),
                                                                                        E, 0.2), hk, tb["num_graphs"])
    key, start = keys["x"], np.concatenate([[0], np.cumsum(_sizes(ob))])
    flips, worst = 0, 0.0
    for g in range(B):
        n = start[g + 1] - start[g]
        own = start[g] + np.argsort(-key[start[g]:start[g + 1]], kind="stable")[:k]
        got = perm[g].numpy()
        assert np.array_equal(got[:min(n, k)] >= 0, np.ones(min(n, k), bool)) and (got[min(n, k):] < 0).all()
        for t in range(min(n, k)):
            if got[t] != own[t]:
                flips += 1
                worst = max(worst, abs(float(key[got[t]]) - float(key[own[t]])))
    assert worst <= 1e-5, worst
    print("dgcnn_rs k=%d: %d pooled positions ordered differently from the fp64 sort, keys within %.1e"
          % (k, flips, worst))
    monkeypatch.setattr(pyg_restated, "global_sort_pool", _pool_in_order(perm))
    check_step(m, ref, b, ob, 0.001, 0.2, hk)


# ---- 8. evaluation ------------------------------------------------------------------------------------------------
def test_eval_and_ensemble_large():
    """150 test pairs of ml_100k* at h = 1 without a node cap, batch 32 (ragged last batch): per-pair predictions,
    eval_rmse, eval_loss, test_once, and a two-checkpoint ensemble"""
    import math
    import os
    import tempfile
    from igmc_b200.train_eval import eval_rmse_ensemble
    ds = _ml_100k()
    eu, ev, el = [a[:150] for a in ds["test"]]
    d, ob = _dataset_and_oracle(ds["adj_train"], (eu, ev, el), ds["class_values"], 1, None)
    assert _sizes(ob).max() > 568
    ref, m = _models(4, 5)
    ref.eval()
    pred_ref, y = _oracle_eval(ref, ob)
    _check_eval(m, d, pred_ref, y, (32,), "l2 eval")
    assert _is_l2(m, d.extract_batch(np.arange(32)))
    # ensemble of two checkpoints: the mean of the two models' predictions (train_eval.py eval_rmse_ensemble)
    ref2, m2 = _models(4, 5)
    with torch.no_grad():
        for p in ref2.parameters():
            p.mul_(0.9)
    m2.load_state_dict({k: v.float() for k, v in ref2.state_dict().items()})
    ref2.eval()
    pred_ref2, _ = _oracle_eval(ref2, ob)
    with tempfile.TemporaryDirectory() as tmp:
        cks = []
        for k, mm in enumerate((m, m2)):
            cks.append(os.path.join(tmp, "model_checkpoint%d.pth" % k))
            torch.save(mm.state_dict(), cks[-1])
        got = eval_rmse_ensemble(m, cks, d, None, batch_size=32)
    want = math.sqrt(float((((pred_ref + pred_ref2) / 2 - y) ** 2).mean()))
    assert abs(got - want) <= 1e-4, (got, want)


# ---- 9. TrainEngine -----------------------------------------------------------------------------------------------
def _engine_run(use_graph, check_oracle):
    from igmc_b200.models import FusedAdam
    from igmc_b200.train_eval import TrainEngine, shard_batches
    from igmc_b200.util_functions import MyDynamicDataset
    ds = _ml_100k()
    n, cv, B = 300, ds["class_values"], 50
    tu, tv, tl = [a[:n] for a in ds["train"]]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 2, 1.0, 200, None, None, cv)
    ref, m = _models(6, 5)
    opt = FusedAdam(m, lr=1e-3)
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
                # the step rebuilt on the host: batch from the epoch's sample seed, masks from the step's seed
                seed = eng.drop_seed(eng.steps)
                ob = extract_np.extract_batch(g, tu[idx], tv[idx], tl[idx], cv, 2, 1.0, 200,
                                              seed=splitmix64(eng.sample_seed + ep), pair_ids=idx)
                ref.load_state_dict(sd)
                loss_ref, out_ref = oracle_train_step(ref, ob, 0.001, edge_keep_reference(seed, ob["edge_index"].shape[1],
                                                                                           0.2),
                                                      hidden_keep_reference(seed, len(idx), 0.5))
                ws = next(v for key, v in m._ws.items() if key[2] and key[1] == len(idx))
                assert_step_matches(m, ref, ws["pred"], eng.last_loss, m.flat_grad, loss_ref, out_ref,
                                    "engine epoch %d step %d" % (ep, eng.steps))
        assert eng.exchange is None               # the L2 plan takes the separate gradient assembly + Adam
        assert _lib.l2_csize(next(iter(m._plans.values()))) > 0
        if use_graph:
            assert len(eng.graphs) > 0
    finally:
        eng.close()
    return m.flat_params.clone()


def test_engine_large_subgraphs():
    """two epochs of 300 ml_100k* pairs at h = 2, mnph 200, batch 50: CUDA graphs on and off give bit-identical
    parameters, and so does a second run"""
    p_graph = _engine_run(True, True)
    p_eager = _engine_run(False, False)
    p_again = _engine_run(True, False)
    assert torch.equal(p_graph, p_eager) and torch.equal(p_graph, p_again)


# ---- 10. static dataset -------------------------------------------------------------------------------------------
def test_static_dataset_large():
    """MyDataset (subgraphs extracted once into the device store) on h = 2, mnph 200 pairs"""
    from igmc_b200.util_functions import MyDataset
    ds = _ml_100k()
    tu, tv, tl = [a[:8] for a in ds["train"]]
    cv = ds["class_values"]
    d = MyDataset(None, ds["adj_train"], (tu, tv), tl, 2, 1.0, 200, None, None, cv)
    b = d.extract_batch(np.arange(8))
    ob = extract_np.extract_batch(extract_np.RatingCSR(ds["adj_train"]), tu, tv, tl, cv, 2, 1.0, 200, seed=0,
                                  pair_ids=np.arange(8))
    ref, m = _models(6, 5)
    check_step(m, ref, b, ob, 0.001, 0.2, _hk(8))
    assert _is_l2(m, b)


# ---- 11. the reference's Main.py -----------------------------------------------------------------------------------
def _main_py():
    import os
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "Main.py")
    return p if os.path.isfile(p) else None


@pytest.mark.skipif(_main_py() is None, reason="reference Main.py not available (run oracle/make_ref.py)")
@pytest.mark.parametrize("extra", [["--hop", "2", "--max-nodes-per-hop", "200"], []], ids=["h2_mnph200", "uncapped"])
def test_reference_main_on_large_subgraphs(tmp_path, extra):
    """the reference's unmodified Main.py on 2 000 training pairs over the full ml_100k* matrix
    (tests/main_stubs_large) with the reference's default extraction (no --max-nodes-per-hop: 10000) and with the
    hop-count ablation's h = 2, mnph 200: subgraphs no shared-memory plan takes, trained on the L2 plan.  The stub
    serves that split whatever --data-name says; "ml_1m" only selects Main.py's checkpoint ensemble over epochs
    5..20 (Main.py:438-441; without --ensemble Main.py:472 prints an undefined name after training)."""
    import os
    import re
    import shutil
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([os.path.join(root, "tests", "main_stubs_large"), os.path.join(root, "shims"),
                                         root, env.get("PYTHONPATH", "")])
    env["MPLBACKEND"] = "Agg"
    shutil.copyfile(_main_py(), str(tmp_path / "Main.py"))
    cmd = [sys.executable, "Main.py", "--data-name", "ml_1m", "--testing", "--epochs", "20", "--save-interval", "5",
           "--ensemble", "--keep-old", "--batch-size", "50", "--dynamic-train", "--dynamic-test", "--save-appendix",
           "_l2"] + extra
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + "\n" + r.stderr[-3000:]
    assert "#train: 2000" in r.stdout and "Ensemble test rmse is:" in r.stdout
    res = tmp_path / "results" / "ml_1m_l2_testmode"
    log = (res / "log.txt").read_text().strip().splitlines()
    ep = [l for l in log if re.match(r"Epoch \d+, train loss [\d.]+, test rmse [\d.]+$", l)]
    assert len(ep) == 20, log
    losses = [float(l.split("train loss ")[1].split(",")[0]) for l in ep]
    assert losses[-1] < losses[0]
    for e in (5, 10, 15, 20):
        sd = torch.load(res / ("model_checkpoint%d.pth" % e))
        assert "convs.0.basis" in sd and "lin2.bias" in sd
        assert (res / ("optimizer_checkpoint%d.pth" % e)).is_file()
