"""The paths that real training and evaluation take, against fp64 autograd of oracle/pyg_restated:

* train steps whose hidden dropout is the kernels' own hash draw (no injected mask), checked with its host twin
  ``models.hidden_keep_reference``, on every kernel family: generic plan 0 (csrc/rgcn.cu), the cluster plans and the
  one-launch ``forward_backward`` (csrc/rgcn_rs.cu) and the DGCNN_RS readout (csrc/sortpool.cu); plus the autograd path;
* ``TrainEngine`` driven as ``train()`` drives it, every step rebuilt on the host: the batch from the epoch's sample
  seed, the edge and hidden masks from the step's dropout seed, the gradient the step applied and its loss compared
  with the oracle at the parameters the step started from;
* evaluation at full subgraph size (ml_100k* at mnph 200, flixster, h = 2, DGCNN_RS), with ragged last batches and
  batch size 1, after fused-update training, and with forward edge lists too long to stage.

Bars as everywhere in the suite: ratings within 1e-4 RMSE, losses within 1e-4 relative, gradients within 2e-4 of the
tensor's largest reference entry (DGCNN_RS: tests/helpers.py assert_step_matches), RMSE within 1e-4 absolute."""
import functools
import math

import numpy as np
import pytest
import torch

from igmc_b200.data import load_flixster, make_synthetic_dataset, synth_ratings
from igmc_b200.models import edge_keep_reference, hidden_keep_reference, splitmix64
from oracle import extract_np, pyg_restated
from tests.helpers import REGIMES, assert_step_matches, check_step, oracle_train_step
from tests.test_gpu_regimes import _dense, _dense_block_matrix, _matrix, _ml_100k, _models, _small_batch

pytestmark = pytest.mark.gpu


# ---- A. the kernels' own hidden dropout -----------------------------------------------------------------------------
@pytest.mark.parametrize("plan", [0, 1, 2, 4])
def test_train_step_own_hidden_dropout(plan):
    """fused_step with no injected mask: edge and hidden dropout are both the hash draws of the step's seed"""
    b, ob = _small_batch()
    ref, m = _models(4, 5, plan=plan)
    check_step(m, ref, b, ob, 0.001, 0.2, None)
    assert m._plan(b) == plan


@pytest.mark.parametrize("plan", [0, 2])
def test_dgcnn_rs_step_own_hidden_dropout(plan):
    """the SortPooling readout draws its hidden dropout in csrc/sortpool.cu"""
    b, ob = _small_batch()
    ref, m = _models(4, 5, plan=plan, dgcnn_k=30)
    check_step(m, ref, b, ob, 0.001, 0.2, None)
    assert m._plan(b) == plan


def test_one_launch_step_own_hidden_dropout(monkeypatch):
    """forward_backward as one launch (igmc_forward_backward, what TrainEngine runs) + igmc_grad_reduce"""
    monkeypatch.setenv("IGMC_FUSED_FB", "1")
    b, ob = _small_batch()
    ref, m = _models(4, 5, plan=2)
    launched = []
    one = m._launch_train
    monkeypatch.setattr(m, "_launch_train", lambda *a: launched.append(1) or one(*a))
    B, E = ob["num_graphs"], ob["edge_index"].shape[1]
    m._step = 30
    seed = splitmix64(m.drop_seed + 31)            # forward_backward draws after its _step += 1
    loss_ref, out_ref = oracle_train_step(ref, ob, 0.001, edge_keep_reference(seed, E, 0.2),
                                          hidden_keep_reference(seed, B, 0.5))
    saved = m.forward_backward(b)
    m._launch_grad_reduce(b, saved, loss_scale=1.0 / B, arr=0.001)
    b.check()
    assert launched and m._step == 31
    assert_step_matches(m, ref, saved["ws"]["pred"], saved["ws"]["loss"], m.flat_grad, loss_ref, out_ref, "one launch")


@pytest.mark.parametrize("plan", [0, 2])
def test_autograd_step_draws_before_counting_the_step(plan):
    """``m(b)`` in train mode + ``backward``: forward builds its dropout from ``_step`` BEFORE ``_step += 1``"""
    b, ob = _small_batch()
    ref, m = _models(4, 5, plan=plan)
    B, E = ob["num_graphs"], ob["edge_index"].shape[1]
    m._step = 30
    seed = splitmix64(m.drop_seed + 30)
    loss_ref, out_ref = oracle_train_step(ref, ob, 0.0, edge_keep_reference(seed, E, 0.2),
                                          hidden_keep_reference(seed, B, 0.5))
    m.zero_grad()
    out = m(b)
    assert m._step == 31
    loss = torch.nn.functional.mse_loss(out, b.y)
    loss.backward()
    b.check()
    grad = torch.zeros_like(m.flat_params)
    for e, (_, _, p) in zip(m._layout, m._named_order()):
        m._pview(grad, e).copy_(p.grad)
    assert_step_matches(m, ref, out.detach(), loss.detach(), grad, loss_ref, out_ref, "autograd")


# ---- B. TrainEngine step by step ------------------------------------------------------------------------------------
def _sliced_dataset_class():
    from igmc_b200.util_functions import MyDataset

    class SlicedDataset(MyDataset):
        """a static dataset that also carries PyG's ``slices``: TrainEngine trains it through ``step`` ->
        ``_launch_static`` (no pipeline, no CUDA graph; the dropout seed comes from the model's step count)"""
        slices = None
    return SlicedDataset


# name -> what differs from the default: fused update kernel, CUDA graphs, zero-copy step I/O, 40 training pairs
# (five full batches of 8), the "auto" kernel plan (cluster plan 4 at these shapes), IGMC, dynamic extraction
ENGINE_CASES = {
    "default": dict(),
    "separate_update": dict(fused=False),
    "eager": dict(graph=False),
    "no_zero_copy": dict(zc=False),
    "separate_update_no_zero_copy": dict(fused=False, zc=False),
    "ragged_last_batch": dict(n=44),
    "plan0": dict(plan=0),
    "dgcnn_rs": dict(dgcnn=True),
    "static_store": dict(static="store"),
    "static_sliced": dict(static="sliced"),
}


@pytest.mark.parametrize("case", sorted(ENGINE_CASES))
def test_engine_steps_match_oracle(case, monkeypatch):
    """two epochs of TrainEngine as ``train()`` runs them (prime + step_pipe, or step for a sliced dataset); after
    every step the applied gradient and the loss against the oracle at the parameters the step started from"""
    from igmc_b200.models import FusedAdam
    from igmc_b200.train_eval import TrainEngine, shard_batches
    from igmc_b200.util_functions import MyDataset, MyDynamicDataset
    c = dict(dict(fused=True, graph=True, zc=True, n=40, plan="auto", dgcnn=False, static=None), **ENGINE_CASES[case])
    monkeypatch.setenv("IGMC_ZERO_COPY", "1" if c["zc"] else "0")
    ds = make_synthetic_dataset("tiny", seed=0)
    n, cv, B = c["n"], ds["class_values"], 8
    tu, tv, tl = [a[:n] for a in ds["train"]]
    cls = {None: MyDynamicDataset, "store": MyDataset, "sliced": _sliced_dataset_class()}[c["static"]]
    d = cls(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, 10, None, None, cv)
    ref, m = _models(4, 5, plan=c["plan"], dgcnn_k=10 if c["dgcnn"] else None)
    opt = FusedAdam(m, lr=1e-3)
    if c["fused"]:   # the update kernel also writes the assembled gradient it applied into flat_grad
        monkeypatch.setattr(opt, "reduce_update", functools.partial(FusedAdam.reduce_update, opt, grad_copy=m.flat_grad))
    eng = TrainEngine(d, m, opt, B, ARR=0.001, use_graph=c["graph"], sample_seed=5)
    eng.fused_update = c["fused"]
    assert eng.zero_copy == c["zc"] and eng.pipelined() == (c["static"] != "sliced")
    g = extract_np.RatingCSR(ds["adj_train"])
    gen = torch.Generator().manual_seed(3)
    worst = [0.0, 0.0]
    try:
        for ep in (1, 2):
            batches = shard_batches(torch.randperm(n, generator=gen).numpy(), B, 0, 1)
            if eng.pipelined():
                eng.prime(batches[0][0], ep, batches[0][1])
            for k, (idx, G) in enumerate(batches):
                sd = {key: v.detach().double().cpu().clone() for key, v in m.state_dict().items()}
                if eng.pipelined():
                    nxt = batches[k + 1] if k + 1 < len(batches) else None
                    eng.step_pipe(nxt[0] if nxt else None, ep, nxt[1] if nxt else None)
                    seed = eng.drop_seed(eng.steps)
                else:
                    eng.step(idx, epoch=ep, G=G)
                    seed = splitmix64(m.drop_seed + m._step)     # fused_step of _launch_static
                torch.cuda.synchronize()
                eng.check()
                nb = len(idx)
                # static datasets were extracted once with the dataset's seed (0); the engine's sample seed is per epoch
                sample_seed = 0 if c["static"] else splitmix64(eng.sample_seed + ep)
                ob = extract_np.extract_batch(g, tu[idx], tv[idx], tl[idx], cv, 1, 1.0, 10, seed=sample_seed,
                                              pair_ids=idx)
                if eng.pipelined():   # the buffers the step trained on (a replay does not refresh eng.batches)
                    trained = d.extractor._out_cache[(nb, eng.slot ^ 1)]
                    assert torch.equal(trained["y"][:nb].cpu(), torch.from_numpy(ob["y"].astype(np.float32)))
                    assert np.array_equal(np.diff(trained["node_ptr"][:nb + 1].cpu().numpy()),
                                          np.bincount(ob["batch"], minlength=nb))
                ref.load_state_dict(sd)
                E = ob["edge_index"].shape[1]
                loss_ref, out_ref = oracle_train_step(ref, ob, 0.001, edge_keep_reference(seed, E, 0.2),
                                                      hidden_keep_reference(seed, nb, 0.5))
                ws = next(v for key, v in m._ws.items() if key[2] and key[1] == nb)
                pred = ws["sp"]["pred"] if "sp" in ws else ws["pred"]
                tag = "%s epoch %d step %d" % (case, ep, eng.steps)
                r = assert_step_matches(m, ref, pred, eng.last_loss, m.flat_grad, loss_ref, out_ref, tag)
                worst = [max(a, x) for a, x in zip(worst, r)]
                if eng.exchange is not None and c["zc"]:     # the update kernel also stores it in the pinned ring
                    assert eng.loss_of_update(eng._updates - 1) == float(eng.last_loss)
        assert eng.steps == 2 * len(batches)
        # the fused update kernel needs a cluster plan, the IGMC readout and the pipelined engine
        assert (eng.exchange is not None) == (c["fused"] and c["plan"] != 0 and not c["dgcnn"] and eng.pipelined())
        if c["graph"] and eng.pipelined():
            assert len(eng.graphs) > 0
        print("%s: worst prediction RMSE %.2e, worst relative gradient error %.2e" % (case, worst[0], worst[1]))
    finally:
        eng.close()


# ---- C. evaluation at full size -------------------------------------------------------------------------------------
def _oracle_eval(ref, ob):
    """eval-mode predictions of the restated model (moved to the GPU, still fp64: full-size batches are large) and
    the ratings, on the host"""
    tb = pyg_restated.to_torch_batch(ob, torch.float64, device="cuda")
    ref = ref.cuda().eval()
    with torch.no_grad():
        if isinstance(ref, pyg_restated.DGCNN_RSRef):
            out = ref(tb["x"], tb["edge_index"], tb["edge_type"], tb["batch"], num_graphs=tb["num_graphs"])
        else:
            out = ref(tb["x"], tb["edge_index"], tb["edge_type"])
    return out.cpu(), tb["y"].cpu()


def _dataset_and_oracle(A, pairs, cv, h, mnph, seed=9):
    from igmc_b200.util_functions import MyDynamicDataset
    pu, pv, pl = [np.asarray(x, np.int64) for x in pairs]
    d = MyDynamicDataset(None, A, (pu, pv), pl, h, 1.0, mnph, None, None, cv, seed=seed)
    ob = extract_np.extract_batch(extract_np.RatingCSR(A), pu, pv, pl, cv, h, 1.0, mnph, seed=seed,
                                  pair_ids=np.arange(len(pu)))
    return d, ob


def _check_eval(m, d, pred_ref, y, batch_sizes, tag):
    """per-pair eval predictions, eval_rmse, eval_loss and test_once of ``m`` on ``d`` against the oracle's"""
    from igmc_b200.train_eval import eval_loss, eval_rmse, test_once
    mse_ref = float(((pred_ref - y) ** 2).mean())
    for bs in batch_sizes:
        m.eval()
        preds = []
        with torch.no_grad():
            for s in range(0, len(d), bs):
                preds.append(m(d.extract_batch(np.arange(s, min(s + bs, len(d))))).double().cpu())
        p = torch.cat(preds)
        assert p.shape == pred_ref.shape
        rmse_p = float(torch.sqrt(torch.mean((p - pred_ref) ** 2)))
        assert rmse_p <= 1e-4, (tag, bs, rmse_p)
        got = eval_rmse(m, d, None, batch_size=bs)
        assert abs(got - math.sqrt(mse_ref)) <= 1e-4, (tag, bs, got, math.sqrt(mse_ref))
        loss = eval_loss(m, d, None, True, batch_size=bs)
        assert abs(loss - mse_ref) <= 1e-4 * max(1.0, mse_ref), (tag, bs, loss, mse_ref)
        once = test_once(d, m, bs)
        assert abs(once - math.sqrt(mse_ref)) <= 1e-4, (tag, bs, once, math.sqrt(mse_ref))
        print("%s batch %d: prediction RMSE %.2e, |eval RMSE - oracle| %.2e (oracle RMSE %.4f)"
              % (tag, bs, rmse_p, abs(got - math.sqrt(mse_ref)), math.sqrt(mse_ref)))


def _eval_data(case):
    """(rating matrix, 150 test pairs, class values, h, mnph, R) of one full-size evaluation case"""
    if case == "flixster":
        ds, h, mnph = load_flixster(), 1, 10000
    else:
        ds = _ml_100k()
        h, mnph = {"ml_100k_mnph200": (1, 200), "ml_100k_h2": (2, 40), "dgcnn_rs_ml_100k": (1, 100)}[case]
    eu, ev, el = [a[:150] for a in ds["test"]]
    return ds["adj_train"], (eu, ev, el), ds["class_values"], h, mnph, len(ds["class_values"])


@pytest.mark.parametrize("case", ["ml_100k_mnph200", "flixster", "ml_100k_h2", "dgcnn_rs_ml_100k"])
def test_eval_full_size_matches_oracle(case):
    """150 test pairs: a ragged last batch at batch size 32, and batch size 1"""
    A, pairs, cv, h, mnph, R = _eval_data(case)
    d, ob = _dataset_and_oracle(A, pairs, cv, h, mnph)
    ref, m = _models(2 * h + 2, R, dgcnn_k=30 if case.startswith("dgcnn") else None)
    ref.eval()
    pred_ref, y = _oracle_eval(ref, ob)
    if case == "ml_100k_mnph200":
        assert d.extractor.cap * 2 == 402
    _check_eval(m, d, pred_ref, y, (32, 1), case)
    if case == "ml_100k_mnph200":
        assert m._plan(d.extract_batch(np.arange(32))) == 4


def test_ensemble_eval_full_size(tmp_path):
    """eval_rmse_ensemble of three reference-format checkpoints on ml_100k* at mnph 200 (ragged last batch)"""
    from igmc_b200.models import IGMC
    from igmc_b200.train_eval import eval_rmse_ensemble
    A, pairs, cv, h, mnph, R = _eval_data("ml_100k_mnph200")
    d, ob = _dataset_and_oracle(A, pairs, cv, h, mnph)
    ckpts, preds = [], []
    for k in range(3):
        torch.manual_seed(100 + k)
        ref = pyg_restated.IGMCRef(4, (32, 32, 32, 32), 5, 4, 0.2)
        path = tmp_path / "model_checkpoint{}.pth".format(k)
        torch.save(ref.state_dict(), path)
        ckpts.append(str(path))
        pred, y = _oracle_eval(ref.double().eval(), ob)
        preds.append(pred)
    want = math.sqrt(float(((torch.stack(preds, 1).mean(1) - y) ** 2).mean()))
    m = IGMC(d, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True, adj_dropout=0.2).cuda()
    got = eval_rmse_ensemble(m, ckpts, d, None, batch_size=32)
    print("ensemble: |RMSE - oracle| %.2e (oracle RMSE %.4f)" % (abs(got - want), want))
    assert abs(got - want) <= 1e-4, (got, want)


def test_eval_after_fused_update_training():
    """eval right after TrainEngine's fused update (whose kernel re-prepares W_r and lets the next forward skip
    prep_weights): the oracle at the current parameters, and bit for bit a fresh model loaded from state_dict()"""
    from igmc_b200.models import IGMC, FusedAdam
    from igmc_b200.train_eval import TrainEngine, eval_rmse
    from igmc_b200.util_functions import MyDynamicDataset
    ds = make_synthetic_dataset("tiny", seed=0)
    tu, tv, tl = [a[:40] for a in ds["train"]]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, 10, None, None, ds["class_values"])
    ref, m = _models(4, 5)
    opt = FusedAdam(m, lr=1e-2)
    eng = TrainEngine(d, m, opt, 8, ARR=0.001)
    try:
        eng.prime(np.arange(0, 8), epoch=1)
        for s in range(5):
            eng.step_pipe(np.arange((s + 1) * 8, (s + 2) * 8) if s < 4 else None, epoch=1)
        eng.check()
        assert eng.exchange is not None and m._prepped
    finally:
        eng.close()
    eu, ev, el = [a[:60] for a in ds["test"]]
    test, ob = _dataset_and_oracle(ds["adj_train"], (eu, ev, el), ds["class_values"], 1, 10)
    got = eval_rmse(m, test, None, batch_size=16)
    assert m._plan(test.extract_batch(np.arange(16))) > 0
    ref.load_state_dict({k: v.double().cpu() for k, v in m.state_dict().items()})
    pred_ref, y = _oracle_eval(ref.eval(), ob)
    want = math.sqrt(float(((pred_ref - y) ** 2).mean()))
    print("eval after training: |RMSE - oracle| %.2e (oracle RMSE %.4f)" % (abs(got - want), want))
    assert abs(got - want) <= 1e-4, (got, want)
    fresh = IGMC(test, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True, adj_dropout=0.2).cuda()
    fresh.load_state_dict(m.state_dict())
    fresh.kernel_plan = m.kernel_plan
    assert eval_rmse(fresh, test, None, batch_size=16) == got


def _header_rows(m, b):
    """forward list-image headers [entries, -, staged, own nodes] of an eval-mode staging of ``b`` and its capacity"""
    st = m.stage_batch(b, training=False)
    assert set(st) == {"fwd"}
    img, t = st["fwd"]
    return t["tab"][:, :4].cpu().numpy(), img.lcap


def test_eval_forward_on_global_lists():
    """R = 5, plan 1, n_cap 202: a pair inside the fully rated 101 x 101 block has all its ~20 400 in-entries on one
    CTA, beyond the forward's list capacity, so the eval forward gathers from global memory (``Ls.lst == nullptr``)"""
    r = REGIMES["fwd_global_eval"]
    A, (u, v, lab) = _dense_block_matrix(r["R"])
    blk = np.nonzero((u < 101) & (v < 101))[0]
    bg = np.nonzero(u >= 101)[0]
    pick = np.array([blk[17], bg[0], blk[5000], bg[1], blk[9999]])
    d, ob = _dataset_and_oracle(A, (u[pick], v[pick], lab[pick]), np.arange(1, 6, dtype=np.float32), 1, 100)
    ref, m = _models(4, r["R"], plan=r["plan"])
    ref.eval()
    m.eval()
    b = d.extract_batch(np.arange(len(pick)))
    assert b._priv["n_cap"] == r["n_cap"]
    hdr, lcap = _header_rows(m, b)
    inblk = np.array([0, 2, 4])
    assert np.all(hdr[inblk, 2] == 0) and np.all(hdr[inblk, 0] >= r["entries"]) and lcap < r["entries"], (hdr, lcap)
    pred_ref, y = _oracle_eval(ref, ob)
    with torch.no_grad():
        staged = m(b).double().cpu()            # on the images of stage_batch
        b._stage = None
        own = m(b).double().cpu()               # staged by the forward kernel itself
    b.check()
    for p in (staged, own):
        rmse = float(torch.sqrt(torch.mean((p - pred_ref) ** 2)))
        assert rmse <= 1e-4, rmse
    _check_eval(m, d, pred_ref, y, (2,), "fwd_global_eval")


def test_eval_hinted_lists_overflow_to_global():
    """mnph 200 (n_cap 402, plan 4): the model first sees a sparse ml_100k*-sized batch, which sizes its list buffers
    (list_hint); then it evaluates pairs inside a fully rated 201 x 201 block, 18 000 - 21 000 in-entries on each of
    the 4 CTAs - above the 16 384 entries any hint can buy"""
    from igmc_b200.train_eval import eval_rmse
    r = REGIMES["fwd_global_eval_hinted"]
    R = r["R"]
    cv = np.arange(1, R + 1, dtype=np.float32)
    bu, bv, bl = synth_ratings(700, 1400, 50000, num_classes=R, seed=6)
    A, (u, v, lab) = _matrix([_dense(201, 201, 1.1, R, 7), (bu + 201, bv + 201, bl)], 901, 1601)
    sparse = np.nonzero(u >= 201)[0][:16]
    blk = np.nonzero(u < 201)[0][[5, 999, 20000, 40000]]
    pick = np.concatenate([blk, sparse[:4]])
    ds_sparse, ob_sparse = _dataset_and_oracle(A, (u[sparse], v[sparse], lab[sparse]), cv, 1, 200)
    ds_blk, ob_blk = _dataset_and_oracle(A, (u[pick], v[pick], lab[pick]), cv, 1, 200)
    ref, m = _models(4, R)
    pred_ref, y = _oracle_eval(ref, ob_sparse)
    got = eval_rmse(m, ds_sparse, None, batch_size=8)      # (test_once would re-flatten the model: a new hint)
    assert abs(got - math.sqrt(float(((pred_ref - y) ** 2).mean()))) <= 1e-4
    hint = int(m._cmodel.list_hint)
    assert hint > 0
    b = ds_blk.extract_batch(np.arange(8))
    assert b._priv["n_cap"] == r["n_cap"] and m._plan(b) == r["plan"]
    m.eval()
    hdr, lcap = _header_rows(m, b)
    rows = hdr.reshape(8, r["plan"], 4)[:4]     # the 4 block pairs, all their CTAs
    assert np.all(rows[..., 2] == 0) and np.all(rows[..., 0] >= r["entries"]) and lcap < r["entries"], (hdr, lcap)
    pred_ref, y = _oracle_eval(ref, ob_blk)
    _check_eval(m, ds_blk, pred_ref, y, (8,), "block after hint")
