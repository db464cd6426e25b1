"""Per-pair gradients and influence on the GPU (igmc_b200/recommend.py pair_gradients / influence / self_influence,
csrc/influence.cu).

* pair_gradients against fp64 autograd on the extractor's own subgraphs, loss seed and score seed, every parameter
  tensor within 2e-4 of its reference's largest entry: plans 1, 2, 4, plan 0 (R = 13), the L2 plan, pyg-2, NB 2, h = 2,
  multiply_by 2, a cold-start pair, a padded tail and B = 1;
* on every plan the per-pair loss gradients of a batch, summed and divided by B, are fused_step(ARR=0)'s flat_grad
  per element within 2 KAPPA["grad"] u M of the batch's magnitude pass (each side is within KAPPA["grad"] u M of the
  same fp64 value); the per-element bounds of each pair's own gradient are in tests/test_gpu_pair_grad_bounds.py;
* influence and self_influence per element within kappa_infl * 2^-24 * M of fp64 dot products of the kernel's own
  per-pair gradients; the order, top-k truncation, determinism across B / graph replay / runs, checkpoints, no host
  sync in the steady state, graph updates and DGCNN_RS."""
import os
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.util_functions import RatingGraph, SubgraphExtractor
from oracle import extract_np
from tests import error_bounds as eb
from tests import pyg2_oracle
from tests.helpers import batch_equal
from tests.test_gpu_explain import _ds, _model, _pairs, _r13, _subgraph, _with_cold_start

pytestmark = pytest.mark.gpu

KAPPA_INFL = 16.0     # the smallest power of two at least 4x the largest ratio measured on an H100 (DESIGN §13)


def _mk(R, h=1, rgcn="pyg-1.4", NB=4, mb=1, plan="auto", seed=0):
    from igmc_b200.models import IGMC
    torch.manual_seed(seed)
    m = IGMC(2 * h + 2, latent_dim=[32] * 4, num_relations=R, num_bases=NB, regression=True, rgcn=rgcn,
             multiply_by=mb)
    if rgcn == "pyg-2":
        with torch.no_grad():
            for c in m.convs:
                c.bias.uniform_(-0.3, 0.3)
    m = m.cuda()
    m.kernel_plan = plan
    return m


def _entries(m):
    """parameter name -> layout entry of the flat bucket"""
    ent = {id(p): e for e, (_, _, p) in zip(m._layout, m._named_order())}
    return {n: ent[id(p)] for n, p in m.named_parameters()}


def _ref_grads(m, R, h, rgcn, NB, mb, sub, y):
    """fp64 autograd of (f - y)^2 (y given) or f on the restated model: name -> gradient"""
    x, ei, et, _ = sub
    ref = pyg2_oracle.igmc_ref(rgcn, 2 * h + 2, (32,) * 4, R, NB, 0.0, mb)
    ref.load_state_dict({k: v.double().cpu() for k, v in m.state_dict().items()})
    ref = ref.double().cuda().eval()
    f = ref(x.double(), ei, et).sum()
    q = (f - y) ** 2 if y is not None else f
    names = [n for n, _ in ref.named_parameters()]
    gs = torch.autograd.grad(q, [p for _, p in ref.named_parameters()], allow_unused=True)
    return {n: (torch.zeros_like(p) if g is None else g) for (n, p), g in zip(ref.named_parameters(), gs)}, names


CASES = {
    # name: (dataset, R, h, mnph, NB, rgcn, multiply_by, plan, batch size)
    "plan 1": ("ml_1m", 5, 1, 100, 4, "pyg-1.4", 1, 1, 64),
    "plan 2 pyg-2": ("ml_1m", 5, 1, 100, 4, "pyg-2", 1, 2, 64),
    "plan 4 NB=2": ("ml_1m", 5, 1, 100, 2, "pyg-1.4", 1, 4, 64),
    "plan 0 R=13 padded tail": ("r13", 13, 1, 50, 4, "pyg-1.4", 1, 0, 2),
    "L2 plan multiply_by 2": ("ml_1m", 5, 1, 100, 4, "pyg-1.4", 2, _lib.plan_l2(2), 64),
    "h=2 B=1": ("ml_1m", 5, 2, 20, 4, "pyg-2", 1, "auto", 1),
}


@pytest.mark.parametrize("name", list(CASES))
def test_pair_gradients_match_fp64_autograd(name):
    dsn, R, h, mnph, NB, rgcn, mb, plan, B = CASES[name]
    A = _with_cold_start(_r13() if dsn == "r13" else _ds(dsn)["adj_train"])
    m = _mk(R, h, rgcn, NB, mb, plan)
    u, v = _pairs(A)
    y = np.array([3.0, 1.0, 5.0])
    seed = 5
    ent = _entries(m)
    for yy in (y, None):
        G = rc.pair_gradients(m, A, u, v, yy, h=h, max_nodes_per_hop=mnph, batch_size=B, sample_seed=seed)
        assert G.shape == (1, 3, m._cmodel.param_count) and m.kernel_plan == plan
        for q in range(3):
            sub, _ = _subgraph(A, R, int(u[q]), int(v[q]), h, mnph, seed)
            want, names = _ref_grads(m, R, h, rgcn, NB, mb, sub, None if yy is None else float(yy[q]))
            for n in names:
                got = m._pview(G[0, q], ent[n]).double()
                w = want[n]
                scale = float(w.abs().max())
                err = float((got - w).abs().max())
                assert err <= 2e-4 * scale or (scale == 0 and err == 0), (name, q, n, err, scale)


def _train_batch(A, R, u, v, lab, mnph, seed, B):
    ni = A.shape[1]
    ex = SubgraphExtractor(RatingGraph(A), [0], [0], [0], np.arange(1, R + 1, dtype=np.float32), 1, 1.0, mnph,
                           max_batch=B, seed=seed)
    return ex.extract(pairs=(u, v, lab), pair_ids=u.astype(np.int64) * ni + v)


@pytest.mark.parametrize("plan", [1, 2, 4, 0, _lib.plan_l2(2)])
def test_pair_gradients_sum_to_the_train_step(plan):
    A = _ds("ml_1m")["adj_train"]
    R = 13 if plan == 0 else 5
    if plan == 0:
        A = _r13()
    m = _mk(R, plan=plan)
    m.adj_dropout, m.hidden_dropout_p = 0.0, 0.0
    coo = A.tocoo()
    rng = np.random.default_rng(1)
    k = rng.choice(A.nnz, 40, replace=False)
    u, v = coo.row[k].astype(np.int64), coo.col[k].astype(np.int64)
    lab = (coo.data[k] - 1).astype(np.int64)
    y = (lab + 1).astype(np.float32)
    b = _train_batch(A, R, u, v, lab, 100, 2, 40)
    assert np.array_equal(b.y.cpu().numpy(), y)
    m.fused_step(b, ARR=0.0)
    want = m.flat_grad.double().cpu()
    # M of the batch gradient: the magnitude pass of the step's own saved tensors on the oracle batch of its pairs
    ni = A.shape[1]
    ob = extract_np.extract_batch(extract_np.RatingCSR(A), u, v, lab, np.arange(1, R + 1, dtype=np.float32), 1, 1.0,
                                  100, seed=2, pair_ids=u * ni + v)
    assert all(batch_equal(b, ob).values())
    ws = next(w for k, w in m._ws.items() if k[1] == 40 and k[2])
    saved = eb.device_saved(m, ws, len(ob["x"]), True)
    params = {k: p.detach().double().cpu() for k, p in m.state_dict().items()}
    aggr = "mean_per_relation" if m.rgcn == "pyg-2" else "mean_all"
    _, mgrads = eb.backward(params, eb.Graph(ob), saved, aggr, False, 0.0, mag=True)
    idx, _, M = eb.flat_terms(m, mgrads, mgrads)
    G = rc.pair_gradients(m, A, u, v, y, max_nodes_per_hop=100, batch_size=40, sample_seed=2)
    got = G[0].double().sum(0).cpu() / 40
    # each side is within KAPPA["grad"] u M of the same fp64 value (tests/test_influence_host.py pins the identity)
    r, pad, worst = eb.ratio(got[idx], want[idx], M)
    print("plan %s: per-pair gradients summed / B against flat_grad, largest err/(u M) %.3f" % (plan, r))
    assert r <= 2 * eb.KAPPA["grad"] and pad == 0, (plan, r, pad, worst)


def _setup(R=5, plan="auto", N=200, T=12, seed=0):
    A = _ds("ml_1m")["adj_train"]
    m = _mk(R, plan=plan, seed=seed)
    coo = A.tocoo()
    rng = np.random.default_rng(3)
    k = rng.choice(A.nnz, N, replace=False)
    train = (coo.row[k], coo.col[k], coo.data[k].astype(np.float32))
    kt = rng.choice(A.nnz, T, replace=False)
    test = (coo.row[kt], coo.col[kt], coo.data[kt].astype(np.float32))
    return A, m, train, test


def _bound_check(got, ref, M, what):
    got = got.double()
    assert torch.isfinite(got).all(), what
    zero = M == 0
    assert torch.equal(got[zero], torch.zeros_like(got[zero])), what
    ratio = ((got - ref).abs() / (M * 2.0 ** -24)).where(~zero, torch.zeros_like(M))
    r = float(ratio.max()) if ratio.numel() else 0.0
    print("%s: largest ratio %.3f (kappa %.1f)" % (what, r, KAPPA_INFL))
    assert r <= KAPPA_INFL, (what, r)


def _ref_infl(Gb, Gt, lrs):
    """fp64 sum_k eta_k <G_b, G_t> and M = sum_k |eta_k| sum_p |g_bp| |g_tp|: [N, T]"""
    ref = sum(e * Gb[k].double() @ Gt[k].double().T for k, e in enumerate(lrs))
    M = sum(abs(e) * Gb[k].double().abs() @ Gt[k].double().abs().T for k, e in enumerate(lrs))
    return ref, M


@pytest.mark.parametrize("labelled", [True, False])
def test_influence_within_the_error_bound_and_in_order(labelled):
    A, m, train, test = _setup()
    N, T = len(train[0]), len(test[0])
    te = test if labelled else test[:2]
    kw = dict(max_nodes_per_hop=100, batch_size=64, sample_seed=1)
    eng = rc.InferenceEngine(m, A, **kw)
    try:
        eng.start_influence(train, te, N)
        while eng.run["phase"] == "test":
            assert eng.step()
        tconv, tfac = eng.run["tconv"].clone(), eng.run["tfac"].clone()
        inf = eng.finish()
    finally:
        eng.close()
    Gt = rc.pair_gradients(m, A, *te, **kw)
    Gb = rc.pair_gradients(m, A, *train, **kw)
    PC = m._cmodel.conv_param_count
    assert torch.equal(tconv[0], Gt[0][:, :PC])              # the pass used pair_gradients' own gradients
    assert torch.equal(tfac[0][:, -1], Gt[0][:, m._cmodel.off_lin2_b])   # dpred: d q_t / d lin2.bias
    ref, M = _ref_infl(Gb, Gt, [1.0])
    got = torch.full((N, T), float("nan"), dtype=torch.float64, device="cuda")
    for t in range(T):
        idx = inf.pro_index[t]
        assert sorted(idx.tolist()) == list(range(N))        # k = N: every training pair listed
        got[idx, t] = inf.pro_value[t].double()
        pi, pv, ci, cv = rc.influence_order_host(got[:, t].float().cpu().numpy(), N)
        assert np.array_equal(inf.pro_index[t].cpu().numpy(), pi)
        assert np.array_equal(inf.con_index[t].cpu().numpy(), ci)
        assert np.array_equal(inf.con_value[t].cpu().numpy(), cv)
    _bound_check(got, ref, M, "influence labelled=%s" % labelled)
    # self-influence: the same bound, and influence of pair i against itself as a labelled test pair
    s = rc.self_influence(m, A, train, **kw)
    sref = (Gb[0].double() ** 2).sum(1)
    _bound_check(s.view(-1, 1), sref.view(-1, 1), sref.view(-1, 1), "self_influence")
    if labelled:
        own = rc.influence(m, A, train, (train[0][:5], train[1][:5], train[2][:5]), N, **kw)
        for i in range(5):
            v = float(own.pro_value[i][own.pro_index[i] == i])
            assert abs(v - float(s[i])) <= 2 * KAPPA_INFL * 2.0 ** -24 * float(sref[i]), i


def test_topk_prefix_determinism_and_graph_replay():
    A, m, train, test = _setup(plan=2)
    kw = dict(max_nodes_per_hop=100, sample_seed=1)
    runs = [rc.influence(m, A, train, test, k, batch_size=B, **kw) for k, B in ((256, 50), (10, 50), (256, 256))]
    eng = rc.InferenceEngine(m, A, batch_size=50, use_graph=False, **kw)
    runs.append(eng.influence(train, test, 256))
    runs.append(eng.influence(train, test, 256))
    eng.close()
    a = runs[0]
    for f in a._fields:
        assert torch.equal(getattr(runs[1], f), getattr(a, f)[:, :10]), f
        for r in runs[2:]:
            assert torch.equal(getattr(r, f), getattr(a, f)), f
    N = len(train[0])
    assert (a.pro_index[:, N:] == -1).all() and (a.pro_value[:, N:] == -float("inf")).all()
    assert (a.con_value[:, N:] == float("inf")).all()
    s1 = rc.self_influence(m, A, train, batch_size=50, **kw)
    s2 = rc.self_influence(m, A, train, batch_size=256, **kw)
    assert torch.equal(s1, s2)


def test_checkpoints_and_the_model_is_left_as_it_was():
    A, m, train, test = _setup(N=60, T=5)
    own = m.flat_params.clone()
    lrs = [0.5, 2.0, -1.0]
    kw = dict(max_nodes_per_hop=100, batch_size=64, sample_seed=1)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for c in range(3):
            paths.append(os.path.join(tmp, "ck%d.pth" % c))
            torch.save(_mk(5, seed=c + 1).state_dict(), paths[-1])
        N = len(train[0])
        ens = rc.influence(m, A, train, test, N, checkpoints=paths, lrs=lrs, **kw)
        s = rc.self_influence(m, A, train, checkpoints=paths, lrs=lrs, **kw)
        Gb = rc.pair_gradients(m, A, *train, checkpoints=paths, **kw)
        Gt = rc.pair_gradients(m, A, *test, checkpoints=paths, **kw)
    assert torch.equal(m.flat_params, own) and m.kernel_plan == "auto"
    ref, M = _ref_infl(Gb, Gt, lrs)
    got = torch.zeros(N, len(test[0]), dtype=torch.float64, device="cuda")
    for t in range(len(test[0])):
        got[ens.pro_index[t], t] = ens.pro_value[t].double()
    _bound_check(got, ref, M, "influence K=3")
    sref = sum(e * (Gb[k].double() ** 2).sum(1) for k, e in enumerate(lrs))
    sM = sum(abs(e) * (Gb[k].double() ** 2).sum(1) for k, e in enumerate(lrs))
    _bound_check(s.double().view(-1, 1), sref.view(-1, 1), sM.view(-1, 1), "self_influence K=3")


def test_steady_state_steps_do_not_sync_and_updates_raise():
    A, m, train, test = _setup(N=120, T=4)
    g = RatingGraph(A, reserve_nnz=100)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=100, batch_size=8, sample_seed=1)
    try:
        eng.start_influence(train, test, 5)
        while eng.run["phase"] == "test":
            assert eng.step()
        for _ in range(4):          # eager warm-up and capture of both slots of the training pass
            assert eng.step()
        assert len(eng.graphs) == 2
        torch.cuda.set_sync_debug_mode("error")
        try:
            while eng.step():
                pass
        finally:
            torch.cuda.set_sync_debug_mode("default")
        eng.finish()
        assert int(eng.extractor.err.item()) == 0
        eng.start_self_influence(train)
        assert eng.step()
        g.update(np.array([0]), np.array([0]), np.array([3]))
        with pytest.raises(RuntimeError):
            eng.step()
    finally:
        eng.close()
    d = _model(5, dgcnn=True)
    with pytest.raises(NotImplementedError):
        rc.pair_gradients(d, A, train[0][:2], train[1][:2])
