"""Scoring and ranking unrated pairs on the GPU (igmc_b200/recommend.py, csrc/recommend.cu).

* the candidate kernels bit for bit against their host twins (tests/test_recommend_host.py), tail padding included;
* predict_pairs against the existing eval forward on the same batches (same pairs, B and pair ids), bit for bit, on
  every kernel plan, h = 2, rgcn="pyg-2" and DGCNN_RS; and against the fp64 restated forward on the oracle's subgraphs;
* recommend against a stable sort of the engine's own scores, across batch sizes, CUDA graphs on / off, users spanning
  several batches and several users per batch; never a rated item with exclude_rated;
* a three-checkpoint ensemble; steady-state steps without a host synchronisation."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from igmc_b200.util_functions import RatingGraph, SubgraphExtractor, _stream_ptr
from oracle import extract_np, pyg_restated
from tests import pyg2_oracle
from tests import support

pytestmark = pytest.mark.gpu


def _mixed_pairs(A, n, seed):
    """n pairs: half unrated, half rated (scored without their target edge)"""
    rng = np.random.default_rng(seed)
    nu, ni = A.shape
    Ad = A.tocoo()
    r = rng.choice(A.nnz, n // 2, replace=False)
    ru, rv = Ad.row[r], Ad.col[r]
    uu, uv = [], []
    rated = set(zip(Ad.row.tolist(), Ad.col.tolist()))
    while len(uu) < n - n // 2:
        a, b = int(rng.integers(nu)), int(rng.integers(ni))
        if (a, b) not in rated:
            uu.append(a)
            uv.append(b)
    u = np.concatenate([ru, uu]).astype(np.int64)
    v = np.concatenate([rv, uv]).astype(np.int64)
    p = rng.permutation(n)
    return u[p], v[p]


def _loop_scores(m, A, u, v, B, h, mnph, seed):
    """the existing path: per-batch extraction of explicit pairs + the eval forward, tail batch padded with the last
    pair so that every batch has the same B"""
    g = RatingGraph(A)
    R = m.num_relations
    ex = SubgraphExtractor(g, [0], [0], [0], np.arange(1, R + 1, dtype=np.float32), h, 1.0, mnph, max_batch=B,
                           seed=seed)
    ni = A.shape[1]
    out = []
    m.eval()
    with torch.no_grad():
        for s in range(0, len(u), B):
            idx = np.minimum(np.arange(s, s + B), len(u) - 1)
            b = ex.extract(pairs=(u[idx], v[idx], np.zeros(B, np.int64)), pair_ids=u[idx] * ni + v[idx])
            out.append(m(b)[:min(B, len(u) - s)].clone())
            b.check()
    return torch.cat(out)


# ---- 1. candidate kernels vs host twins ------------------------------------------------------------------------------
@pytest.mark.parametrize("exclude", [True, False])
@pytest.mark.parametrize("which", ["all", "none", "some", "row"])
def test_candidate_kernels_match_host_twin(which, exclude):
    A = support.adj("ml_100k")
    g = RatingGraph(A)
    rp, ci, ni = g.host["row_ptr"].astype(np.int64), g.host["col_idx"].astype(np.int64), g.num_items
    deg = np.diff(rp)
    empty = int(np.argmin(deg))
    rng = np.random.default_rng(3)
    users = np.array([0, int(np.argmax(deg)), 5, 5, 17, 900] + ([empty] if deg[empty] == 0 else []), np.int64)
    unrated = np.setdiff1d(np.arange(ni), ci)
    cand = dict(all=None, none=unrated[:3] if len(unrated) else np.array([ni - 1]),
                some=np.unique(rng.choice(ni, 300)), row=ci[rp[5]:rp[6]].copy())[which]
    plan = rc.candidate_plan_host(rp, ci, ni, users, cand, exclude)
    eng = rc.InferenceEngine(support.model(5), A, batch_size=64, max_nodes_per_hop=10)
    P = eng.start_recommend(users, 5, items=cand, exclude_rated=exclude)
    assert P == int(plan[0][-1])
    run = eng.run
    assert np.array_equal(run["user_off"].cpu().numpy(), plan[0])
    if plan[1] is not None:
        assert np.array_equal(run["rated_off"].cpu().numpy(), plan[1])
        assert np.array_equal(run["rated_pos"][:len(plan[2])].cpu().numpy(), plan[2])
    if P == 0:
        return
    # every batch of pairs, one past the end (all padding), straight from the kernel
    B = 64
    cursor = torch.zeros(1, dtype=torch.int64, device="cuda")
    s = eng.slots[0]
    for pos in range(0, P + B, B):
        _lib.check(eng.lib.igmc_candidate_pairs(C.byref(eng.graph._c), C.byref(run["Cd"]), cursor.data_ptr(), B,
                                                s["u"].data_ptr(), s["v"].data_ptr(), s["pid"].data_ptr(),
                                                s["tag"].data_ptr(), eng.extractor.err.data_ptr(), _stream_ptr()),
                   "igmc_candidate_pairs")
        want = rc.candidate_pairs_host(rp, ci, ni, users, cand, exclude, plan, pos, B)
        got = np.stack([s[k].cpu().numpy().astype(np.int64) for k in ("u", "v", "pid", "tag")])
        assert np.array_equal(got, want), pos
        assert int(cursor.item()) == pos + B
    assert int(eng.extractor.err.item()) == 0
    eng.close()


# ---- 2. predict_pairs == the existing eval forward ------------------------------------------------------------------
PLANS = {
    # name: (dataset, h, mnph, B, model kwargs, expected plan)
    "relation-space ml_1m": ("ml_1m", 1, 100, 50, {}, 2),
    "plan 4 ml_100k": ("ml_100k", 1, 200, 50, {}, 4),
    "plan 0 R=13": ("r13", 1, 50, 50, {}, 0),
    "L2 plan ml_100k uncapped": ("ml_100k", 1, None, 50, {}, "l2"),
    "h=2": ("ml_1m", 2, 20, 50, {}, None),
    "pyg-2": ("ml_1m", 1, 100, 50, dict(rgcn="pyg-2"), 2),
    "DGCNN_RS": ("ml_1m", 1, 100, 50, dict(dgcnn=True), None),
}


@pytest.mark.parametrize("name", list(PLANS))
def test_predict_pairs_equals_eval_forward(name):
    dsn, h, mnph, B, kw, plan = PLANS[name]
    ds = support.dataset(dsn)
    A = ds["adj_train"]
    m = support.model(ds["num_relations"], h=h, **kw, pyg2_bias=True)
    u, v = _mixed_pairs(A, 2 * B + 17, seed=1)
    got = rc.predict_pairs(m, A, u, v, h=h, max_nodes_per_hop=mnph, batch_size=B, sample_seed=7)
    want = _loop_scores(m, A, u, v, B, h, mnph, 7)
    assert got.shape == (len(u),) and got.dtype == torch.float32
    assert torch.equal(got, want), (name, float((got - want).abs().max()))
    cl = next(iter(m._plans.values()))
    if plan == "l2":
        assert _lib.l2_csize(cl) > 0
    elif plan is not None:
        assert cl == plan, (name, cl)
    # device inputs give the same scores
    got_dev = rc.predict_pairs(m, A, torch.as_tensor(u, device="cuda"), torch.as_tensor(v, device="cuda"), h=h,
                               max_nodes_per_hop=mnph, batch_size=B, sample_seed=7)
    assert torch.equal(got, got_dev)


# ---- 3. against the fp64 restated forward -----------------------------------------------------------------------------
@pytest.mark.parametrize("rgcn", ["pyg-1.4", "pyg-2"])
def test_predict_pairs_against_oracle(rgcn):
    ds = support.dataset("ml_1m")
    A, R, mnph, seed = ds["adj_train"], 5, 100, 7
    m = support.model(R, rgcn=rgcn, pyg2_bias=True)
    ref = pyg2_oracle.igmc_ref(rgcn, 4, (32,) * 4, R, 4, 0.0)
    ref.load_state_dict({k: v.double().cpu() for k, v in m.state_dict().items()})
    ref = pyg_restated.set_formulation(ref.double(), "transform").cuda().eval()
    u, v = _mixed_pairs(A, 120, seed=2)
    got = rc.predict_pairs(m, A, u, v, max_nodes_per_hop=mnph, batch_size=50, sample_seed=seed)
    ni = A.shape[1]
    ob = extract_np.extract_batch(extract_np.RatingCSR(A), u, v, np.zeros(len(u), np.int64),
                                  np.arange(1, R + 1, dtype=np.float32), 1, 1.0, mnph, seed=seed, pair_ids=u * ni + v)
    tb = pyg_restated.to_torch_batch(ob, torch.float64, device="cuda")
    with torch.no_grad():
        out = ref(tb["x"], tb["edge_index"], tb["edge_type"]).cpu()
    rmse = float(torch.sqrt(torch.mean((got.double().cpu() - out) ** 2)))
    print("%s: predict_pairs vs fp64 oracle RMSE %.2e" % (rgcn, rmse))
    assert rmse <= 1e-4, rmse


# ---- 4. top-k ----------------------------------------------------------------------------------------------------------
def _candidates(A, users, cand, exclude):
    ni = A.shape[1]
    base = np.arange(ni) if cand is None else np.unique(cand)
    out = []
    for u in users:
        rated = A.indices[A.indptr[u]:A.indptr[u + 1]]
        out.append(base[~np.isin(base, rated)] if exclude else base)
    return out


def _check_topk(A, users, cand, exclude, ks, scores_of, ti_ts):
    lists = _candidates(A, users, cand, exclude)
    for k in ks:
        ti, ts = ti_ts[k]
        ti, ts = ti.cpu().numpy(), ts.cpu().numpy()
        for j, u in enumerate(users):
            ws, wi = rc.rank_host(scores_of[j], lists[j], k)
            assert np.array_equal(ti[j], wi), (k, j)
            assert np.array_equal(ts[j], ws, equal_nan=True), (k, j)
            if exclude:
                assert not np.isin(ti[j][ti[j] >= 0], A.indices[A.indptr[u]:A.indptr[u + 1]]).any()


def test_recommend_matches_sorted_predictions():
    """ml_1m* full catalogue of 3 users (a user spans many batches) and a 40-item list for 12 users (several users per
    batch); k = 1, 10, 100; B = 50 and 256 on the same plan; CUDA graphs on and off"""
    ds = support.dataset("ml_1m")
    A, mnph = ds["adj_train"], 100
    m = support.model(5)
    m.kernel_plan = 1                      # the same plan at both batch sizes
    cases = [(np.array([3, 10, 4000]), None), (np.arange(100, 112), np.random.default_rng(0).choice(3706, 40))]
    for users, cand in cases:
        lists = _candidates(A, users, cand, True)
        pu = np.concatenate([np.full(len(l_), u) for u, l_ in zip(users, lists)])
        pv = np.concatenate(lists)
        flat = rc.predict_pairs(m, A, pu, pv, max_nodes_per_hop=mnph, batch_size=50, sample_seed=3).cpu().numpy()
        scores_of = np.split(flat, np.cumsum([len(l_) for l_ in lists])[:-1])
        results = {}
        for B in (50, 256):
            for use_graph in (True, False):
                eng = rc.InferenceEngine(m, A, max_nodes_per_hop=mnph, batch_size=B, sample_seed=3,
                                         use_graph=use_graph)
                res = {k: eng.recommend(users, k, items=cand) for k in (1, 10, 100)}
                if use_graph and eng.run is None and len(pv) > 4 * B:
                    assert len(eng.graphs) == 2
                eng.close()
                _check_topk(A, users, cand, True, (1, 10, 100), scores_of, res)
                results[(B, use_graph)] = res
        first = results[(50, True)]
        for key, res in results.items():
            for k in (1, 10, 100):
                assert torch.equal(res[k][0], first[k][0]) and torch.equal(res[k][1], first[k][1]), key
    # the public function, exclude_rated=False: rated items compete too (scored without their target edge)
    users = np.array([7, 8])
    lists = _candidates(A, users, np.arange(50), False)
    ti, ts = rc.recommend(m, A, users, 10, items=np.arange(50), exclude_rated=False, max_nodes_per_hop=mnph,
                          batch_size=50, sample_seed=3)
    flat = rc.predict_pairs(m, A, np.repeat(users, 50), np.tile(np.arange(50), 2), max_nodes_per_hop=mnph,
                            batch_size=50, sample_seed=3).cpu().numpy()
    _check_topk(A, users, np.arange(50), False, (10,), [flat[:50], flat[50:]], {10: (ti, ts)})


def test_recommend_short_lists_pad():
    """a user with fewer candidates than k: item -1 / score -inf in the empty slots; a user who rated every candidate
    gets only empty slots"""
    ds = support.dataset("ml_100k")
    A = ds["adj_train"]
    m = support.model(5)
    u0 = 0
    row = A.indices[A.indptr[u0]:A.indptr[u0 + 1]]
    cand = np.concatenate([row[:3], np.setdiff1d(np.arange(A.shape[1]), row)[:4]])
    ti, ts = rc.recommend(m, A, [u0, u0], 10, items=cand, max_nodes_per_hop=200, batch_size=50)
    ti, ts = ti.cpu().numpy(), ts.cpu().numpy()
    assert (ti[:, 4:] == -1).all() and np.isneginf(ts[:, 4:]).all() and (ti[:, :4] >= 0).all()
    assert np.array_equal(ti[0], ti[1])
    ti, ts = rc.recommend(m, A, [u0], 5, items=row[:3], max_nodes_per_hop=200, batch_size=50)
    assert (ti.cpu().numpy() == -1).all()


# ---- 5. ensemble --------------------------------------------------------------------------------------------------------
def test_ensemble_of_three_checkpoints():
    ds = support.dataset("ml_100k")
    A, mnph = ds["adj_train"], 200
    m = support.model(5)
    u, v = _mixed_pairs(A, 130, seed=4)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for c in range(3):
            mc = support.model(5, seed=c + 1)
            paths.append(os.path.join(tmp, "model_checkpoint%d.pth" % c))
            torch.save(mc.state_dict(), paths[-1])
        own = m.flat_params.clone()
        got = rc.predict_pairs(m, A, u, v, max_nodes_per_hop=mnph, batch_size=50, checkpoints=paths)
        assert torch.equal(m.flat_params, own)          # the model keeps its own parameters
        single = [rc.predict_pairs(m, A, u, v, max_nodes_per_hop=mnph, batch_size=50, checkpoints=[p]) for p in paths]
        ti, ts = rc.recommend(m, A, [1, 2], 20, items=np.arange(60), max_nodes_per_hop=mnph, batch_size=50,
                              checkpoints=paths)
    s = [x.cpu().numpy() for x in single]
    want = ((s[0] + s[1]) + s[2]) / np.float32(3)
    assert np.array_equal(got.cpu().numpy(), want)
    ens = torch.stack(single, 1).mean(1)            # eval_loss_ensemble's averaging
    assert float((got - ens).abs().max()) <= 1e-6
    for mc_single in single:   # each checkpoint on its own is a different model
        assert not torch.equal(mc_single, got)
    assert ti.shape == (2, 20) and (ti[:, 0] >= 0).all()


# ---- 6. steady state: no host synchronisation, repeatable, clean error word ---------------------------------------------
def test_steady_state_steps_do_not_sync():
    ds = support.dataset("ml_1m")
    A = ds["adj_train"]
    m = support.model(5)
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=100, batch_size=50, sample_seed=1)
    outs = []
    try:
        for rep in range(2):
            P = eng.start_recommend([11, 12], 25)
            assert P > 20 * 50
            for _ in range(4):          # eager warm-up and capture of both batch slots
                eng.step()
            assert len(eng.graphs) == 2
            torch.cuda.set_sync_debug_mode("error")
            try:
                while eng.step():
                    pass
            finally:
                torch.cuda.set_sync_debug_mode("default")
            outs.append(eng.finish())
            assert int(eng.extractor.err.item()) == 0
    finally:
        eng.close()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
