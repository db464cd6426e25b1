"""The train engine's steps under the per-element fp32 error bounds of tests/error_bounds.py.

``TrainEngine`` runs as ``train()`` runs it (prime + step_pipe: pipelined extraction, pre-staged list images, CUDA
graph replay, zero-copy step I/O).  Before every step the parameters, both Adam moments and the step counter are
snapshot; after it:

* the step's states, predictions, ``d hid`` and gradient against fp64 from the snapshot parameters, on the oracle
  batch of the engine's sample seed and the edge / hidden masks of its dropout seed (``check_device(params=...)``);
* the Adam update per element against ``adam_terms`` (fp64 from the snapshot and the gradient the step applied), and
  the step counter exactly;
* after a fused update (``igmc_reduce_update``, which also prepares the next step's weights): every prepared W_r and
  W_r^T entry against fp64 from the new parameters, root columns copied exactly, padding exactly zero.

IGMC at 5 to 8 layers needs more blocks for the fused kernel than an H100 holds at once; the engine must take the
separate kernels (gradient assembly, then ``igmc_adam_step``) there even when the fused update is on."""
import ctypes
import functools

import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200.data import make_synthetic_dataset
from igmc_b200.models import edge_keep_reference, hidden_keep_reference, splitmix64
from oracle import extract_np
from tests import error_bounds as eb
from tests.test_gpu_error_bounds import _report
from tests.test_gpu_regime_bounds import build_model, case

pytestmark = pytest.mark.gpu

# name -> what differs from R = 5, L = 4, fused update on, PyG 1.4 conv, a fresh optimizer (steps 1..4, bias
# corrections far from 1) and no weight decay.  resume: Adam state loaded at step 5000 with weight decay 1e-2 and the
# lr lowered through sync_lr between two replays.  Four steps, so that a step's graph key repeats and a captured
# CUDA graph runs (asserted at the end)
ENGINE_CASES = {
    **{"L%d_%s" % (L, "fused" if f else "separate"): dict(L=L, fused=f) for L in (1, 4, 5, 8) for f in (True, False)},
    "R8_fused": dict(R=8),
    "pyg2_fused": dict(rgcn="pyg-2"),
    "resumed_5000_fused": dict(resume=True),
    "resumed_5000_separate": dict(resume=True, fused=False),
}
B, ARR, SAMPLE_SEED = 8, 0.001, 5


def _resume(opt, m):
    """Adam state at step 5000 with moments of a plausible size (|m| ~ 1e-3, v ~ (1.5 m)^2)"""
    sd = opt.state_dict()
    gen = torch.Generator().manual_seed(7)
    for st in sd["state"].values():
        ea = torch.randn(st["exp_avg"].shape, generator=gen) * 1e-3
        st.update(step=torch.tensor(5000.0), exp_avg=ea, exp_avg_sq=(1.5 * ea) ** 2 + 1e-8)
    opt.load_state_dict(sd)


@pytest.mark.parametrize("name", list(ENGINE_CASES))
def test_engine_step_bounds(name, monkeypatch):
    from igmc_b200.models import FusedAdam
    from igmc_b200.train_eval import TrainEngine
    from igmc_b200.util_functions import MyDynamicDataset
    c = dict(dict(L=4, R=5, fused=True, rgcn="pyg-1.4", resume=False), **ENGINE_CASES[name])
    monkeypatch.setenv("IGMC_ZERO_COPY", "1")
    ds = make_synthetic_dataset("tiny", seed=0)
    cv = ds["class_values"]
    tu, tv, tl = ds["train"]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, 10, None, None, cv)
    R = c["R"]    # R = 8 on 5 rating levels: relations 5..7 have no edge, their tiles still run
    m = build_model(case(None, R=R, L=c["L"], rgcn=c["rgcn"], plan="auto"))
    wd = 1e-2 if c["resume"] else 0.0
    opt = FusedAdam(m, lr=1e-3, weight_decay=wd)
    if c["resume"]:
        _resume(opt, m)
    if c["fused"]:   # the update kernel also writes the assembled gradient it applied into flat_grad
        monkeypatch.setattr(opt, "reduce_update", functools.partial(FusedAdam.reduce_update, opt, grad_copy=m.flat_grad))
    eng = TrainEngine(d, m, opt, B, ARR=ARR, sample_seed=SAMPLE_SEED)
    eng.fused_update = c["fused"]
    g = extract_np.RatingCSR(ds["adj_train"])
    b1, b2 = opt.param_groups[0]["betas"]
    eps = opt.param_groups[0]["eps"]
    steps, bad = 4, []
    try:
        eng.prime(np.arange(0, B), epoch=1)
        for s in range(steps):
            if c["resume"] and s == 2:
                opt.param_groups[0]["lr"] = 2e-4
                eng.sync_lr()
            idx = np.arange(s * B, (s + 1) * B)
            sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
            p0, m0, v0 = m.flat_params.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone()
            step0 = int(opt.step_count[0])
            eng.step_pipe(np.arange((s + 1) * B, (s + 2) * B) if s < steps - 1 else None, epoch=1)
            torch.cuda.synchronize()
            eng.check()
            tag = "%s step %d" % (name, step0 + 1)
            assert _lib.is_rs(m._plan(eng.batches[eng.slot ^ 1]))
            ob = extract_np.extract_batch(g, tu[idx], tv[idx], tl[idx], cv, 1, 1.0, 10,
                                          seed=splitmix64(eng.sample_seed + 1), pair_ids=idx)
            trained = d.extractor._out_cache[(B, eng.slot ^ 1)]
            assert torch.equal(trained["y"][:B].cpu(), torch.from_numpy(ob["y"].astype(np.float32)))
            seed = eng.drop_seed(eng.steps)
            ek = edge_keep_reference(seed, ob["edge_index"].shape[1], m.adj_dropout)
            hk = hidden_keep_reference(seed, B, m.hidden_dropout_p)
            ws = next(v for k, v in m._ws.items() if k[2] and k[1] == B)
            bad += _report(tag, "step", eb.check_device(m, ob, ws, True, ek, ARR, hk, params=sd))
            # the update the step applied to the snapshot, with the gradient it assembled
            assert int(opt.step_count[0]) == step0 + 1
            terms = eb.adam_terms(p0.cpu(), m0.cpu(), v0.cpu(), m.flat_grad.cpu(), step0 + 1,
                                  opt.param_groups[0]["lr"], b1, b2, eps, wd)
            got = [t.cpu() for t in (opt.exp_avg, opt.exp_avg_sq, m.flat_params)]
            bad += _report(tag, "adam", eb.adam_check(got, terms))
            if eng.exchange is not None:     # the fused kernel prepared the next step's weights
                assert m._prepped
                bad += _report(tag, "wprep", eb.wprep_check(m._wprep_buf(), eb.wprep_terms(
                    m.state_dict(), c["L"], R, m._cmodel.in_dim0)))
        # the one-kernel update where its grid is resident (<= 4 layers at in0 4 on an H100), the separate kernels
        # otherwise
        blocks, resident = ctypes.c_int(), ctypes.c_int()
        assert _lib.load().igmc_reduce_update_grid(ctypes.byref(m._cmodel), ctypes.byref(blocks),
                                                   ctypes.byref(resident)) == 0
        assert (eng.exchange is not None) == (c["fused"] and blocks.value <= resident.value)
        if c["fused"] and c["L"] >= 5:
            assert blocks.value > resident.value
        assert len(eng.graphs) > 0
    finally:
        eng.close()
    assert not bad, bad
