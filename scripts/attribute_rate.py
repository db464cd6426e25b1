#!/usr/bin/env python
"""Attribution rate of ``attribute_pairs`` against ``explain_pairs`` on ml_1m* (make_synthetic_dataset("ml_1m",
seed=0), max_nodes_per_hop 100), on the same 50 random pairs as scripts/explain_rate.py:

* attributed pairs/s of the whole run (base pass, one host sync, gradient pass, per-pair sort) and gradient-pass
  subgraphs/s (from the end of the base pass to the ordered result: P subgraphs, each an L2-plan eval forward and one
  igmc_edge_grad backward);
* explained pairs/s of ``explain_pairs`` (occlusion: one forward per rating) on the same engine.

The two run in one process, alternated, ``--reps`` times each per batch size; device-event timing.  For information
only: per pair, the Spearman correlation of -grad with the occlusion delta and the overlap of the two top-10 lists.

    python scripts/attribute_rate.py [--pairs 50] [--reps 3] [--batch 50 512]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
from scipy.stats import spearmanr

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC  # noqa: E402
from scripts.explain_rate import MNPH, device_info  # noqa: E402


def _positions(eng, start, pu, pv):
    """one run; (result, per-position values [T] on the host)"""
    start(pu, pv)
    while eng.step():
        pass
    vals = eng.run["occ"].clone()
    return eng.finish(), vals.cpu().numpy()


def timed_attribute(eng, pu, pv):
    """(whole run s, gradient pass s) of one attribution run"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    ev[0].record()
    eng.start_attribute(pu, pv)
    more = True
    while more and eng.run["phase"] == "base":
        more = eng.step()
    ev[1].record()
    while eng.step():
        pass
    eng.finish()
    ev[2].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[2]) / 1000.0, ev[1].elapsed_time(ev[2]) / 1000.0


def timed_explain(eng, pu, pv):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    eng.explain_pairs(pu, pv)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1000.0


def agreement(ex, occ, grad):
    """per pair with >= 3 ratings: Spearman(-grad, delta) and |top-10 by |grad|| & top-10 by |delta||| / 10"""
    off, score = ex.offsets.cpu().numpy(), ex.score.cpu().numpy()
    rho, overlap = [], []
    for q in range(len(score)):
        d, g = occ[off[q]:off[q + 1]] - score[q], grad[off[q]:off[q + 1]]
        if len(d) < 3 or np.isnan(d).any() or np.isnan(g).any():
            continue
        rho.append(float(spearmanr(-g, d)[0]))
        k = min(10, len(d))
        overlap.append(len(set(np.argsort(-np.abs(g), kind="stable")[:k]) &
                           set(np.argsort(-np.abs(d), kind="stable")[:k])) / k)
    return dict(pairs=len(rho), spearman_median=round(float(np.median(rho)), 3),
                spearman_min=round(float(np.min(rho)), 3), top10_overlap_mean=round(float(np.mean(overlap)), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, nargs="+", default=[50, 512])
    a = ap.parse_args()
    name, pl = device_info()
    A = make_synthetic_dataset("ml_1m", seed=0)["adj_train"]
    torch.manual_seed(1)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda().eval()
    rng = np.random.default_rng(0)
    pu = rng.integers(0, A.shape[0], a.pairs).astype(np.int64)
    pv = rng.integers(0, A.shape[1], a.pairs).astype(np.int64)
    P = len(pu)
    res = dict(gpu=name, power_limit=pl, pairs=P, max_nodes_per_hop=MNPH, reps=a.reps, rows=[])
    for B in a.batch:
        eng = rc.InferenceEngine(m, A, max_nodes_per_hop=MNPH, batch_size=B, sample_seed=0)
        ex, occ = _positions(eng, eng.start_explain, pu, pv)          # warm-up of both runs, and their values
        at, grad = _positions(eng, eng.start_attribute, pu, pv)
        assert torch.equal(at.score, ex.score) and torch.equal(at.offsets, ex.offsets)
        T = int(ex.offsets[-1])
        times = dict(attribute=[], gradient_pass=[], explain=[])
        for _ in range(a.reps):
            t, tg = timed_attribute(eng, pu, pv)
            times["attribute"].append(t)
            times["gradient_pass"].append(tg)
            times["explain"].append(timed_explain(eng, pu, pv))
        eng.close()
        med = {k: float(np.median(v)) for k, v in times.items()}
        row = dict(batch=B, ratings=T, base_plan=m._plans.get(next(iter(k for k in m._plans if k[1] == B)), None),
                   gradient_plan=next(iter(eng._grad_plans.values()), None),
                   attribute_pairs_per_s=round(P / med["attribute"], 1),
                   gradient_pass_subgraphs_per_s=dict(median=round(P / med["gradient_pass"], 1),
                                                      min=round(P / max(times["gradient_pass"]), 1),
                                                      max=round(P / min(times["gradient_pass"]), 1)),
                   explain_pairs_per_s=round(P / med["explain"], 1),
                   attribute_over_explain=round(med["explain"] / med["attribute"], 2),
                   agreement=agreement(ex, occ, grad))
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
