#!/usr/bin/env python
"""Train-step rate (subgraphs/s) of the two RGCNConv layers: IGMC(..., rgcn="pyg-1.4") (one mean over all in-edges,
the default) and rgcn="pyg-2" (one mean per relation), through the full pipelined step (TrainEngine.step_pipe with
CUDA graphs: extraction of the next batch, the one-launch train kernel, the fused reduce / exchange / Adam kernel).

Both models live in one process and are timed alternately, ``--reps`` times each, ``--steps`` steps per timed run
(CUDA events around the run, after warm-up and graph capture).  Reports the median and the min-max spread per layer.

    python scripts/relation_mean_rate.py [--steps 200] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC, FusedAdam  # noqa: E402
from igmc_b200.train_eval import TrainEngine  # noqa: E402
from igmc_b200.util_functions import MyDynamicDataset  # noqa: E402

B = 50
ARR = 0.001
LAYERS = ("pyg-1.4", "pyg-2")
# (name, synthetic preset, max nodes per hop, edge dropout)
CONFIGS = [("ml_1m* mnph 100, no dropout", "ml_1m", 100, 0.0),
           ("ml_100k* mnph 200, adj_dropout 0.2", "ml_100k", 200, 0.2)]


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


class Arm:
    """one model + optimizer + pipelined engine, with its own cursor over a fixed pair permutation"""

    def __init__(self, ds, mnph, adj_dropout, rgcn, warmup):
        tu, tv, tl = ds["train"]
        self.d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, mnph, None, None, ds["class_values"],
                                  seed=0)
        torch.manual_seed(1)
        self.m = IGMC(self.d, latent_dim=[32] * 4, num_relations=ds["num_relations"], num_bases=4, regression=True,
                      adj_dropout=adj_dropout, rgcn=rgcn).cuda()
        self.opt = FusedAdam(self.m, lr=1e-3)
        self.eng = TrainEngine(self.d, self.m, self.opt, B, ARR=ARR, use_graph=True)
        self.perm = np.random.default_rng(1000).permutation(len(tu))
        self.k = 0
        self.eng.prime(self.next_idx(), epoch=1)
        for _ in range(warmup):
            self.eng.step_pipe(self.next_idx(), epoch=1)
        torch.cuda.synchronize()
        self.eng.check()

    def next_idx(self):
        idx = self.perm[(self.k * B + np.arange(B)) % len(self.perm)]
        self.k += 1
        return idx

    def run(self, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            self.eng.step_pipe(self.next_idx(), epoch=1)
        e1.record()
        torch.cuda.synchronize()
        self.eng.check()
        return B * steps / (e0.elapsed_time(e1) / 1000.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    name, pl = device_info()
    res = dict(gpu=name, power_limit=pl, batch=B, steps=a.steps, reps=a.reps, configs=[])
    for tag, preset, mnph, p in CONFIGS:
        ds = make_synthetic_dataset(preset, seed=0)
        arms = {r: Arm(ds, mnph, p, r, a.warmup) for r in LAYERS}
        for r, arm in arms.items():   # both layers took the fast path: one-launch train kernel + fused update
            assert arm.eng.exchange is not None and len(arm.eng.graphs) > 0, r
        rates = {r: [] for r in LAYERS}
        for _ in range(a.reps):
            for r in LAYERS:
                rates[r].append(arms[r].run(a.steps))
        row = dict(config=tag, plan=arms["pyg-2"].m._plan(arms["pyg-2"].eng.batches[0]))
        for r in LAYERS:
            v = np.array(rates[r])
            row[r] = dict(median=round(float(np.median(v)), 1), min=round(float(v.min()), 1),
                          max=round(float(v.max()), 1))
        row["pyg-2 / pyg-1.4"] = round(row["pyg-2"]["median"] / row["pyg-1.4"]["median"], 3)
        for arm in arms.values():
            arm.eng.close()
        res["configs"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
