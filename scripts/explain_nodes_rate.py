#!/usr/bin/env python
"""Node explanation rate on ml_1m* (make_synthetic_dataset("ml_1m", seed=0), max_nodes_per_hop 100): per batch size,

* ``explain_nodes``: explained pairs/s and occluded subgraphs/s (one per non-target node of each pair's subgraph),
* ``explain_pairs`` in the same process: pairs/s and occluded subgraphs/s (one per rating),
* ``attribute_nodes``: attributed pairs/s (the base pass and one gradient pass over the pairs),

each through its ``InferenceEngine`` method, the three alternated ``--reps`` times; device-event timing around each
whole run, median (min-max) over the repetitions.

    python scripts/explain_nodes_rate.py [--pairs 50] [--reps 3] [--batch 50 512]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from explain_rate import MNPH, device_info, timed  # noqa: E402
from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC  # noqa: E402


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
        runs = dict(explain_nodes=lambda: eng.explain_nodes(pu, pv), explain_pairs=lambda: eng.explain_pairs(pu, pv),
                    attribute_nodes=lambda: eng.attribute_nodes(pu, pv))
        sizes = dict(explain_nodes=int(runs["explain_nodes"]().offsets[P]),     # warm-up and the position totals
                     explain_pairs=int(runs["explain_pairs"]().offsets[P]))
        runs["attribute_nodes"]()
        times = {k: [] for k in runs}
        for _ in range(a.reps):
            for k, fn in runs.items():
                times[k].append(timed(fn)[0])
        eng.close()
        row = dict(batch=B)
        for k, v in times.items():
            v = np.array(v)
            row[k] = dict(pairs_per_s=dict(median=round(float(P / np.median(v)), 1), min=round(float(P / v.max()), 1),
                                           max=round(float(P / v.min()), 1)))
            if k in sizes:
                row[k]["occluded"] = sizes[k]
                row[k]["occluded_per_s"] = round(float(sizes[k] / np.median(v)), 1)
        row["explain_nodes / explain_pairs pairs/s"] = round(float(np.median(times["explain_pairs"]) /
                                                                   np.median(times["explain_nodes"])), 3)
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
