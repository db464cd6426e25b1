#!/usr/bin/env python
"""Rate of counterfactual explanations (``counterfactual``) on ml_1m* (make_synthetic_dataset("ml_1m", seed=0): 6 040 x
3 706, 900 188 ratings), max_nodes_per_hop 100, against the same greedy search done by hand: one ``RatingSessions``
build and one ``predict_sessions`` call per greedy step (``counterfactual_host``).

An IGMC is fine-tuned briefly (``OnlineTrainer``, ``--train-steps`` steps of batch 50) so that its rankings mean
something; ``--users`` users with ``--min-deg``..``--max-deg`` ratings are drawn, and per user the query is X = the item
at rank k = 10 of ``recommend(k=11)`` and Y = the item at rank 11.  The two variants run on the same queries, are
alternated ``--reps`` times, and must give equal results.  Reported: queries/s and forwards/s (two per trial, the base
pass included), median and min-max over host wall clock around each whole run (both end in a device synchronise), with
the GPU's name and power limit read in the same run.

    python scripts/counterfactual_rate.py [--users 50] [--max-removals 10] [--batch 256] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC, FusedAdam  # noqa: E402
from igmc_b200.train_eval import OnlineTrainer  # noqa: E402
from igmc_b200.util_functions import RatingGraph  # noqa: E402

MNPH, K = 100, 10


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def stats(v, digits=1):
    v = np.asarray(v)
    return dict(median=round(float(np.median(v)), digits), min=round(float(v.min()), digits),
                max=round(float(v.max()), digits))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=50)
    ap.add_argument("--min-deg", type=int, default=20)
    ap.add_argument("--max-deg", type=int, default=200)
    ap.add_argument("--max-removals", type=int, default=10)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--train-steps", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, pl = device_info()
    A = make_synthetic_dataset("ml_1m", seed=0)["adj_train"]
    g = RatingGraph(A)
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    OnlineTrainer(m, g, FusedAdam(m, lr=1e-3), batch_size=50, max_nodes_per_hop=MNPH).train(a.train_steps)
    torch.cuda.synchronize()

    rng = np.random.default_rng(0)
    deg = np.diff(g.host["row_ptr"])
    users = rng.choice(np.flatnonzero((deg >= a.min_deg) & (deg <= a.max_deg)), a.users, replace=False)
    opts = dict(max_nodes_per_hop=MNPH, batch_size=a.batch)
    top, _ = rc.recommend(m, g, users, K + 1, **opts)
    top = top.cpu().numpy()
    items, rivals = top[:, K - 1], top[:, K]
    M = a.max_removals
    rp, ci, rt = g.host["row_ptr"], g.host["col_idx"], g.host["rating"]

    def scorer(u, deleted, targets):
        sess = np.array([s for s, d in enumerate(deleted) for _ in d], np.int64)
        it = np.array([i for d in deleted for i in d], np.int64)
        S = rc.RatingSessions(g, np.asarray(u, np.int64), sess, it, np.zeros(len(it), np.int64))
        return rc.predict_sessions(m, S, np.arange(len(u)), targets, **opts).cpu().numpy()

    def device():
        cf = rc.counterfactual(m, g, users, items, rivals, M, **opts)
        return rc.Counterfactual(*(t.cpu().numpy() for t in cf))

    def host():
        return rc.counterfactual_host(rp, ci, rt, users, items, rivals, M, scorer)

    runs = dict(device=device, host_loop=host)
    first = {k: fn() for k, fn in runs.items()}            # warm-up, and the results compared
    for f in rc.Counterfactual._fields:
        x, y = getattr(first["device"], f), getattr(first["host_loop"], f)
        assert np.array_equal(x, y, equal_nan=f in ("score", "rival_score")), f
    cf = first["device"]
    # forwards: the base pass's two per query, then two per trial: step t of a query has deg - t trials
    fw = 2 * len(users) + sum(2 * (int(deg[u]) - t) for q, u in enumerate(users) for t in range(int(cf.size[q])))
    times = {k: [] for k in runs}
    for _ in range(a.reps):
        for k, fn in runs.items():
            times[k].append(wall(fn)[0])
    res = dict(gpu=name, power_limit=pl, dataset="ml_1m*", max_nodes_per_hop=MNPH, batch_size=a.batch,
               train_steps=a.train_steps, queries=len(users), k=K, max_removals=M, reps=a.reps, forwards=fw,
               found=int(cf.found.sum()), mean_size=round(float(cf.size.mean()), 2),
               size_histogram=np.bincount(cf.size, minlength=M + 1).tolist())
    for k in runs:
        res[k] = dict(queries_per_s=stats([len(users) / t for t in times[k]]),
                      forwards_per_s=stats([fw / t for t in times[k]]),
                      seconds=stats(times[k], 4))
    res["device / host_loop"] = round(float(np.median(times["host_loop"]) / np.median(times["device"])), 2)
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
