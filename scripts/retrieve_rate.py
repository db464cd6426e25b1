#!/usr/bin/env python
"""Two-stage ranking: the bridge-count retriever (``corated_items``, csrc/retrieve.cu) proposing M items per user and
the engine ranking only those (``recommend(retrieve=M)``), against ranking the full catalogue.

* ml_1m* (make_synthetic_dataset("ml_1m", seed=0), max_nodes_per_hop 100, batch 512): the retriever alone for 500 and
  6 040 query users (M = 200), CUDA events around each call;
* ml_1m*, 500 users: ``recommend(retrieve=M)`` for M = 100 / 200 / 500 and the full catalogue - candidate pairs and
  wall time (device events around the whole call, the retriever included), runs alternated ``--reps`` times,
  median and min-max;
* the real flixster split (``load_flixster``) after a short training run in this process: the overlap of each user's
  k = 10 list from ``retrieve=M`` with the full-catalogue k = 10 list (ml_1m* is synthetic: its overlap means little).

    python scripts/retrieve_rate.py [--reps 3] [--epochs 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import load_flixster, make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC, FusedAdam  # noqa: E402
from igmc_b200.train_eval import TrainEngine  # noqa: E402
from igmc_b200.util_functions import MyDynamicDataset, RatingGraph  # noqa: E402

MNPH = 100
B = 512
K = 10
MS = (100, 200, 500)


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1000.0, r


def stats(v, nd=4):
    v = np.array(v)
    return dict(median=round(float(np.median(v)), nd), min=round(float(v.min()), nd), max=round(float(v.max()), nd))


def ml_1m(a):
    ds = make_synthetic_dataset("ml_1m", seed=0)
    A = ds["adj_train"]
    g = RatingGraph(A)
    nu, ni = g.shape
    out = dict(retriever=[], ranking=[])
    for U in (500, nu):
        users = np.random.default_rng(0).choice(nu, U, replace=False)
        rc.corated_items(g, users, 200)                      # warm-up
        t = [timed(lambda: rc.corated_items(g, users, 200))[0] for _ in range(a.reps)]
        row = dict(users=U, m=200, seconds=stats(t), users_per_s=round(U / float(np.median(t)), 1))
        out["retriever"].append(row)
        print(json.dumps(row), flush=True)
    torch.manual_seed(1)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda().eval()
    users = np.random.default_rng(0).choice(nu, 500, replace=False)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=MNPH, batch_size=B, sample_seed=0)
    cases = [("full", None)] + [("retrieve %d" % M, M) for M in MS]
    pairs, times = {}, {c: [] for c, _ in cases}
    for c, M in cases:                                          # warm-up and pair counts
        pairs[c] = eng.start_recommend(users, K, retrieve=M)
        eng.finish()
    for _ in range(a.reps):
        for c, M in cases:
            times[c].append(timed(lambda: eng.recommend(users, K, retrieve=M))[0])
    eng.close()
    full = float(np.median(times["full"]))
    for c, _ in cases:
        row = dict(case=c, users=500, pairs=pairs[c], seconds=stats(times[c]),
                   speedup_vs_full=round(full / float(np.median(times[c])), 2))
        out["ranking"].append(row)
        print(json.dumps(row), flush=True)
    return out


def flixster(a):
    ds = load_flixster()
    A = ds["adj_train"]
    tu, tv, tl = ds["train"]
    R = ds["num_relations"]
    d = MyDynamicDataset(None, A, (tu, tv), tl, 1, 1.0, ds["max_nodes_per_hop"], None, None, ds["class_values"],
                         seed=3)
    torch.manual_seed(0)
    m = IGMC(d, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True, adj_dropout=0.2).cuda()
    m.train()
    opt = FusedAdam(m, lr=1e-3)
    bs = 50
    eng = TrainEngine(d, m, opt, bs, ARR=0.001, use_graph=True)
    rng = np.random.default_rng(0)
    for ep in range(1, a.epochs + 1):
        perm = rng.permutation(len(tu))
        for s in range(0, len(perm) - bs + 1, bs):
            eng.step(perm[s:s + bs], epoch=ep)
    eng.check()
    m.eval()
    g = RatingGraph(A)
    deg = np.diff(A.indptr)
    users = np.random.default_rng(1).choice(np.flatnonzero(deg > 0), 300, replace=False)
    full_i, _ = rc.recommend(m, g, users, K, max_nodes_per_hop=ds["max_nodes_per_hop"], batch_size=B)
    full_i = full_i.cpu().numpy()
    rows = []
    for M in MS:
        ti, _ = rc.recommend(m, g, users, K, retrieve=M, max_nodes_per_hop=ds["max_nodes_per_hop"], batch_size=B)
        ti = ti.cpu().numpy()
        ov = [len(set(ti[j][ti[j] >= 0]) & set(full_i[j][full_i[j] >= 0])) / float(K) for j in range(len(users))]
        row = dict(m=M, users=len(users), overlap_at_10=dict(mean=round(float(np.mean(ov)), 3),
                                                             median=round(float(np.median(ov)), 3)))
        rows.append(row)
        print(json.dumps(row), flush=True)
    return dict(epochs=a.epochs, rows=rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--epochs", type=int, default=2)
    a = ap.parse_args()
    name, pl = device_info()
    res = dict(gpu=name, power_limit=pl, max_nodes_per_hop=MNPH, batch=B, k=K, reps=a.reps)
    res["ml_1m"] = ml_1m(a)
    res["flixster"] = flixster(a)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
