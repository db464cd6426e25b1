#!/usr/bin/env python
"""Ranking users for items (``recommend_users``, ``corated_users``): how fast the item side runs on the engine.

ml_1m* (make_synthetic_dataset("ml_1m", seed=0)), max_nodes_per_hop 100, batch sizes 50 and 512, an untrained IGMC
(the rate does not depend on the weights):

* engine: 100 items ranked over all 6 040 users (k = 10, their raters excluded) by ``InferenceEngine.recommend_users``
  - candidate pairs/s, device events around the whole call;
* loop: what a caller had to write before - per item ``predict_pairs`` over its unrated users, then a sort on the host
  - over the same pairs; the script checks that both give the same lists;
* the retriever alone (``corated_users``) for 100 and 3 706 query items at M = 200;
* ``recommend_users(retrieve=M)`` for M = 100 and 500 against all users, the same 100 items.

Every arm runs once to warm up, then the arms are alternated ``--reps`` times; median and min-max.  The card's name
and power limit are read in the same run.

    python scripts/recommend_users_rate.py [--reps 3] [--out result.json]
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
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC  # noqa: E402
from igmc_b200.util_functions import RatingGraph  # noqa: E402

MNPH = 100
BATCHES = (50, 512)
K = 10
ITEMS = 100
M_RETRIEVER = 200
MS = (100, 500)


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


def loop_arm(m, g, items, lists, B):
    """per item predict_pairs over its candidate users, then a stable host sort: (users [I, K], scores [I, K])"""
    tu = np.full((len(items), K), -1, np.int64)
    ts = np.full((len(items), K), -np.inf, np.float32)
    for j, v in enumerate(items):
        s = rc.predict_pairs(m, g, lists[j], np.full(len(lists[j]), v), max_nodes_per_hop=MNPH, batch_size=B,
                             sample_seed=0).cpu().numpy()
        ts[j], tu[j] = rc.rank_host(s, lists[j], K)
    return tu, ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("recommend_users_rate.py measures on a CUDA device; none is available")
    name, pl = device_info()
    ds = make_synthetic_dataset("ml_1m", seed=0)
    A = ds["adj_train"]
    g = RatingGraph(A)
    nu, ni = g.shape
    items = np.random.default_rng(0).choice(ni, ITEMS, replace=False)
    col = g.host["col_ptr"]
    raters = [g.host["row_idx"][col[v]:col[v + 1]] for v in items]
    lists = [np.setdiff1d(np.arange(nu), r) for r in raters]
    pairs = int(sum(len(x) for x in lists))
    torch.manual_seed(1)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda().eval()
    res = dict(gpu=name, power_limit=pl, dataset="ml_1m*", max_nodes_per_hop=MNPH, k=K, items=ITEMS, users=nu,
               pairs=pairs, reps=a.reps, batches=[])

    retr = {ITEMS: items, ni: np.arange(ni)}
    for n in retr:                                                  # warm-up
        rc.corated_users(g, retr[n], M_RETRIEVER)
    t_retr = {n: [] for n in retr}

    for B in BATCHES:
        eng = rc.InferenceEngine(m, g, max_nodes_per_hop=MNPH, batch_size=B, sample_seed=0)
        cases = [("all users", None)] + [("retrieve %d" % M, M) for M in MS]
        P, times = {}, {c: [] for c, _ in cases}
        for c, M in cases:                                          # warm-up and pair counts
            P[c] = eng.start_recommend_users(items, K, retrieve=M)
            eng.finish()
        t_loop = []
        eng_lists = loop_lists = None
        for _ in range(a.reps):
            for c, M in cases:
                t, r = timed(lambda: eng.recommend_users(items, K, retrieve=M))
                times[c].append(t)
                if M is None:
                    eng_lists = r
            t, loop_lists = timed(lambda: loop_arm(m, g, items, lists, B))
            t_loop.append(t)
            for n in retr:
                t_retr[n].append(timed(lambda: rc.corated_users(g, retr[n], M_RETRIEVER))[0])
        eng.close()
        same = bool(np.array_equal(eng_lists[0].cpu().numpy(), loop_lists[0]) and
                    np.array_equal(eng_lists[1].cpu().numpy(), loop_lists[1]))
        assert P["all users"] == pairs
        full = float(np.median(times["all users"]))
        row = dict(batch=B, plan=next(iter(m._plans.values())) if m._plans else None,
                   engine=dict(seconds=stats(times["all users"]), pairs_per_s=stats([pairs / t for t in
                                                                                     times["all users"]], 0)),
                   loop=dict(seconds=stats(t_loop), pairs_per_s=stats([pairs / t for t in t_loop], 0)),
                   engine_over_loop=round(float(np.median(t_loop)) / full, 2), lists_equal=same,
                   retrieve=[dict(m=M, pairs=P["retrieve %d" % M], seconds=stats(times["retrieve %d" % M]),
                                  speedup_vs_all_users=round(full / float(np.median(times["retrieve %d" % M])), 2))
                             for M in MS])
        res["batches"].append(row)
        print(json.dumps(row), flush=True)
    res["retriever"] = [dict(items=n, m=M_RETRIEVER, seconds=stats(t_retr[n]),
                             items_per_s=round(n / float(np.median(t_retr[n])), 1)) for n in retr]
    print(json.dumps(res["retriever"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
