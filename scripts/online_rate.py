#!/usr/bin/env python
"""Rate of online fine-tuning (``OnlineTrainer``) on ml_1m* (make_synthetic_dataset("ml_1m", seed=0): 6 040 x 3 706,
900 188 ratings), max_nodes_per_hop 100, batch 50.

* ``steady``: subgraphs/s of ``OnlineTrainer.train`` against ``TrainEngine.step_pipe`` over the same graph's ratings
  (host wall clock around ``--steps`` steps that end in a device synchronise, after warm-up and capture);
* ``serve``: a round of update 100 ratings of 50 users, 20 fine-tune steps, ``recommend(k=10)`` for those users over the
  full catalogue, with the trainer kept alive against ``MyDynamicDataset`` + ``TrainEngine`` rebuilt over the graph's
  ratings every round (prime + 20 ``step_pipe``); and the kept trainer's re-plan and recapture cost after an update
  (its first ``train(20)`` after the update minus a steady ``train(20)``).

The variants are alternated ``--reps`` times; median and min-max are reported with the GPU's name and power limit read
in the same run.

    python scripts/online_rate.py [--reps 3] [--steps 400] [--out result.json]
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
from igmc_b200.train_eval import OnlineTrainer, TrainEngine  # noqa: E402
from igmc_b200.util_functions import MyDynamicDataset, RatingGraph  # noqa: E402

MNPH, B, K, FT_STEPS = 100, 50, 10, 20


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


def stats(v):
    v = np.asarray(v)
    return dict(median=round(float(np.median(v)), 3), min=round(float(v.min()), 3), max=round(float(v.max()), 3))


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def engine_steps(eng, perm, n, start=0):
    """prime + n step_pipe over consecutive batches of ``perm`` (the last step extracts nothing)"""
    eng.prime(perm[start:start + B], 1)
    for s in range(n):
        nxt = perm[start + (s + 1) * B:start + (s + 2) * B] if s < n - 1 else None
        eng.step_pipe(nxt, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, pl = device_info()
    ds = make_synthetic_dataset("ml_1m", seed=0)
    A = ds["adj_train"]
    coo = A.tocoo()
    tu, tv, tl = coo.row, coo.col, (coo.data - 1).astype(np.int64)
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    opt = FusedAdam(m, lr=1e-4)
    res = dict(gpu=name, power_limit=pl, dataset="ml_1m*", nnz=int(A.nnz), batch_size=B, max_nodes_per_hop=MNPH,
               reps=a.reps)

    # ---- steady state ----
    g = RatingGraph(A, reserve_nnz=100 * (a.reps * 3 + 10))
    d = MyDynamicDataset(None, g, (tu, tv), tl, 1, 1.0, MNPH, None, None, ds["class_values"])
    eng = TrainEngine(d, m, opt, B, ARR=0.001)
    tr = OnlineTrainer(m, g, opt, batch_size=B, max_nodes_per_hop=MNPH)
    rng = np.random.default_rng(0)
    perm = rng.permutation(len(tu))
    need = (a.steps + 1) * B
    engine_steps(eng, perm, 20)          # warm-up: eager steps, capture of every graph variant
    tr.train(20)
    t_eng, t_tr = [], []
    for r in range(a.reps):
        off = (r * need) % (len(perm) - need)
        t_eng.append(a.steps * B / wall(lambda: engine_steps(eng, perm, a.steps, off)) * 1e3)
        t_tr.append(a.steps * B / wall(lambda: tr.train(a.steps)) * 1e3)
    eng.close()
    res["steady"] = dict(steps=a.steps, train_engine_subgraphs_per_s=stats(t_eng),
                         online_trainer_subgraphs_per_s=stats(t_tr))
    res["steady"]["online / engine"] = round(np.median(t_tr) / np.median(t_eng), 3)
    print(json.dumps(res["steady"]), flush=True)

    # ---- serve round ----
    users = rng.choice(A.shape[0], 50, replace=False)

    def delta():
        u = np.repeat(users, 2).astype(np.int64)
        return u, rng.integers(0, A.shape[1], len(u)), rng.integers(1, 6, len(u))

    def kept():
        tr.update(*delta())
        tr.train(FT_STEPS)
        rc.recommend(m, g, users, K, max_nodes_per_hop=MNPH)

    def rebuilt():
        g.update(*delta())
        h = g.host
        ru = np.repeat(np.arange(g.num_users), np.diff(h["row_ptr"]))
        dd = MyDynamicDataset(None, g, (ru, h["col_idx"]), h["rating"].astype(np.int64), 1, 1.0, MNPH, None, None,
                              ds["class_values"])
        e = TrainEngine(dd, m, opt, B, ARR=0.001)
        engine_steps(e, rng.permutation(len(ru)), FT_STEPS)
        e.close()
        rc.recommend(m, g, users, K, max_nodes_per_hop=MNPH)

    kept(), rebuilt()                    # warm-up
    t_keep, t_reb, t_replan = [], [], []
    for _ in range(a.reps):
        t_keep.append(wall(kept))
        t_reb.append(wall(rebuilt))
        tr.update(*delta())
        first = wall(lambda: tr.train(FT_STEPS))
        t_replan.append(first - wall(lambda: tr.train(FT_STEPS)))
    tr.close()
    res["serve"] = dict(users=50, ratings_per_round=100, fine_tune_steps=FT_STEPS, k=K,
                        kept_trainer_ms_per_round=stats(t_keep), rebuilt_engine_ms_per_round=stats(t_reb),
                        replan_and_recapture_ms=stats(t_replan))
    res["serve"]["rebuilt / kept"] = round(np.median(t_reb) / np.median(t_keep), 2)
    print(json.dumps(res["serve"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
