#!/usr/bin/env python
"""Monte-Carlo-dropout draws: rates on ml_1m* (make_synthetic_dataset("ml_1m", seed=0), max_nodes_per_hop 100) and
what the spread says on the real flixster split.

* throughput: forwards/s of ``predict_draws`` at S = 8 on ``--pairs`` random pairs, against ``predict_pairs`` pairs/s
  and ``explain_pairs``' occluded subgraphs/s (``--explain-pairs`` pairs) in the same process, per batch size;
* exploration cost: ``recommend(retrieve=100, k=10)`` for ``--users`` users with draws None / 1 / 8 (beta 1 at S = 8);
* spread: IGMC trained on tests/golden/flixster_ratings.npz through ``train_multiple_epochs``, then on the 2 617 test
  ratings the Spearman correlation of std with |y - mean| and the RMSE of mean against that of the eval score.

The model of the two rate parts is an untrained IGMC with the constructor's adj_dropout 0.2 (the ml_1m preset trains
without edge dropout; a draw then only drops hidden units).  Variants alternate ``--reps`` times; device-event timing
around each whole run, median (min-max).

    python scripts/draws_rate.py [--pairs 2000] [--batch 256 512] [--users 500] [--epochs 40] [--out FILE]
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


def _stat(n, times):
    v = np.array(times)
    return dict(median=round(float(n / np.median(v)), 1), min=round(float(n / v.max()), 1),
                max=round(float(n / v.min()), 1))


def throughput(m, A, a, rng):
    pu = rng.integers(0, A.shape[0], a.pairs)
    pv = rng.integers(0, A.shape[1], a.pairs)
    eu, ev = pu[:a.explain_pairs], pv[:a.explain_pairs]
    rows = []
    for B in a.batch:
        eng = rc.InferenceEngine(m, A, max_nodes_per_hop=MNPH, batch_size=B, sample_seed=0)
        runs = dict(draws=lambda: eng.predict_draws(pu, pv, 8), pairs=lambda: eng.predict_pairs(pu, pv),
                    explain=lambda: eng.explain_pairs(eu, ev))
        occluded = int(runs["explain"]().offsets[-1])     # warm-up of every variant, and the occlusion total
        runs["draws"]()
        runs["pairs"]()
        times = {k: [] for k in runs}
        for _ in range(a.reps):
            for k, fn in runs.items():
                times[k].append(timed(fn)[0])
        eng.close()
        row = dict(batch=B, draws_forwards_per_s=_stat(8 * a.pairs, times["draws"]),
                   pairs_per_s=_stat(a.pairs, times["pairs"]),
                   explain_occluded_per_s=_stat(occluded, times["explain"]), explain_occluded=occluded)
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def exploration(m, A, a, rng):
    users = rng.choice(A.shape[0], a.users, replace=False)
    eng = rc.InferenceEngine(m, A, max_nodes_per_hop=MNPH, batch_size=256, sample_seed=0)
    runs = {"None": lambda: eng.recommend(users, 10, retrieve=100),
            "1": lambda: eng.recommend(users, 10, retrieve=100, draws=1),
            "8": lambda: eng.recommend(users, 10, retrieve=100, draws=8, beta=1.0)}
    for fn in runs.values():
        fn()
    times = {k: [] for k in runs}
    for _ in range(a.reps):
        for k, fn in runs.items():
            times[k].append(timed(fn)[0])
    eng.close()
    out = {k: dict(ms=dict(median=round(1e3 * float(np.median(v)), 2), min=round(1e3 * min(v), 2),
                           max=round(1e3 * max(v), 2))) for k, v in times.items()}
    print(json.dumps(dict(exploration=out)), flush=True)
    return out


def spread(a):
    from scipy import stats
    from igmc_b200.train_eval import train_multiple_epochs
    from igmc_b200.util_functions import MyDataset
    ds = make_synthetic_dataset("flixster", seed=0)
    assert ds.get("real"), "the flixster fixture is missing"
    A, cv = ds["adj_train"], ds["class_values"]
    tu, tv, tl = ds["train"]
    su, sv, sl = ds["test"]
    mk = lambda u, v, l: MyDataset(None, A, (u, v), l, 1, 1.0, ds["max_nodes_per_hop"], None, None, cv, seed=0)  # noqa
    train, test = mk(tu, tv, tl), mk(su, sv, sl)
    torch.manual_seed(1)
    m = IGMC(train, latent_dim=[32] * 4, num_relations=ds["num_relations"], num_bases=4, regression=True,
             adj_dropout=ds["adj_dropout"]).cuda()
    rmse_train = train_multiple_epochs(train, test, m, a.epochs, 50, 1e-3, 0.1, max(a.epochs // 2, 1), 0, ARR=0.001)
    m.eval()
    y = cv[sl].astype(np.float64)
    kw = dict(max_nodes_per_hop=ds["max_nodes_per_hop"], batch_size=256)
    score = rc.predict_pairs(m, A, su, sv, **kw).double().cpu().numpy()
    out = dict(epochs=a.epochs, test_ratings=len(y), train_multiple_epochs_test_rmse=round(float(rmse_train), 4),
               eval_rmse=round(float(np.sqrt(np.mean((score - y) ** 2))), 4))
    for S in (8, 32):
        d = rc.predict_draws(m, A, su, sv, S, draw_seed=1, **kw)
        mean, sd = d.mean.double().cpu().numpy(), d.std.double().cpu().numpy()
        rho = stats.spearmanr(sd, np.abs(y - mean))
        out["S=%d" % S] = dict(mean_rmse=round(float(np.sqrt(np.mean((mean - y) ** 2))), 4),
                               spearman_std_vs_abs_err=round(float(rho.correlation), 4),
                               spearman_p=float(rho.pvalue), median_std=round(float(np.median(sd)), 4))
    print(json.dumps(dict(spread=out)), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=2000)
    ap.add_argument("--explain-pairs", type=int, default=50)
    ap.add_argument("--users", type=int, default=500)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--epochs", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, pl = device_info()
    res = dict(gpu=name, power_limit=pl, max_nodes_per_hop=MNPH, pairs=a.pairs, reps=a.reps)
    A = make_synthetic_dataset("ml_1m", seed=0)["adj_train"]
    torch.manual_seed(1)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda().eval()
    rng = np.random.default_rng(0)
    res["throughput"] = throughput(m, A, a, rng)
    res["exploration"] = exploration(m, A, a, rng)
    if a.epochs > 0:
        res["spread"] = spread(a)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
