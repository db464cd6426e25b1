#!/usr/bin/env python
"""Rate and effect of diversified lists (``recommend_diverse``).

Rate: ml_1m* (make_synthetic_dataset("ml_1m", seed=0): 6 040 x 3 706, 900 188 ratings), max_nodes_per_hop 100, batch
256, every user, k = 10, pools of 50 and 100 over the full catalogue, an IGMC fine-tuned briefly (``OnlineTrainer``,
``--train-steps`` steps of batch 50).  On one engine, per pool size:

* ``recommend(k=pool)`` alone against ``recommend_diverse`` at the first penalty, alternated ``--reps`` times (host
  wall clock around each whole run, both ending in a device synchronise);
* the diverse stage alone (union, co-counts, selection) on the finished pools, by CUDA events, at both penalties;
* the union size Nu;
* a by-hand host path from the same pools: the pools copied to the host, scipy co-counts restricted to the union and
  a numpy greedy vectorised over the users.

Every list is checked equal (items, scores, keys) to the host path's before any time is kept.

Effect: the real flixster split (make_synthetic_dataset("flixster")), IGMC trained ``--epochs`` epochs through
``train_multiple_epochs`` as scripts/draws_rate.py does; every user's pool of 50, k = 10, for each penalty in
{0, 0.25, 0.5, 1, 2}: the mean pairwise similarity within a list, the mean model score of a list and the catalogue
coverage (distinct items over all lists).  The GPU's name and power limit are read in the same run.

    python scripts/diverse_rate.py [--reps 2] [--train-steps 300] [--epochs 5] [--out F]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as ssp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC, FusedAdam  # noqa: E402
from igmc_b200.train_eval import OnlineTrainer  # noqa: E402
from igmc_b200.util_functions import RatingGraph  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from counterfactual_rate import device_info, stats, wall  # noqa: E402

MNPH, BATCH, K_TOP = 100, 256, 10
PENALTIES = (0.5, 2.0)


def union_counts(g, pool_i):
    """(union [Nu], dense co-counts [Nu, Nu] int64 over it, column degrees [num_items]) by scipy"""
    hp = g.host
    union = np.unique(pool_i[pool_i >= 0])
    nnz = int(hp["row_ptr"][g.num_users])
    B = ssp.csr_matrix((np.ones(nnz, np.int32), hp["col_idx"][:nnz], hp["row_ptr"]), shape=(g.num_users, g.num_items))
    Bu = B[:, union]
    return union, np.asarray((Bu.T @ Bu).toarray(), np.int64), np.diff(hp["col_ptr"]).astype(np.int64)


def by_hand(g, pool_i_dev, pool_s_dev, k, penalty):
    """the host path: pools to the host, scipy co-counts over their union, a numpy greedy over every user at once"""
    pool_i, pool_s = pool_i_dev.cpu().numpy(), pool_s_dev.cpu().numpy()
    union, Cm, deg = union_counts(g, pool_i)
    U, P = pool_i.shape
    idx = np.where(pool_i >= 0, np.searchsorted(union, np.maximum(pool_i, 0)), 0)
    d = np.where(pool_i >= 0, deg[np.maximum(pool_i, 0)], 0)
    live = pool_i >= 0
    m = np.zeros((U, P), np.float32)
    pen = np.float32(penalty)
    rows = np.arange(U)
    out = [np.full((U, k), -1, np.int64), np.full((U, k), -np.inf, np.float32), np.full((U, k), -np.inf, np.float32)]
    for s in range(k):
        key = (pool_s - pen * m).astype(np.float32)
        nan = np.isnan(key)
        ok = live & ~nan
        mx = np.where(ok, key, -np.inf).max(1)
        first = ok & (key == mx[:, None])
        has0, has1 = first.any(1), (live & nan).any(1)
        c = np.where(has0, first.argmax(1), (live & nan).argmax(1))
        got = has0 | has1
        r = rows[got]
        cc = c[got]
        out[0][r, s], out[1][r, s], out[2][r, s] = pool_i[r, cc], pool_s[r, cc], key[r, cc]
        live[r, cc] = False
        cnt = Cm[idx[r, cc][:, None], idx[r]]                           # c of the chosen item with every entry
        prod = d[r, cc][:, None].astype(np.float64) * d[r].astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            sim = np.where(prod > 0, cnt / np.sqrt(prod), 0.0).astype(np.float32)
        m[r] = np.where(live[r], np.maximum(m[r], sim), m[r])
    return out, len(union)


def stage_ms(eng, pool_i, pool_s, k, penalty, reps=5):
    """the diverse stage alone by CUDA events: median and min-max ms over ``reps`` runs after one warm-up"""
    eng._diverse(pool_i, pool_s, k, penalty)
    t = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        eng._diverse(pool_i, pool_s, k, penalty)
        b.record()
        b.synchronize()
        t.append(a.elapsed_time(b))
    return stats(t, 2)


def rate(a):
    Adj = make_synthetic_dataset("ml_1m", seed=0)["adj_train"]
    g = RatingGraph(Adj)
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    OnlineTrainer(m, g, FusedAdam(m, lr=1e-3), batch_size=50, max_nodes_per_hop=MNPH).train(a.train_steps)
    torch.cuda.synchronize()
    users = np.arange(g.num_users)
    res = dict(dataset="ml_1m*", users=len(users), max_nodes_per_hop=MNPH, batch=BATCH, k=K_TOP, reps=a.reps,
               train_steps=a.train_steps, runs={})
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=MNPH, batch_size=BATCH)
    try:
        eng.recommend(users[:64], 100)                                  # warm-up: shapes, plans and captured steps
        for pool in (50, 100):
            t_pool, (pi, ps) = wall(lambda: eng.recommend(users, pool))
            r = dict()
            for pen in PENALTIES:
                t_hand, (want, Nu) = wall(lambda: by_hand(g, pi, ps, K_TOP, pen))
                got = eng._diverse(pi, ps, K_TOP, pen)
                for x, y in zip(got, want):
                    assert np.array_equal(x.cpu().numpy(), y), (pool, pen)
                r["penalty=%g" % pen] = dict(Nu=Nu, stage_ms=stage_ms(eng, pi, ps, K_TOP, pen),
                                             by_hand_s=round(t_hand, 3))
            pen = PENALTIES[0]
            d = eng.recommend_diverse(users, K_TOP, pen, pool)
            for x, y in zip(d, eng._diverse(pi, ps, K_TOP, pen)):
                assert torch.equal(x, y)
            times = dict(recommend=[t_pool], recommend_diverse=[])
            for _ in range(a.reps):
                times["recommend_diverse"].append(wall(lambda: eng.recommend_diverse(users, K_TOP, pen, pool))[0])
                times["recommend"].append(wall(lambda: eng.recommend(users, pool))[0])
            r["seconds"] = {kk: stats(v, 2) for kk, v in times.items()}
            r["stage share of the pool run at penalty %g" % pen] = round(
                r["penalty=%g" % pen]["stage_ms"]["median"] / 1e3 / float(np.median(times["recommend"])), 5)
            res["runs"]["pool=%d" % pool] = r
            print(json.dumps({"pool=%d" % pool: r}), flush=True)
    finally:
        eng.close()
    return res


def effect(a):
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
    rmse = train_multiple_epochs(train, test, m, a.epochs, 50, 1e-3, 0.1, max(a.epochs // 2, 1), 0, ARR=0.001)
    m.eval()
    g = RatingGraph(A)
    users = np.arange(g.num_users)
    out = dict(dataset="flixster (real split)", users=len(users), epochs=a.epochs, test_rmse=round(float(rmse), 4),
               pool=50, k=K_TOP, penalties={})
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=ds["max_nodes_per_hop"], batch_size=BATCH)
    try:
        pi, ps = eng.recommend(users, 50)
        union, Cm, deg = union_counts(g, pi.cpu().numpy())
        for pen in (0.0, 0.25, 0.5, 1.0, 2.0):
            d = eng._diverse(pi, ps, K_TOP, pen)
            items, scores = d.items.cpu().numpy(), d.scores.cpu().numpy()
            sims, means = [], []
            for row, sc in zip(items, scores):
                row = row[row >= 0]
                if len(row) >= 2:
                    ix = np.searchsorted(union, row)
                    prod = np.outer(deg[row], deg[row]).astype(np.float64)
                    with np.errstate(divide="ignore", invalid="ignore"):
                        S = np.where(prod > 0, Cm[np.ix_(ix, ix)] / np.sqrt(prod), 0.0)
                    sims.append(S[np.triu_indices(len(row), 1)].mean())
                if len(row):
                    means.append(float(np.mean(sc[:len(row)])))
            r = dict(mean_pairwise_sim=round(float(np.mean(sims)), 4), mean_list_score=round(float(np.mean(means)), 4),
                     coverage=int(len(np.unique(items[items >= 0]))), catalogue=g.num_items)
            out["penalties"]["%g" % pen] = r
            print(json.dumps({"penalty=%g" % pen: r}), flush=True)
    finally:
        eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--train-steps", type=int, default=300)
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--skip-rate", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, pl = device_info()
    print(json.dumps(dict(gpu=name, power_limit=pl)), flush=True)
    t0 = time.time()
    res = dict(gpu=name, power_limit=pl)
    if not a.skip_rate:
        res["rate"] = rate(a)
    res["effect"] = effect(a)
    res["wall_s"] = round(time.time() - t0, 1)
    print(json.dumps(res, indent=1), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
