#!/usr/bin/env python
"""Cost of changing the rating graph in place (``RatingGraph.update``) against rebuilding it, on ml_1m*
(make_synthetic_dataset("ml_1m", seed=0): 6 040 x 3 706, 900 188 ratings).

* ``update``: ``graph.update`` with deltas of 1, 100, 10 000 and 1 000 000 entries (a quarter each inserts,
  overwrites, deletes of rated pairs and deletes of absent pairs, so nnz stays level); host wall clock around the call
  (it ends in its one host synchronisation) and CUDA events around it;
* ``rebuild``: the same change the only other way: scipy edit of the matrix + ``RatingGraph(A)`` + a new
  ``InferenceEngine`` (which re-extracts its first batch when it runs) - host wall clock, device synchronised;
* ``serve``: update 100 ratings of 50 users, then ``recommend(k=10)`` for those users over the full catalogue, with
  one engine kept alive versus graph and engine rebuilt every round.

Every workload runs ``--reps`` times, the two sides alternated; median and min-max are reported with the GPU's name and
power limit read in the same run.  Before timing, the kept engine's top-k is checked bit for bit against a rebuilt one.

    python scripts/graph_update_rate.py [--reps 5] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as ssp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC  # noqa: E402
from igmc_b200.util_functions import RatingGraph  # noqa: E402

MNPH = 100
K = 10
B = 256


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


def apply_scipy(A, u, v, x):
    """the rebuild path's edit: last occurrence of a pair wins, value 0 deletes"""
    M = np.int64(A.shape[1])
    o = np.lexsort((v, u))
    su, sv, sx = u[o], v[o], x[o]
    keep = np.r_[(su[1:] != su[:-1]) | (sv[1:] != sv[:-1]), True]
    su, sv, sx = su[keep], sv[keep], sx[keep]
    coo = A.tocoo()
    stay = ~np.isin(coo.row.astype(np.int64) * M + coo.col, su * M + sv)
    ins = sx > 0
    return ssp.csr_matrix((np.concatenate([coo.data[stay], sx[ins].astype(np.float32)]),
                           (np.concatenate([coo.row[stay], su[ins]]), np.concatenate([coo.col[stay], sv[ins]]))),
                          shape=A.shape, dtype=np.float32)


def delta(rng, A, n, users=None):
    coo = A.tocoo()
    k = rng.integers(0, 4, n)
    if users is not None:              # n ratings of the given users: inserts / overwrites of random items
        u = np.repeat(users, n // len(users)).astype(np.int64)
        return u, rng.integers(0, A.shape[1], len(u)).astype(np.int64), rng.integers(1, 6, len(u)).astype(np.int64)
    e = rng.integers(0, A.nnz, n)
    u = np.where(k < 2, coo.row[e], rng.integers(0, A.shape[0], n)).astype(np.int64)
    v = np.where(k < 2, coo.col[e], rng.integers(0, A.shape[1], n)).astype(np.int64)
    x = np.where((k == 0) | (k == 2), rng.integers(1, 6, n), 0).astype(np.int64)
    return u, v, x


def stats(v):
    v = np.asarray(v)
    return dict(median=round(float(np.median(v)), 3), min=round(float(v.min()), 3), max=round(float(v.max()), 3))


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1, 100, 10000, 1000000])
    ap.add_argument("--serve-rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, pl = device_info()
    ds = make_synthetic_dataset("ml_1m", seed=0)
    A0 = ds["adj_train"]
    torch.manual_seed(1)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda().eval()
    rng = np.random.default_rng(0)
    res = dict(gpu=name, power_limit=pl, dataset="ml_1m*", nnz=int(A0.nnz), reps=a.reps, batch_size=B,
               max_nodes_per_hop=MNPH, update=[], serve=None)

    # ---- update vs rebuild, per delta size ----
    # (room for the inserts of every timed delta: deletes drawn from the original matrix thin out)
    g = RatingGraph(A0, reserve_nnz=sum(a.sizes) * a.reps // 2 + 1000)
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=MNPH, batch_size=B)
    g.update(*delta(rng, A0, 1000))          # warm-up: module load, allocator, workspace
    for n in a.sizes:
        t_upd, t_ev, t_reb = [], [], []
        for _ in range(a.reps):
            u, v, x = delta(rng, A0, n)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            g.update(u, v, x)
            e1.record()
            torch.cuda.synchronize()
            t_upd.append((time.perf_counter() - t0) * 1e3)
            t_ev.append(e0.elapsed_time(e1))
            # the rebuild path for the same change (from the original matrix: the same matrix size)
            t, _ = wall(lambda: rc.InferenceEngine(m, RatingGraph(apply_scipy(A0, u, v, x)), max_nodes_per_hop=MNPH,
                                                   batch_size=B))
            t_reb.append(t)
        row = dict(delta=n, update_wall_ms=stats(t_upd), update_events_ms=stats(t_ev), rebuild_wall_ms=stats(t_reb))
        row["rebuild / update"] = round(row["rebuild_wall_ms"]["median"] / row["update_wall_ms"]["median"], 1)
        res["update"].append(row)
        print(json.dumps(row), flush=True)
    eng.close()

    # ---- serve loop: update 100 ratings of 50 users, recommend for them ----
    users = rng.choice(A0.shape[0], 50, replace=False)
    g = RatingGraph(A0, reserve_nnz=100 * (a.reps * a.serve_rounds + 2))
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=MNPH, batch_size=B)
    A = A0
    # correctness first: one round on both sides, bit for bit
    u, v, x = delta(rng, A, 100, users)
    g.update(u, v, x)
    A = apply_scipy(A, u, v, x)
    got = eng.recommend(users, K)
    fresh = rc.InferenceEngine(m, RatingGraph(A), max_nodes_per_hop=MNPH, batch_size=B)
    want = fresh.recommend(users, K)
    fresh.close()
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), "kept and rebuilt engines differ"
    t_keep, t_reb = [], []
    for _ in range(a.reps):
        def kept():
            for _ in range(a.serve_rounds):
                u, v, x = delta(rng, A0, 100, users)
                g.update(u, v, x)
                eng.recommend(users, K)

        def rebuilt():
            Ar = A0
            for _ in range(a.serve_rounds):
                u, v, x = delta(rng, A0, 100, users)
                Ar = apply_scipy(Ar, u, v, x)
                e = rc.InferenceEngine(m, RatingGraph(Ar), max_nodes_per_hop=MNPH, batch_size=B)
                e.recommend(users, K)
                e.close()
        t, _ = wall(kept)
        t_keep.append(t / a.serve_rounds)
        t, _ = wall(rebuilt)
        t_reb.append(t / a.serve_rounds)
    eng.close()
    res["serve"] = dict(users=50, ratings_per_round=100, k=K, kept_engine_ms_per_round=stats(t_keep),
                        rebuilt_ms_per_round=stats(t_reb))
    res["serve"]["rebuilt / kept"] = round(res["serve"]["rebuilt_ms_per_round"]["median"] /
                                           res["serve"]["kept_engine_ms_per_round"]["median"], 2)
    print(json.dumps(res["serve"]), flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
