#!/usr/bin/env python
"""Rate of group recommendation (``recommend_groups``) on ml_1m* (make_synthetic_dataset("ml_1m", seed=0): 6 040 x
3 706, 900 188 ratings), max_nodes_per_hop 100, k = 10, against the same lists composed by hand on the same engine:
the union of the members' rows excluded in numpy, every (member, candidate) pair through ``predict_pairs``, the
aggregate in torch (fp64 member by member for the mean, strict compares for the minimum) and a stable sort.

An IGMC is fine-tuned briefly (``OnlineTrainer``, ``--train-steps`` steps of batch 50).  ``--groups`` seeded groups of
2..8 users, drawn from the users with 20..200 ratings, are ranked over the full catalogue with ``mean`` and ``min``
at every ``--batch`` size.  The two sides must give equal lists before any time is kept, and are then alternated
``--reps`` times.  Reported per batch size and aggregate: real member pairs per second, median and min-max over host
wall clock around each whole run (both end in a device synchronise); the padding fill ratio of the fused run, real
positions / (steps x B), with units of the largest group size M taking B // M x M positions of each batch; and the
GPU's name and power limit, read in the same run.

    python scripts/group_rate.py [--groups 1000] [--batch 256 512] [--reps 2] [--train-steps 300] [--out F]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC, FusedAdam  # noqa: E402
from igmc_b200.train_eval import OnlineTrainer  # noqa: E402
from igmc_b200.util_functions import RatingGraph  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from counterfactual_rate import device_info, stats, wall  # noqa: E402

MNPH, K_TOP = 100, 10


def by_hand(eng, g, groups, members, agg, k):
    """the lists composed from predict_pairs: (items [G, k], scores [G, k]) as host arrays"""
    rp, ci, ni = g.host["row_ptr"], g.host["col_idx"], g.num_items
    cand = [np.setdiff1d(np.arange(ni), np.concatenate([ci[rp[u]:rp[u + 1]] for u in grp])) for grp in groups]
    units = np.concatenate([np.full(len(c), j, np.int64) for j, c in enumerate(cand)])
    items = np.concatenate(cand).astype(np.int64)
    M = members.shape[1]
    mem = members[units]                                          # [units, M], -1 past each group's size
    valid = mem >= 0
    x = torch.full(mem.shape, float("nan"), dtype=torch.float32, device=eng.dev)
    vt = torch.from_numpy(valid).to(eng.dev)
    x[vt] = eng.predict_pairs(mem[valid], np.broadcast_to(items[:, None], mem.shape)[valid])
    if agg == "mean":
        total = torch.zeros(len(items), dtype=torch.float64, device=eng.dev)
        for j in range(M):                                        # member order, one add per member
            total = total + torch.where(vt[:, j], x[:, j].double(), torch.zeros_like(total))
        key = (total / vt.sum(1)).float()
    else:
        key = x[:, 0].clone()
        for j in range(1, M):
            key = torch.where(vt[:, j] & (x[:, j] < key), x[:, j], key)
        key = torch.where(torch.isnan(x).logical_and(vt).any(1), torch.full_like(key, float("nan")), key)
    # a stable sort per group: key descending, the candidates (ascending within a group) in order on ties
    out_i, out_s = np.full((len(groups), k), -1, np.int64), np.full((len(groups), k), -np.inf, np.float32)
    off = np.concatenate([[0], np.cumsum([len(c) for c in cand])])
    for j in range(len(groups)):
        kk = key[off[j]:off[j + 1]]
        order = torch.sort(kk, descending=True, stable=True).indices[:k]
        n = len(order)
        out_i[j, :n] = items[off[j]:off[j + 1]][order.cpu().numpy()]
        out_s[j, :n] = kk[order].cpu().numpy()
    return out_i, out_s, int(valid.sum()), len(items)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1000)
    ap.add_argument("--batch", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--train-steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, pl = device_info()
    print(json.dumps(dict(gpu=name, power_limit=pl)), flush=True)
    Adj = make_synthetic_dataset("ml_1m", seed=0)["adj_train"]
    g = RatingGraph(Adj)
    nu = g.num_users
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    OnlineTrainer(m, g, FusedAdam(m, lr=1e-3), batch_size=50, max_nodes_per_hop=MNPH).train(a.train_steps)
    torch.cuda.synchronize()

    rng = np.random.default_rng(0)
    deg = np.diff(g.host["row_ptr"])[:nu]
    pool = np.flatnonzero((deg >= 20) & (deg <= 200))
    groups = [[int(u) for u in rng.choice(pool, int(rng.integers(2, 9)), replace=False)] for _ in range(a.groups)]
    members = rc._group_members(groups, nu, min(a.batch))
    M = members.shape[1]
    res = dict(gpu=name, power_limit=pl, dataset="ml_1m*", max_nodes_per_hop=MNPH, k=K_TOP, groups=a.groups,
               group_sizes=[int(x) for x in np.bincount([len(x) for x in groups])[2:]], train_steps=a.train_steps,
               reps=a.reps, runs={})
    for B in a.batch:
        eng = rc.InferenceEngine(m, g, max_nodes_per_hop=MNPH, batch_size=B)
        try:
            for agg in ("mean", "min"):
                def fused():
                    ti, ts = eng.recommend_groups(groups, K_TOP, agg)
                    return ti.cpu().numpy(), ts.cpu().numpy()

                def hand():
                    return by_hand(eng, g, groups, members, agg, K_TOP)
                got, want = fused(), hand()                       # warm-up, and the results compared
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (B, agg)
                pairs, units = want[2], want[3]
                times = dict(fused=[], by_hand=[])
                for _ in range(a.reps):
                    times["fused"].append(wall(fused)[0])
                    times["by_hand"].append(wall(hand)[0])
                Gu = B // M
                steps = (units + Gu - 1) // Gu
                r = dict(member_pairs=pairs, units=units, fill=round(pairs / (steps * B), 4))
                for kk, t in times.items():
                    r[kk] = dict(pairs_per_s=stats([pairs / x for x in t], 0), seconds=stats(t, 2))
                r["fused / by_hand"] = round(float(np.median(times["by_hand"]) / np.median(times["fused"])), 2)
                res["runs"]["B=%d %s" % (B, agg)] = r
                print(json.dumps({"B=%d %s" % (B, agg): r}), flush=True)
        finally:
            eng.close()
    print(json.dumps(dict(rate=res), indent=1), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
