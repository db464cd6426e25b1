"""Keeping served top-k lists current as ratings arrive: RecommendationCache.update against graph.update followed by a
full re-rank (InferenceEngine.recommend) of the same users.

Setup: ml_1m* (the synthetic ml_1m-sized matrix), max_nodes_per_hop 100, batch 256, all 6 040 users, k = 10, cache
depth 10 and 50.  Each round draws one batch of 1 / 10 / 100 / 1 000 edits (inserts, overwrites and deletes) and applies
it to three copies of the graph: one per cache and one for the full side, timed in turn (full, depth 10, depth 50).
Every round checks both caches' lists bit for bit against the full side's before its times are kept.  Reports the
median and min-max wall time, the rescored pairs and the users that fell back to a full re-rank, with the GPU name and
power limit read in the same run.

    python scripts/recommend_cache_rate.py [--reps 2] [--out result.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from graph_update_rate import B, K, MNPH, delta, device_info, stats, wall  # noqa: E402
from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC  # noqa: E402
from igmc_b200.util_functions import RatingGraph  # noqa: E402

DEPTHS = (10, 50)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1, 10, 100, 1000])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, pl = device_info()
    A0 = make_synthetic_dataset("ml_1m", seed=0)["adj_train"]
    torch.manual_seed(1)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda().eval()
    users = np.arange(A0.shape[0])
    reserve = dict(reserve_nnz=sum(a.sizes) * a.reps + 16)
    g_full = RatingGraph(A0, **reserve)
    eng = rc.InferenceEngine(m, g_full, max_nodes_per_hop=MNPH, batch_size=B)
    caches = {d: rc.RecommendationCache(m, RatingGraph(A0, **reserve), users, K, depth=d, max_nodes_per_hop=MNPH,
                                        batch_size=B) for d in DEPTHS}
    rng = np.random.default_rng(0)
    res = dict(gpu=name, power_limit=pl, dataset="ml_1m*", users=len(users), k=K, batch_size=B,
               max_nodes_per_hop=MNPH, reps=a.reps, rows=[])

    def full_side(u, v, x):
        g_full.update(u, v, x)
        return eng.recommend(users, K)
    for n in a.sizes:
        t = {"full": []}
        t.update({d: [] for d in DEPTHS})
        info = {d: [] for d in DEPTHS}
        for _ in range(a.reps):
            u, v, x = delta(rng, _scipy(g_full), n)
            ms, (wi, ws) = wall(lambda: full_side(u, v, x))
            t["full"].append(ms)
            for d, c in caches.items():
                ms, out = wall(lambda: c.update(u, v, x))
                gi, gs = c.lists()
                assert torch.equal(gi, wi) and torch.equal(gs.view(torch.int32), ws.view(torch.int32)), (n, d, out)
                t[d].append(ms)
                info[d].append(out)
        row = dict(edits=n, full_ms=stats(t["full"]))
        for d in DEPTHS:
            row["depth%d" % d] = dict(ms=stats(t[d]), rescored_pairs=[o["rescored_pairs"] for o in info[d]],
                                      fallback_users=[o["rebuilt_users"] for o in info[d]],
                                      full_rebuild=[o["full"] for o in info[d]])
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    for c in caches.values():
        c.close()
    eng.close()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


def _scipy(g):
    """the graph as a scipy CSR (delta draws its overwrites and deletes from the current ratings)"""
    import scipy.sparse as ssp
    h = g.host
    return ssp.csr_matrix((h["rating"].astype(np.float32) + 1, h["col_idx"], h["row_ptr"]), shape=g.shape)


if __name__ == "__main__":
    main()
