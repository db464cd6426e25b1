#!/usr/bin/env python
"""Scoring rate (candidate pairs/s) of the full-catalogue ranking workload: every unrated item of 500 ml_1m* users
(make_synthetic_dataset("ml_1m", seed=0), max_nodes_per_hop 100, about 1.8 M pairs), by

* the inference engine (``InferenceEngine.recommend``: on-device candidate pairs, extraction of the next batch beside
  the forward, streaming top-k merge, one CUDA graph per batch slot), and
* the per-batch Python loop a user of the existing API writes: ``extractor.extract(pairs=..., pair_ids=...)`` +
  ``model._launch_forward`` + a copy of the predictions, on the same pairs in the same order, at the same B.

Both run in one process, alternated, ``--reps`` times each per batch size; device-event timing around each whole run.
Before timing, the engine's scores of the same pairs (``predict_pairs`` mode) are checked bit for bit against the
loop's, and its top-k against a stable sort of those scores for a few users.

    python scripts/recommend_rate.py [--users 500] [--reps 2] [--batch 50 256 512]
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
from igmc_b200.util_functions import SubgraphExtractor  # noqa: E402

MNPH = 100
K = 10


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


class Loop:
    """the existing API, one batch at a time"""

    def __init__(self, m, eng, pu, pv, B):
        self.m, self.B = m, B
        g = eng.graph
        self.ex = SubgraphExtractor(g, [0], [0], [0], np.arange(1, m.num_relations + 1, dtype=np.float32), 1, 1.0,
                                    MNPH, max_batch=B, seed=0)
        self.drop = m.make_dropout(False)
        n = len(pu)
        self.batches = []
        for s in range(0, n, B):
            idx = np.minimum(np.arange(s, s + B), n - 1)      # the tail padded to B, as the engine does
            self.batches.append((pu[idx], pv[idx], np.zeros(B, np.int64), pu[idx] * g.num_items + pv[idx],
                                 min(B, n - s)))
        self.out = torch.empty(len(self.batches) * B, dtype=torch.float32, device="cuda")

    def run(self):
        for k, (u, v, lab, pid, _) in enumerate(self.batches):
            b = self.ex.extract(pairs=(u, v, lab), pair_ids=pid)
            pred, _ = self.m._launch_forward(b, False, self.drop)
            self.out[k * self.B:(k + 1) * self.B].copy_(pred)
        b.check()

    def scores(self):
        keep = np.concatenate([np.arange(k * self.B, k * self.B + n) for k, (*_, n) in enumerate(self.batches)])
        return self.out[torch.as_tensor(keep, device="cuda")]


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1000.0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=500)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--batch", type=int, nargs="+", default=[50, 256, 512])
    a = ap.parse_args()
    name, pl = device_info()
    ds = make_synthetic_dataset("ml_1m", seed=0)
    A = ds["adj_train"]
    torch.manual_seed(1)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda().eval()
    users = np.random.default_rng(0).choice(A.shape[0], a.users, replace=False)
    ni = A.shape[1]
    lists = [np.setdiff1d(np.arange(ni), A.indices[A.indptr[u]:A.indptr[u + 1]]) for u in users]
    pu = np.concatenate([np.full(len(l_), u, np.int64) for u, l_ in zip(users, lists)])
    pv = np.concatenate(lists).astype(np.int64)
    P = len(pu)
    res = dict(gpu=name, power_limit=pl, users=a.users, pairs=P, max_nodes_per_hop=MNPH, k=K, reps=a.reps, rows=[])
    for B in a.batch:
        eng = rc.InferenceEngine(m, A, max_nodes_per_hop=MNPH, batch_size=B, sample_seed=0)
        loop = Loop(m, eng, pu, pv, B)
        loop.run()
        ref = loop.scores()
        got = eng.predict_pairs(pu, pv)
        assert torch.equal(got, ref), "engine and loop scores differ at B = %d" % B
        flat = got.cpu().numpy()
        top_i, top_s = eng.recommend(users, K)
        off = np.concatenate([[0], np.cumsum([len(l_) for l_ in lists])])
        for j in range(min(5, len(users))):
            ws, wi = rc.rank_host(flat[off[j]:off[j + 1]], lists[j], K)
            assert np.array_equal(top_i[j].cpu().numpy(), wi) and np.array_equal(top_s[j].cpu().numpy(), ws)
        rates = dict(engine=[], loop=[])
        for _ in range(a.reps):
            t, _ = timed(lambda: eng.recommend(users, K))
            rates["engine"].append(P / t)
            t, _ = timed(loop.run)
            rates["loop"].append(P / t)
        eng.close()
        row = dict(batch=B, plan=m._plans.get(next(iter(k for k in m._plans if k[1] == B)), None))
        for kk, v in rates.items():
            v = np.array(v)
            row[kk] = dict(median=round(float(np.median(v)), 1), min=round(float(v.min()), 1),
                           max=round(float(v.max()), 1))
        row["engine / loop"] = round(row["engine"]["median"] / row["loop"]["median"], 3)
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
