#!/usr/bin/env python
"""Explanation rate of ``explain_pairs`` on ml_1m* (make_synthetic_dataset("ml_1m", seed=0), max_nodes_per_hop 100):
explained pairs/s and occluded subgraphs/s (one per rating of each pair's enclosing subgraph), by

* the inference engine (``InferenceEngine.explain_pairs``: base pass, one host sync for the rating total, occlusion
  pass with on-device positions, masks and extraction beside the forward, one CUDA graph per batch slot, the per-pair
  sort), and
* the per-batch Python loop a user of the existing API writes for the occlusion pass alone: ``extractor.extract(
  pairs=..., pair_ids=...)`` of B positions, an edge mask built with torch ops from the batch's ``edge_ptr``, and
  ``model._launch_forward`` in training mode with that mask and no dropout, on the same positions at the same B.

Both run in one process, alternated, ``--reps`` times each per batch size; device-event timing around each whole run.
Before timing, the loop's occluded scores are checked bit for bit against the engine's.

    python scripts/explain_rate.py [--pairs 50] [--reps 3] [--batch 50 512]
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


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


class Loop:
    """the occlusion pass over the existing API, one batch of positions at a time"""

    def __init__(self, m, eng, pu, pv, num_edges, B):
        self.m, self.B = m, B
        g = eng.graph
        self.ex = SubgraphExtractor(g, [0], [0], [0], np.arange(1, m.num_relations + 1, dtype=np.float32), 1, 1.0,
                                    MNPH, max_batch=B, seed=0)
        q = np.repeat(np.arange(len(pu)), num_edges)
        j = np.concatenate([np.arange(n) for n in num_edges])
        T = len(q)
        self.batches = []
        for s in range(0, T, B):
            idx = np.minimum(np.arange(s, s + B), T - 1)      # the tail padded to B, as the engine does
            u, v = pu[q[idx]], pv[q[idx]]
            self.batches.append((u, v, np.zeros(B, np.int64), u * g.num_items + v,
                                 torch.as_tensor(j[idx], device="cuda"), min(B, T - s)))
        self.out = torch.empty(len(self.batches) * B, dtype=torch.float32, device="cuda")

    def run(self):
        for k, (u, v, lab, pid, j, _) in enumerate(self.batches):
            b = self.ex.extract(pairs=(u, v, lab), pair_ids=pid)
            ep = b._priv["edge_ptr"][:self.B + 1].long()
            a = ep[:-1] + j
            keep = torch.ones(b._priv["edge_cap"], dtype=torch.uint8, device="cuda")
            keep[a] = 0
            keep[a + (ep[1:] - ep[:-1]) // 2] = 0
            pred, _ = self.m._launch_forward(b, True, self.m.make_dropout(False, edge_keep=keep))
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
    ap.add_argument("--pairs", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, nargs="+", default=[50, 512])
    a = ap.parse_args()
    name, pl = device_info()
    A = make_synthetic_dataset("ml_1m", seed=0)["adj_train"]
    torch.manual_seed(1)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda().eval()
    rng = np.random.default_rng(0)
    pu = rng.integers(0, A.shape[0], a.pairs).astype(np.int64)
    pv = rng.integers(0, A.shape[1], a.pairs).astype(np.int64)
    P = len(pu)
    res = dict(gpu=name, power_limit=pl, pairs=P, max_nodes_per_hop=MNPH, reps=a.reps, rows=[])
    for B in a.batch:
        eng = rc.InferenceEngine(m, A, max_nodes_per_hop=MNPH, batch_size=B, sample_seed=0)
        eng.start_explain(pu, pv)
        while eng.step():
            pass
        occ = eng.run["occ"]
        ex = eng.finish()
        num_edges = ex.num_edges.cpu().numpy()
        T = int(num_edges.sum())
        loop = Loop(m, eng, pu, pv, num_edges, B)
        loop.run()
        assert torch.equal(loop.scores(), occ), "engine and loop occluded scores differ at B = %d" % B
        times = dict(engine=[], loop=[])
        for _ in range(a.reps):
            t, _ = timed(lambda: eng.explain_pairs(pu, pv))
            times["engine"].append(t)
            t, _ = timed(loop.run)
            times["loop"].append(t)
        eng.close()
        row = dict(batch=B, occluded=T, plan=m._plans.get(next(iter(k for k in m._plans if k[1] == B)), None))
        for kk, v in times.items():
            v = np.array(v)
            row[kk] = dict(pairs_per_s=round(float(P / np.median(v)), 1),
                           occluded_per_s=dict(median=round(float(T / np.median(v)), 1),
                                               min=round(float(T / v.max()), 1), max=round(float(T / v.min()), 1)))
        row["engine / loop"] = round(float(np.median(times["loop"]) / np.median(times["engine"])), 3)
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
