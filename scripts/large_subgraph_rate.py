#!/usr/bin/env python
"""Train-step rate (subgraphs/s, batch 50) on enclosing subgraphs too large for the shared-memory kernel plans, i.e.
on the L2 plan (csrc/rgcn_l2.cu), next to the PyG formulation on torch CUDA (bench.gpu_baseline's model: index_select
+ bmm + scatter-mean, autograd, torch.optim.Adam) on the same batches.

Both arms time the model half of a step only (forward + loss + backward + gradient assembly + Adam) on four batches
extracted once on the device, with CUDA events, after warm-up; every figure is the median of ``--reps`` timed runs.

    python scripts/large_subgraph_rate.py [--steps 20] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200 import _lib  # noqa: E402
from igmc_b200.data import build_adj, make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC, FusedAdam  # noqa: E402
from igmc_b200.util_functions import MyDynamicDataset  # noqa: E402
from oracle import pyg_restated  # noqa: E402

B = 50
ARR = 0.001


def device_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        pl = "unknown (%s)" % e
    return name, pl


def synthetic_r71():
    """600 x 600 ratings with 71 levels; the longest row has 281 entries, so n_cap = 2 * 282 = 564"""
    R, nu, nv = 71, 600, 600
    rng = np.random.default_rng(4)
    u, v = np.nonzero(rng.random((nu, nv)) < 0.3)
    keep = ~((u == 0) & (v >= 281))
    u, v = np.concatenate([u[keep], np.zeros(281, np.int64)]), np.concatenate([v[keep], np.arange(281)])
    uv = np.unique(u * nv + v)
    u, v = uv // nv, uv % nv
    lab = rng.integers(0, R, len(u))
    A = build_adj(u, v, lab, nu, nv)
    perm = rng.permutation(len(u))
    return dict(adj_train=A, train=(u[perm], v[perm], lab[perm]), class_values=np.arange(1, R + 1, dtype=np.float32),
                adj_dropout=0.2)


def batches(ds, h, mnph, k=4):
    tu, tv, tl = ds["train"]
    n = k * B
    d = MyDynamicDataset(None, ds["adj_train"], (tu[:n], tv[:n]), tl[:n], h, 1.0, mnph, None, None,
                         ds["class_values"], seed=1)
    out = [d.extract_batch(np.arange(i * B, (i + 1) * B)) for i in range(k)]
    for b in out:
        b.adjacency()
    return out


def time_steps(fn, n_batches, steps, reps):
    for k in range(3):
        fn(k % n_batches)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(steps):
            fn(k % n_batches)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / steps)
    return float(np.median(ms))


def ours(bs, in0, R, plan, steps, reps, adj_dropout):
    torch.manual_seed(0)
    m = IGMC(in0, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True, adj_dropout=adj_dropout).cuda()
    m.kernel_plan = plan
    opt = FusedAdam(m, lr=1e-3)

    def one(k):
        loss = m.fused_step(bs[k], ARR=ARR)
        opt.step(loss_in=loss)
    ms = time_steps(one, len(bs), steps, reps)
    for b in bs:
        b.check()
    return ms, m._plan(bs[0])


def baseline(bs, in0, R, steps, reps, adj_dropout):
    torch.manual_seed(1)
    ref = pyg_restated.IGMCRef(in0, (32, 32, 32, 32), R, 4, adj_dropout).cuda().train()
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    tbs = [dict(x=b.x.clone(), edge_index=b.edge_index.clone(), edge_type=b.edge_type.clone(), y=b.y.clone())
           for b in bs]

    def one(k):
        opt.zero_grad()
        loss, _ = pyg_restated.train_loss(ref, tbs[k], ARR)
        loss.backward()
        opt.step()
    return time_steps(one, len(bs), max(2, steps // 4), reps)


def rate(ms):
    return round(B / (ms / 1000.0), 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    name, pl = device_info()
    res = dict(gpu=name, power_limit=pl, batch=B, steps=a.steps, reps=a.reps, configs=[])
    ml = make_synthetic_dataset("ml_100k", seed=0)
    ml["adj_dropout"] = 0.2
    configs = [("ml_100k* h=1 no node cap", ml, 1, None, 5),
               ("ml_100k* h=2 mnph=200", ml, 2, 200, 5),
               ("synthetic R=71 n_cap=564", synthetic_r71(), 1, None, 71)]
    for tag, ds, h, mnph, R in configs:
        bs = batches(ds, h, mnph)
        in0 = 2 * h + 2
        ms, plan = ours(bs, in0, R, "auto", a.steps, a.reps, ds["adj_dropout"])
        row = dict(config=tag, n_cap=bs[0]._priv["n_cap"], plan=plan, l2_ctas=_lib.l2_csize(plan),
                   ours_subgraphs_s=rate(ms), ours_ms=round(ms, 3))
        # CTAs per subgraph of the L2 plan: what the selection rule (models.l2_cluster) rests on
        row["l2_by_ctas"] = {c: rate(ours(bs, in0, R, _lib.plan_l2(c), a.steps, a.reps, ds["adj_dropout"])[0])
                             for c in (1, 2, 4, 8)}
        bl = baseline(bs, in0, R, a.steps, a.reps, ds["adj_dropout"])
        row.update(baseline_subgraphs_s=rate(bl), baseline_ms=round(bl, 3), speedup=round(bl / ms, 2))
        res["configs"].append(row)
        print(json.dumps(row), flush=True)
    # the cost of L2-resident features: ml_100k* at mnph 200 (402-node subgraphs) on plan 4 and on the L2 plan,
    # alternated run by run
    bs = batches(ml, 1, 200)
    alt = {4: [], "l2": []}
    for _ in range(a.reps):
        alt[4].append(ours(bs, 4, 5, 4, a.steps, 1, 0.2)[0])
        alt["l2"].append(ours(bs, 4, 5, _lib.plan_l2(4), a.steps, 1, 0.2)[0])
    bl = baseline(bs, 4, 5, a.steps, a.reps, 0.2)
    row = dict(config="ml_100k* h=1 mnph=200: plan 4 vs L2 plan (4 CTAs), alternated",
               plan4_subgraphs_s=rate(float(np.median(alt[4]))), l2_subgraphs_s=rate(float(np.median(alt["l2"]))),
               baseline_subgraphs_s=rate(bl))
    res["configs"].append(row)
    print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
