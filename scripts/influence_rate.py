#!/usr/bin/env python
"""Training-pair rate of ``influence`` on ml_1m* (make_synthetic_dataset("ml_1m", seed=0), max_nodes_per_hop 100):
the first ``--train`` training ratings of the dataset against T = 64 test pairs of its test split, K = 1 and 3
checkpoints, batch sizes 50 and 256.

* engine arm: the whole ``influence`` call (test-gradient pass, training pass, top-k merges), device events;
* split: the same training pairs through ``self_influence`` (forward, seed, backward, per-pair assembly and a norm per
  pair, no GEMM), so that influence - self_influence - test pass approximates the accumulation (GEMM, factor terms,
  merge);
* loop arm, the only per-pair gradient the training API offers: a B = 1 ``fused_step(ARR=0)`` per training pair (both
  dropout rates 0) and a dot product of its flat_grad with the stored test gradients, over ``--loop`` pairs.

Both arms are first checked to agree (the loop's values against the engine's, max |diff| <= 1e-3 of the largest value),
then alternated ``--reps`` times.  Prints one JSON line per configuration with pairs/s (median, min, max), the GPU name
and its power limit read in the same run.

    python scripts/influence_rate.py [--train 100000] [--loop 200] [--reps 3]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from igmc_b200 import recommend as rc  # noqa: E402
from igmc_b200.data import make_synthetic_dataset  # noqa: E402
from igmc_b200.models import IGMC  # noqa: E402
from igmc_b200.util_functions import RatingGraph, SubgraphExtractor  # noqa: E402
from scripts.explain_rate import MNPH, device_info  # noqa: E402

T_TEST = 64


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1000.0, out


class Loop:
    """B = 1 fused_step per training pair, dot with the stored test gradients [T, param_count]"""

    def __init__(self, m, A, R, seed):
        self.m, self.ni = m, A.shape[1]
        self.ex = SubgraphExtractor(RatingGraph(A), [0], [0], [0], np.arange(1, R + 1, dtype=np.float32), 1, 1.0,
                                    MNPH, max_batch=1, seed=seed)

    def run(self, u, v, lab, Gt):
        out = torch.empty(len(u), Gt.shape[0], device="cuda")
        for i in range(len(u)):
            b = self.ex.extract(pairs=(u[i:i + 1], v[i:i + 1], lab[i:i + 1]), pair_ids=u[i:i + 1] * self.ni + v[i:i + 1])
            self.m.fused_step(b, ARR=0.0)
            out[i] = Gt @ self.m.flat_grad
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train", type=int, default=100000)
    ap.add_argument("--loop", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    ds = make_synthetic_dataset("ml_1m", seed=0)
    A = ds["adj_train"]
    R = len(ds["class_values"])
    tu, tv, tl = (np.asarray(x)[:a.train] for x in ds["train"])
    train = (tu.astype(np.int64), tv.astype(np.int64), (tl + 1).astype(np.float32))
    qu, qv, ql = (np.asarray(x)[:T_TEST] for x in ds["test"])
    test = (qu.astype(np.int64), qv.astype(np.int64), (ql + 1).astype(np.float32))
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True).cuda()
    m.adj_dropout, m.hidden_dropout_p = 0.0, 0.0
    name, pl = device_info()
    N = len(train[0])
    # agreement of the two arms on the loop's subset
    L = a.loop
    sub = tuple(x[:L] for x in train)
    Gt = rc.pair_gradients(m, A, *test, max_nodes_per_hop=MNPH, sample_seed=0)[0]
    loop = Loop(m, A, R, 0)
    lv = loop.run(sub[0], sub[1], (sub[2] - 1).astype(np.int64), Gt)
    inf = rc.influence(m, A, sub, test, L, max_nodes_per_hop=MNPH, sample_seed=0)
    ev = torch.zeros(L, T_TEST, device="cuda")
    for t in range(T_TEST):
        ev[inf.pro_index[t], t] = inf.pro_value[t]
    diff = float((ev - lv).abs().max()) / float(lv.abs().max())
    print(json.dumps(dict(check="loop vs engine", pairs=L, max_rel_diff=diff)), flush=True)
    assert diff <= 1e-3, diff
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for c in range(3):
            paths.append(os.path.join(tmp, "ck%d.pth" % c))
            torch.manual_seed(c + 1)
            torch.save(IGMC(4, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True).state_dict(),
                       paths[-1])
        for K in (1, 3):
            ck = paths[:K] if K > 1 else None
            for B in (50, 256):
                kw = dict(max_nodes_per_hop=MNPH, batch_size=B, checkpoints=ck, sample_seed=0)
                rc.influence(m, A, tuple(x[:2 * B] for x in train), test, 10, **kw)      # warm-up of every shape
                rc.self_influence(m, A, tuple(x[:2 * B] for x in train), **kw)
                t_inf, t_self, t_loop = [], [], []
                for _ in range(a.reps):
                    t_inf.append(timed(lambda: rc.influence(m, A, train, test, 10, **kw))[0])
                    t_self.append(timed(lambda: rc.self_influence(m, A, train, **kw))[0])
                    t_loop.append(timed(lambda: [loop.run(sub[0], sub[1], (sub[2] - 1).astype(np.int64), Gt)
                                                 for _ in range(K)])[0])
                rate = lambda ts, n: dict(median=n / float(np.median(ts)), min=n / max(ts), max=n / min(ts))
                print(json.dumps(dict(K=K, B=B, T=T_TEST, train_pairs=N, engine_pairs_per_s=rate(t_inf, N),
                                      self_influence_pairs_per_s=rate(t_self, N),
                                      accumulation_share=1.0 - float(np.median(t_self)) / float(np.median(t_inf)),
                                      loop_pairs_per_s=rate(t_loop, L), gpu=name, power_limit=pl)), flush=True)


if __name__ == "__main__":
    main()
