#!/usr/bin/env python
"""Rate of question ranking (``elicit``) on ml_1m* (make_synthetic_dataset("ml_1m", seed=0): 6 040 x 3 706, 900 188
ratings), max_nodes_per_hop 100, against the same ranking composed by hand: per session one ``RatingSessions`` of a
session per (question, answer) and one ``predict_sessions`` call, the impact aggregated with torch in slot order and
the questions ranked by a stable sort.

An IGMC is fine-tuned briefly (``OnlineTrainer``, ``--train-steps`` steps of batch 50).  ``--sessions`` sessions, half
new users with 5 random ratings and half graph users with 20..200 ratings, are asked about the ``--questions`` most-rated
items (each session's own rated items excluded); each session's targets are its ``recommend_sessions`` top
``--targets`` items.  With A = 5 answers that is questions x 5 x targets forwards per session.  The two variants run on
the same sessions, are alternated ``--reps`` times and must give equal results.  Reported: forwards/s, median and
min-max over host wall clock around each whole run (both end in a device synchronise), with the GPU's name and power
limit read in the same run.

Does it ask well?  On the real flixster split (tests/golden/flixster_ratings.npz: 3 000 x 3 000, 23 556 training and
2 617 test ratings, 10 rating levels), IGMC is trained as in DESIGN §16 (``train_multiple_epochs``, ``--epochs`` epochs
of batch 50, lr 1e-3 decayed by 0.1 at half time, ARR 0.001).  Every test user with at least ``--min-test`` held-out
ratings and ``--min-train`` training ratings starts from a session that deletes the user's whole training row.  The
questions are restricted to the items the user rated in training, so every answer is known, and the targets are the
user's test items.  Three strategies ask up to five questions each, answered with the true training rating:
``elicit`` (re-asked after each answer, one question per step), popularity (the items with the most training ratings
first, ties by item) and random (a seeded permutation per user).  Reported: the RMSE over all the users' test ratings
of ``predict_sessions`` after 0..5 answers, per strategy.

    python scripts/elicit_rate.py [--part rate|study|both] [--sessions 100] [--questions 200] [--targets 20]
                                  [--batch 256] [--reps 3] [--epochs 30] [--min-test 5] [--min-train 5] [--out F]
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

MNPH, A = 100, 5


def rate(a, name, pl):
    Adj = make_synthetic_dataset("ml_1m", seed=0)["adj_train"]
    g = RatingGraph(Adj)
    nu, ni = g.shape
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=A, num_bases=4, regression=True).cuda()
    OnlineTrainer(m, g, FusedAdam(m, lr=1e-3), batch_size=50, max_nodes_per_hop=MNPH).train(a.train_steps)
    torch.cuda.synchronize()

    rng = np.random.default_rng(0)
    deg = np.diff(g.host["row_ptr"])[:nu]
    half = a.sessions // 2
    graph_users = rng.choice(np.flatnonzero((deg >= 20) & (deg <= 200)), a.sessions - half, replace=False)
    users = np.r_[nu + np.arange(half), graph_users]
    edits = [(s, int(i), int(rng.integers(1, A + 1))) for s in range(half) for i in rng.choice(ni, 5, replace=False)]
    sess_e, items_e, values_e = (np.array([e[k] for e in edits], np.int64) for k in range(3))
    S = rc.RatingSessions(g, users, sess_e, items_e, values_e)
    opts = dict(max_nodes_per_hop=MNPH, batch_size=a.batch)
    targets = rc.recommend_sessions(m, S, a.targets, **opts)[0].cpu().numpy()
    questions = np.sort(np.argsort(-np.diff(g.host["col_ptr"])[:ni], kind="stable")[:a.questions])
    rp, ci, _ = S.rows()
    per_q = [questions[~np.isin(questions, ci[rp[s]:rp[s + 1]])] for s in range(len(users))]
    n = a.questions

    def device():
        items, top = rc.elicit(m, S, n, targets, questions=questions, **opts)
        return items.cpu().numpy(), top.cpu().numpy()

    def by_hand():
        out_i, out_s = np.full((len(users), n), -1, np.int64), np.full((len(users), n), -np.inf, np.float32)
        for s in range(len(users)):
            q, t = per_q[s], targets[s][targets[s] >= 0]                # the real target slots, in slot order
            W = len(t)
            base = (sess_e == s)
            # one session per (question, answer): s's edits plus (q, a + 1)
            k = np.arange(len(q) * A)
            qs, ans = q[k // A], k % A
            nb = int(base.sum())
            sess = np.r_[np.repeat(k, nb), k]
            it = np.r_[np.tile(items_e[base], len(k)), qs]
            val = np.r_[np.tile(values_e[base], len(k)), ans + 1]
            S2 = rc.RatingSessions(g, np.full(len(k), users[s]), sess, it, val)
            x = rc.predict_sessions(m, S2, np.repeat(k, W), np.tile(t, len(k)), **opts)
            x = x.view(len(q), A, W).double()
            rng_ = x.max(dim=1).values - x.min(dim=1).values            # [Q, W], exact in fp64
            total = torch.zeros(len(q), dtype=torch.float64, device=x.device)
            for w in range(W):                                           # slot order
                total = total + rng_[:, w]
            imp = (total / W).float()
            # a stable sort, not torch.topk: topk does not order ties, recommend's order puts the lower item first
            order = torch.sort(imp, descending=True, stable=True).indices[:n]
            out_i[s, :len(order)] = q[order.cpu().numpy()]
            out_s[s, :len(order)] = imp[order].cpu().numpy()
        return out_i, out_s

    runs = dict(elicit=device, by_hand=by_hand)
    first = {k: fn() for k, fn in runs.items()}            # warm-up, and the results compared
    assert np.array_equal(first["elicit"][0], first["by_hand"][0])
    assert np.array_equal(first["elicit"][1], first["by_hand"][1])
    fw = sum(len(q) * A * int((t >= 0).sum()) for q, t in zip(per_q, targets))
    times = {k: [] for k in runs}
    for _ in range(a.reps):
        for k, fn in runs.items():
            times[k].append(wall(fn)[0])
    res = dict(gpu=name, power_limit=pl, dataset="ml_1m*", max_nodes_per_hop=MNPH, batch_size=a.batch,
               train_steps=a.train_steps, sessions=len(users), new_users=half, questions=a.questions,
               targets=int(targets.shape[1]), answers=A, forwards=fw, reps=a.reps)
    for k in runs:
        res[k] = dict(forwards_per_s=stats([fw / t for t in times[k]], 0), seconds=stats(times[k], 3))
    res["elicit / by_hand"] = round(float(np.median(times["by_hand"]) / np.median(times["elicit"])), 2)
    print(json.dumps(dict(rate=res), indent=1), flush=True)
    return res


def study(a):
    from igmc_b200.train_eval import train_multiple_epochs
    from igmc_b200.util_functions import MyDataset
    ds = make_synthetic_dataset("flixster", seed=0)
    assert ds.get("real"), "the flixster fixture is missing"
    Adj, cv, R = ds["adj_train"], ds["class_values"], ds["num_relations"]
    tu, tv, tl = ds["train"]
    su, sv, sl = ds["test"]
    mk = lambda u, v, l: MyDataset(None, Adj, (u, v), l, 1, 1.0, ds["max_nodes_per_hop"], None, None, cv, seed=0)  # noqa
    torch.manual_seed(1)
    train = mk(tu, tv, tl)
    m = IGMC(train, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True,
             adj_dropout=ds["adj_dropout"]).cuda()
    rmse_train = train_multiple_epochs(train, mk(su, sv, sl), m, a.epochs, 50, 1e-3, 0.1, max(a.epochs // 2, 1), 0,
                                       ARR=0.001)
    m.eval()
    g = RatingGraph(Adj)
    rp, ci, rt = g.host["row_ptr"], g.host["col_idx"], g.host["rating"]
    deg = np.diff(rp)[:g.shape[0]]
    ntest = np.bincount(su, minlength=g.shape[0])
    users = np.flatnonzero((ntest >= a.min_test) & (deg >= a.min_train))
    U = len(users)
    W = int(ntest[users].max())
    targets = np.full((U, W), -1, np.int64)                   # each user's test items, -1 padded
    pairs_s, pairs_v, y = [], [], []
    for s, u in enumerate(users):
        t = sv[su == u]
        targets[s, :len(t)] = t
        pairs_s += [s] * len(t)
        pairs_v += list(t)
        y += list(cv[sl[su == u]])
    y = np.asarray(y, np.float64)
    train_rows = [(ci[rp[u]:rp[u + 1]].astype(np.int64), rt[rp[u]:rp[u + 1]].astype(np.int64)) for u in users]
    opts = dict(max_nodes_per_hop=ds["max_nodes_per_hop"], batch_size=max(256, R * W))
    col_deg = np.diff(g.host["col_ptr"])[:g.shape[1]]
    rng = np.random.default_rng(0)
    fixed = dict(popularity=[r[0][np.lexsort((r[0], -col_deg[r[0]]))] for r in train_rows],
                 random=[rng.permutation(r[0]) for r in train_rows])

    def sessions(asked):
        """the users with their training rows deleted and the asked items answered with their training labels"""
        sess, items, vals = [], [], []
        for s, (row, lab) in enumerate(train_rows):
            answered = dict(zip(row.tolist(), (lab + 1).tolist()))
            for i in row:
                sess.append(s)
                items.append(int(i))
                vals.append(0)
            for q in asked[s]:
                sess.append(s)
                items.append(int(q))
                vals.append(answered[int(q)])
        return rc.RatingSessions(g, users, sess, items, vals)

    def rmse(S):
        x = rc.predict_sessions(m, S, pairs_s, pairs_v, **opts).double().cpu().numpy()
        return round(float(np.sqrt(np.mean((x - y) ** 2))), 4)

    steps = 5
    out = {}
    for strategy in ("elicit", "popularity", "random"):
        asked = [[] for _ in range(U)]
        curve = [rmse(sessions(asked))]
        for _ in range(steps):
            if strategy == "elicit":
                S = sessions(asked)
                qrows = np.full((U, max(len(r[0]) for r in train_rows)), -1, np.int64)
                for s, r in enumerate(train_rows):
                    qrows[s, :len(r[0])] = r[0]
                best = rc.elicit(m, S, 1, targets, questions=qrows, **opts)[0].cpu().numpy()[:, 0]
                for s in range(U):
                    if best[s] >= 0:                          # -1: the user's training row is used up
                        asked[s].append(int(best[s]))
            else:
                for s in range(U):
                    if len(asked[s]) < len(fixed[strategy][s]):
                        asked[s].append(int(fixed[strategy][s][len(asked[s])]))
            curve.append(rmse(sessions(asked)))
        out[strategy] = curve
    res = dict(epochs=a.epochs, train_multiple_epochs_test_rmse=round(float(rmse_train), 4), users=U,
               test_ratings=len(y), min_test=a.min_test, min_train=a.min_train,
               full_training_row_rmse=rmse(sessions([list(r[0]) for r in train_rows])),
               rmse_after_answers={k: dict(zip(range(steps + 1), v)) for k, v in out.items()})
    print(json.dumps(dict(study=res), indent=1), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=("rate", "study", "both"), default="both")
    ap.add_argument("--sessions", type=int, default=100)
    ap.add_argument("--questions", type=int, default=200)
    ap.add_argument("--targets", type=int, default=20)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--train-steps", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--epochs", type=int, default=30)
    ap.add_argument("--min-test", type=int, default=5)
    ap.add_argument("--min-train", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, pl = device_info()
    res = dict(gpu=name, power_limit=pl)
    if a.part in ("rate", "both"):
        res["rate"] = rate(a, name, pl)
    if a.part in ("study", "both"):
        res["study"] = study(a)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
