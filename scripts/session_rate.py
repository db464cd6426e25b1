"""Rate of scoring new users from ratings passed with the query (recommend_sessions) against the route that existed
before rating sessions: per user a graph.update insert, recommend([u]) and a graph.update delete.

ml_1m*, max_nodes_per_hop 100, B = 256, 256 new-user sessions of 20 ratings each, drawn from real users' rows.  Both
arms' top-10 lists are checked to be identical before timing.  Reports sessions/s (median and min-max of 3 alternated
runs, device events around whole runs), the card and its power limit."""
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
from igmc_b200.util_functions import RatingGraph  # noqa: E402


def _power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def main(S=256, per=20, k=10, M=200, B=256, mnph=100, full=16):
    ds = make_synthetic_dataset("ml_1m", seed=0)
    A = ds["adj_train"]
    nu, ni = A.shape
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True).cuda()
    g = RatingGraph(A, reserve_nnz=per, reserve_users=1)
    rng = np.random.default_rng(0)
    deg = np.diff(A.indptr)
    donors = rng.choice(np.flatnonzero(deg >= per), S, replace=False)
    session, items, values = [], [], []
    for s, d in enumerate(donors):
        row = A.indices[A.indptr[d]:A.indptr[d + 1]]
        pick = np.sort(rng.choice(len(row), per, replace=False))
        session += [s] * per
        items += row[pick].tolist()
        values += np.rint(A.data[A.indptr[d] + pick]).astype(np.int64).tolist()
    session, items, values = (np.asarray(a, np.int64) for a in (session, items, values))
    users = np.full(S, nu)          # every session is the same unseen user id
    eng = rc.InferenceEngine(m, g, max_nodes_per_hop=mnph, batch_size=B)

    def sessions_arm(n, retrieve):
        sel = session < n
        sess = rc.RatingSessions(g, users[:n], session[sel], items[sel], values[sel])
        return eng.recommend_sessions(sess, k, retrieve=retrieve)

    def update_arm(n, retrieve):
        outs = []
        for s in range(n):
            sel = session == s
            g.update(np.full(sel.sum(), nu), items[sel], values[sel])
            outs.append(eng.recommend([nu], k, retrieve=retrieve))
            g.update(np.full(sel.sum(), nu), items[sel], np.zeros(sel.sum(), np.int64))
        return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])

    res = {}
    for name, n, retrieve in (("retrieve", S, M), ("catalogue", full, None)):
        a, b = sessions_arm(n, retrieve), update_arm(n, retrieve)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), name
        times = {"sessions": [], "update": []}
        for _ in range(3):
            for arm, fn in (("sessions", sessions_arm), ("update", update_arm)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                fn(n, retrieve)
                e1.record()
                torch.cuda.synchronize()
                times[arm].append(n / (e0.elapsed_time(e1) / 1000.0))
        res[name] = {arm: dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v)), sessions=n)
                     for arm, v in times.items()}
    eng.close()
    out = dict(card=torch.cuda.get_device_name(0), power_limit=_power_limit(), k=k, retrieve=M, batch=B, mnph=mnph,
               ratings_per_session=per, sessions_per_s=res)
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
