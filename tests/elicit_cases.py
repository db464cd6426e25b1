"""Cases for igmc_elicit_pairs / igmc_elicit_stats and plain-Python brute forces written from their contracts in
include/igmc_b200.h.  tests/test_elicit_host.py checks the numpy twins in igmc_b200/recommend.py against the brute
forces on the host; tests/test_gpu_elicit_kernels.py calls the kernels on the same cases."""
import struct

import numpy as np

PAIR_THREADS = 512   # csrc/elicit.cu: one chunk of k_el_pairs' position loop and row-length scan
ROW_THREADS = 128    # csrc/elicit.cu: one stride of a k_el_rows row
STATS_THREADS = 128  # csrc/elicit.cu: units per k_el_stats CTA
CONSTANTS = {("elicit.cu", "PAIR_THREADS"): PAIR_THREADS, ("elicit.cu", "ROW_THREADS"): ROW_THREADS,
             ("elicit.cu", "STATS_THREADS"): STATS_THREADS}


def f32(x):
    """x rounded to fp32, as a Python float"""
    return struct.unpack("f", struct.pack("f", x))[0]


# ---- igmc_elicit_pairs ------------------------------------------------------------------------------------------------
def csr(rows):
    """session rows [[(item, label), ...] ascending] -> (row_ptr, col_idx, rating) numpy arrays"""
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    ci = np.array([i for r in rows for i, _ in r], np.int32)
    rt = np.array([lab for r in rows for _, lab in r], np.uint8)
    return rp, ci, rt


def brute_pairs(rows, users, num_items, A, targets, unit_s, unit_q, unit_tag, B):
    """igmc_elicit_pairs from the header, one position and one trial row at a time: (positions, trial rows) with
    positions a list of (links_u, links_v, pair_id, tag, sess) and trial rows a list of (user, [(item, label)])"""
    shared = not isinstance(targets[0], (list, tuple))
    W = len(targets) if shared else len(targets[0])
    U = A * W
    G = B // U
    pos = []
    for i in range(B):
        if i < G * U:
            g, a, w = i // U, (i % U) // W, i % U % W
        else:
            g, a, w = 0, 0, None                                 # padding: unit 0, answer 0
        s, q = unit_s[g], unit_q[g]
        t = -1 if w is None else (targets[w] if shared else targets[s][w])
        u = users[s]
        v = t if t >= 0 else q
        pos.append((u, v, u * num_items + v, unit_tag[g] if t >= 0 else -1, g * A + a))
    trial = []
    for g in range(G):
        for a in range(A):
            s, q = unit_s[g], unit_q[g]
            trial.append((users[s], sorted(rows[s] + [(q, a)])))
    return pos, trial


def _random_rows(rng, S, num_items, deg_max, A):
    rows = []
    for s in range(S):
        d = int(rng.integers(0, deg_max + 1))
        items = np.sort(rng.choice(num_items, d, replace=False))
        rows.append([(int(i), int(rng.integers(0, A))) for i in items])
    return rows


def _unrated(rng, rows, S, num_items, n):
    us, uq = [], []
    while len(us) < n:
        s, q = int(rng.integers(0, S)), int(rng.integers(0, num_items))
        if q not in [i for i, _ in rows[s]]:
            us.append(s)
            uq.append(q)
    return us, uq


def pair_cases():
    """valid cases: dicts of rows, users, num_items, A, targets (a list, or a list of per-session rows), unit_s,
    unit_q, unit_tag and B.  They reach insertion at a row's start, middle and end and into an empty (new-user) row,
    tail padding, a tail unit of the stream (tag -1), empty target slots, duplicate and rated targets, G = 1 with
    U = B, A = 13, and more than one chunk of k_el_pairs' loops"""
    cases = []
    rows = [[(2, 0), (5, 3), (9, 1)], [], [(0, 4)]]
    cases.append(dict(name="map", rows=rows, users=[0, 500, 7], num_items=12, A=5, targets=[1, 5, 11],
                      unit_s=[0, 0, 0, 1, 2], unit_q=[0, 7, 10, 4, 1], unit_tag=[10, 11, 12, 13, 14], B=80))
    cases.append(dict(name="per-session rows", rows=rows, users=[3, 4, 500], num_items=12, A=2,
                      targets=[[3, -1, 4], [-1, -1, 6], [1, 1, -1]], unit_s=[2, 1, 0], unit_q=[5, 0, 11],
                      unit_tag=[0, 1, -1], B=20))
    cases.append(dict(name="G=1 U=B", rows=rows, users=[0, 1, 2], num_items=12, A=5, targets=[0, 2, 2, 9],
                      unit_s=[1], unit_q=[3], unit_tag=[7], B=20))
    rng = np.random.default_rng(3)
    rows = _random_rows(rng, 7, 300, 40, 5)
    us, uq = _unrated(rng, rows, 7, 300, 550)
    cases.append(dict(name="chunks", rows=rows, users=list(range(100, 107)), num_items=300, A=2, targets=[17],
                      unit_s=us, unit_q=uq, unit_tag=list(range(550)), B=1101))
    rows = _random_rows(rng, 4, 50, 12, 13)
    us, uq = _unrated(rng, rows, 4, 50, 3)
    cases.append(dict(name="A=13", rows=rows, users=[9, 8, 7, 6], num_items=50, A=13,
                      targets=[[1, 2], [3, -1], [4, 4], [5, 6]], unit_s=us, unit_q=uq, unit_tag=[2, 1, 0], B=64))
    return cases


# ---- igmc_elicit_stats ----------------------------------------------------------------------------------------------
def brute_stats(preds, K, B, A, W, tag):
    """igmc_elicit_stats from the header: per unit (impact, [answer_mean], tag) with impact / means as Python floats
    rounded to fp32, or None for a unit without real slots"""
    x = []
    for i in range(B):                                      # the fp32 checkpoint mean, summed in checkpoint order
        a = f32(float(preds[0][i]))
        for k in range(1, K):
            a = f32(a + float(preds[k][i]))
        x.append(f32(a / K) if K > 1 else a)
    U = A * W
    out = []
    for g in range(B // U):
        slots = [w for w in range(W) if tag[g * U + w] >= 0]
        if not slots:
            out.append(None)
            continue
        vals = {(a, w): x[g * U + a * W + w] for a in range(A) for w in slots}
        total = 0.0
        for w in slots:
            col = [vals[(a, w)] for a in range(A)]
            total = total + (max(col) - min(col))
        bad = any(v != v for v in vals.values())
        impact = float("nan") if bad else f32(total / len(slots))
        means = []
        for a in range(A):
            m = 0.0
            for w in slots:
                m = m + vals[(a, w)]
            means.append(f32(m / len(slots)))
        out.append((impact, means, tag[g * U + slots[0]]))
    return out


def stats_cases():
    """dicts of preds [K][B], K, B, A, W and tag [B].  They reach a mean an fp32 sum would round, NaN in one answer,
    +inf, inf - inf, +inf and -inf in one answer, a NaN in an empty slot, three checkpoints, units without real
    slots, G = 1 with U = B, and more units than one k_el_stats CTA"""
    cases = []
    # ranges 1, 2^-24, 2^-24: the fp64 sum is 1 + 2^-23 (its mean rounds to another fp32 than an fp32 sum's)
    A, W, B = 2, 3, 13
    p = [0.0] * B
    p[0:3] = [1.0, 2.0 ** -24, 2.0 ** -24]
    p[6:9] = [1.0, 2.0 ** -25, 2.0 ** -25]                  # unit 1 on the same values, halved
    p[3:6] = [0.0, 0.0, 0.0]
    tag = [4] * 6 + [9] * 6 + [-1]
    cases.append(dict(name="fp64 sum", preds=[p], K=1, B=B, A=A, W=W, tag=tag))
    # NaN in one answer, infinities, an empty slot holding NaN that must be ignored
    inf, nan = float("inf"), float("nan")
    A, W = 3, 2
    p = [0.5, nan, 1.0, -2.0, 0.25, 7.0,                     # unit 0: slot 1 is empty (tag -1)
         1.0, 2.0, nan, 3.0, 4.0, 5.0,                      # unit 1: a NaN in answer 1
         inf, 1.0, 0.0, 2.0, 1.0, 3.0,                      # unit 2: +inf in one answer: range inf
         inf, inf, inf, inf, inf, inf,                      # unit 3: inf - inf
         inf, -inf, -inf, 1.0, 0.0, 2.0]                    # unit 4: +inf and -inf in one answer's targets
    tag = [0, -1, 0, -1, 0, -1] + [1] * 6 + [2] * 6 + [3] * 6 + [4] * 6
    cases.append(dict(name="nan and inf", preds=[p], K=1, B=30, A=A, W=W, tag=tag))
    rng = np.random.default_rng(7)
    A, W, B = 5, 4, 300
    p = rng.normal(3, 1, (3, B)).astype(np.float32).tolist()
    tag = [(i // (A * W)) if (i % (A * W)) % W != 3 else -1 for i in range(B)]
    tag = [t if t < 14 else -1 for t in tag]                # units 14 (no real slots): padding
    cases.append(dict(name="K=3", preds=p, K=3, B=B, A=A, W=W, tag=tag))
    A, W, B = 5, 52, 260
    p = rng.normal(0, 1, (1, B)).astype(np.float32).tolist()
    cases.append(dict(name="G=1 U=B", preds=p, K=1, B=B, A=A, W=W, tag=[0] * B))
    A, W, B = 1, 1, 300
    p = rng.normal(0, 1, (1, B)).astype(np.float32).tolist()
    cases.append(dict(name="A=1 many units", preds=p, K=1, B=B, A=A, W=W, tag=list(range(B))))
    return cases
