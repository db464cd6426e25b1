"""Cases for the online fine-tuning kernels (csrc/online.cu), and their brute-force enumerations.

The references are written from the contracts in include/igmc_b200.h in plain Python, not taken from the host twins in
igmc_b200/train_eval.py:
  igmc_online_draw           slot j: key = sample_state(seeds[0], j, 0, 7); a window pair when W > 0 and key >> 32 <
                             recent_thresh, looked up in its user's row by a linear scan; otherwise position p = (h *
                             nnz) >> 64 of the graph, its user the row that holds p (a linear scan over row_ptr)
  igmc_online_recent_append  the entries with 0 < value <= 256 and ids >= 0 written one by one, in input order, at slot
                             (total + rank) % capacity; a negative id or a value outside 0..256 sets the error word
splitmix64 and sample_state are the Python-integer restatements of tests/draw_cases.py.  Every case claims the regimes
it is built to reach; ``REGIMES[kernel](case)`` re-derives them from the case's data alone."""
import functools

import numpy as np

from tests.draw_cases import M64, sample_state, splitmix64

DRAW_THREADS = 128     # csrc/online.cu: slots per k_online_draw block
APPEND_THREADS = 1024  # csrc/online.cu: one chunk of k_online_append's scans
DRAW_HOP_TAG = 7       # csrc/online.cu: sample_state's hop slot of the draw
CONSTANTS = {("online.cu", "DRAW_THREADS"): DRAW_THREADS, ("online.cu", "APPEND_THREADS"): APPEND_THREADS,
             ("online.cu", "DRAW_HOP_TAG"): DRAW_HOP_TAG}

ERR_GRAPH_UPDATE, ERR_ONLINE = 8, 10   # csrc/common.cuh
RING_SENT = -5                         # ring slots no append has written


# ---- the rating graph: empty rows at the start, in the middle and at the end -------------------------------------------
NI = 2 ** 29 + 3       # users >= 4 have pair ids past 2^31
ROWS = ([], [7, 2 ** 29 + 2, 40], [], [], [0, 5, 9, 2 ** 20, 2 ** 29], [11], [3, 4], [], [])
NU = len(ROWS)


@functools.lru_cache(None)
def graph(empty=False):
    """(row_ptr int32, col_idx int32, rating uint8, num_users, num_items); ``empty``: the same users without ratings"""
    rows = [[] for _ in ROWS] if empty else ROWS
    row_ptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    col = np.asarray([c for r in rows for c in sorted(r)], np.int32)
    rating = (np.arange(len(col)) % 5 + 1).astype(np.uint8)
    return row_ptr, col, rating, NU, NI


# ---- igmc_online_draw -------------------------------------------------------------------------------------------------
# window entries: (user, item, the label it was appended with)
PRESENT = [(1, 7, 1), (4, 9, 3), (4, 2 ** 29, 5), (6, 3, 1)]
CHANGED = [(4, 0, 5), (1, 40, 1)]            # G now holds another label
DELETED = [(2, 7, 3), (5, 12, 2)]           # valid ids, not in G
OUTSIDE = [(NU, 7, 1), (1, NI, 2), (-1, 3, 1), (0, -4, 2)]


def _ring(entries, cap, total):
    """the ring after ``total`` appends that end with ``entries`` (W = min(total, cap) of them)"""
    W = min(total, cap)
    ring = np.full((3, cap), RING_SENT, np.int64)
    for k in range(W):
        ring[:, (total - W + k) % cap] = entries[k % len(entries)]
    return ring


def _draw_case(name, B, ring, total, thresh, step, ahead, claims, empty=False, ss=17, ds=0x1234ABCD):
    return dict(kernel="online_draw", name=name, B=B, ring=ring, capacity=ring.shape[1], total=total, thresh=thresh,
                step_count=step, step_ahead=ahead, sample_seed=ss, drop_seed=ds, empty=empty, claims=claims)


def draw_cases():
    mixed = PRESENT + CHANGED + DELETED + OUTSIDE
    cases = [
        _draw_case("every position B=1000", 1000, _ring(PRESENT, 8, 0), 0, 2 ** 31, 5, 0,
                   {"B=1000", "every_position", "W=0", "empty_first", "empty_mid", "empty_last", "ahead=0",
                    "pid>2^31"}),
        _draw_case("B=1 whole window", 1, _ring(PRESENT, 8, 3), 3, 2 ** 32, 0, 1,
                   {"B=1", "W<cap", "thresh=2^32", "ahead=1", "window_present"}),
        _draw_case("B=128 wrapped ring near 2^63", 128, _ring(mixed, 8, 21), 21, 2 ** 31, 2 ** 63 - 1, 1,
                   {"B=128", "wrapped", "thresh=2^31", "step~2^63", "ahead=1", "window_present", "window_changed",
                    "window_deleted", "pid>2^31"}),
        _draw_case("B=129 capacity 1", 129, _ring([(4, 5, 2)], 1, 5), 5, 2 ** 32, 77, 0,
                   {"B=129", "cap=1", "wrapped", "thresh=2^32", "window_changed"}),
        _draw_case("B=1000 window of 40", 1000, _ring(mixed, 64, 40), 40, 2 ** 31, 9, 1,
                   {"B=1000", "W<cap", "thresh=2^31", "window_present", "window_changed", "window_deleted",
                    "window_outside", "every_position"}),
        _draw_case("thresh 0", 129, _ring(PRESENT, 8, 9), 9, 0, 3, 0, {"B=129", "thresh=0", "wrapped"}),
        _draw_case("no ratings", 129, _ring(PRESENT, 8, 8), 8, 2 ** 31, 3, 1, {"nnz=0", "B=129"}, empty=True),
    ]
    # a threshold equal to slot 5's key high word: that slot draws from the graph, the threshold being exclusive
    c = _draw_case("thresh = a key's high word", 128, _ring(PRESENT, 8, 6), 6, 0, 11, 1, {"B=128", "thresh=key_hi"})
    c["thresh"] = keys(c, 0)[5] >> 32
    cases.append(c)
    return cases


def step_seeds(case):
    """seeds [3] of step s = step_count + step_ahead (mod 2^64)"""
    s = (case["step_count"] + case["step_ahead"]) & M64
    return [splitmix64((case["sample_seed"] + s) & M64), splitmix64((case["drop_seed"] + s) & M64),
            splitmix64((case["drop_seed"] + s + 1) & M64)]


def keys(case, rnd):
    seed = step_seeds(case)[0]
    return [sample_state(seed, j, rnd, DRAW_HOP_TAG) for j in range(case["B"])]


def draw_reference(case):
    """(u, v, label, pair_id [B] int64, seeds [3] uint64, err, slots) with slots[j] = (source, position) by the
    contract: source "window" (found in G), "missed" (a window pair G does not hold), "graph" or "none" (no ratings)"""
    row_ptr, col, rat, nu, ni = graph(case["empty"])
    B, W = case["B"], min(case["total"], case["capacity"])
    nnz = int(row_ptr[nu])
    seeds = step_seeds(case)
    out = np.zeros((4, B), np.int64)
    if nnz <= 0:
        return out[0], out[1], out[2], out[3], np.asarray(seeds, np.uint64), ERR_ONLINE, [("none", -1)] * B
    k0, k1 = keys(case, 0), keys(case, 1)
    slots = []
    for j in range(B):
        pos, src = -1, "graph"
        if W > 0 and (k0[j] >> 32) < case["thresh"]:
            e = ((k0[j] & 0xFFFFFFFF) * W) >> 32
            u, v = int(case["ring"][0, e]), int(case["ring"][1, e])
            src = "missed"
            if 0 <= u < nu and 0 <= v < ni:
                for p in range(int(row_ptr[u]), int(row_ptr[u + 1])):
                    if col[p] == v:
                        pos, src = p, "window"
            slots.append((src, e))
        if pos < 0:
            pos = (k1[j] * nnz) >> 64
            u = max(x for x in range(nu) if row_ptr[x] <= pos < row_ptr[x + 1])
            v = int(col[pos])
            if src == "graph":
                slots.append(("graph", pos))
        out[:, j] = (u, v, int(rat[pos]), u * ni + v)
    return out[0], out[1], out[2], out[3], np.asarray(seeds, np.uint64), 0, slots


def draw_regimes(case):
    row_ptr, col, rat, nu, ni = graph(case["empty"])
    B, cap, total = case["B"], case["capacity"], case["total"]
    W = min(total, cap)
    got = set()
    if B in (1, 128, 129, 1000):
        got.add("B=%d" % B)
    deg = np.diff(row_ptr)
    if int(row_ptr[-1]) == 0:
        got.add("nnz=0")
    else:
        if deg[0] == 0:
            got.add("empty_first")
        if deg[-1] == 0:
            got.add("empty_last")
        if any(deg[x] == 0 for x in range(1, nu - 1)):
            got.add("empty_mid")
    got.add("W=0" if W == 0 else ("W<cap" if W < cap else "wrapped" if total > cap else "W=cap"))
    if cap == 1:
        got.add("cap=1")
    if case["thresh"] in (0, 2 ** 31, 2 ** 32):
        got.add("thresh=%s" % {0: "0", 2 ** 31: "2^31", 2 ** 32: "2^32"}[case["thresh"]])
    got.add("ahead=%d" % case["step_ahead"])
    if case["step_count"] >= 2 ** 62:
        got.add("step~2^63")
    if int(row_ptr[-1]) == 0:
        return got
    if W > 0 and any((k >> 32) == case["thresh"] for k in keys(case, 0)):
        got.add("thresh=key_hi")
    u, v, lab, pid, _, _, slots = draw_reference(case)
    if (pid > 2 ** 31).any():
        got.add("pid>2^31")
    drawn = {p for s, p in slots if s == "graph"}
    if drawn == set(range(int(row_ptr[-1]))):
        got.add("every_position")
    for j, (src, e) in enumerate(slots):
        if src == "missed":
            a, b = int(case["ring"][0, e]), int(case["ring"][1, e])
            got.add("window_deleted" if 0 <= a < nu and 0 <= b < ni else "window_outside")
        elif src == "window":
            got.add("window_changed" if lab[j] != case["ring"][2, e] else "window_present")
    return got


# ---- igmc_online_recent_append -----------------------------------------------------------------------------------------
def _delta(D, rng, deletes=0.0, invalid=0.0):
    u = rng.integers(0, 2 ** 31 - 1, D)
    v = rng.integers(0, 2 ** 31 - 1, D)
    x = rng.integers(1, 257, D)
    x[rng.random(D) < deletes] = 0
    bad = np.flatnonzero(rng.random(D) < invalid)
    for k, i in enumerate(bad):
        if k % 4 == 0:
            u[i] = -1 - k
        elif k % 4 == 1:
            v[i] = -3
        elif k % 4 == 2:
            x[i] = 257
        else:
            x[i] = -2
    return np.stack([u, v, x]).astype(np.int64)


def append_cases():
    rng = np.random.default_rng(61)
    spec = [  # (name, capacity, total before, [(D, deletes, invalid)], claims)
        ("D=0", 16, 3, [(0, 0, 0)], {"D=0"}),
        ("D=1 capacity 1", 1, 0, [(1, 0, 0)], {"D=1", "cap=1", "kept=cap"}),
        ("D=1023 deletes", 2000, 7, [(1023, 0.2, 0)], {"D=1023", "kept<cap", "deletes"}),
        ("D=1024 kept = capacity", 1024, 100, [(1024, 0, 0)], {"D=1024", "kept=cap"}),
        ("D=1025 past 2^31", 64, 2 ** 31 + 5, [(1025, 0.1, 0.05)], {"D=1025", "kept>cap", "deletes", "invalid",
                                                                    "total>2^31"}),
        ("D=5000", 777, 3 * 2 ** 31 + 1, [(5000, 0.3, 0.02)], {"D=5000", "kept>cap", "deletes", "invalid",
                                                               "total>2^31"}),
        ("calls wrap the ring", 100, 0, [(60, 0.1, 0), (70, 0, 0), (30, 0.5, 0.1), (250, 0.2, 0)],
         {"wraps", "kept<cap", "kept>cap", "deletes", "invalid"}),
    ]
    cases = []
    for name, cap, total, calls, claims in spec:
        cases.append(dict(kernel="append", name=name, capacity=cap, total=total, claims=claims,
                          calls=[_delta(D, rng, dl, inv) for D, dl, inv in calls]))
    return cases


def append_reference(case):
    """per call (ring_u, ring_v, total, err): the rated entries written one at a time, in input order"""
    ring = np.full((2, case["capacity"]), RING_SENT, np.int64)
    total, out = case["total"], []
    for u, v, x in case["calls"]:
        ring = ring.copy()
        err = 0
        for i in range(len(u)):
            if u[i] < 0 or v[i] < 0 or x[i] < 0 or x[i] > 256:
                err = ERR_GRAPH_UPDATE
                continue
            if x[i] == 0:
                continue
            ring[:, total % case["capacity"]] = (u[i], v[i])
            total += 1
        out.append((ring[0], ring[1], total, err))
    return out


def append_regimes(case):
    cap = case["capacity"]
    got = set()
    total = case["total"]
    if total > 2 ** 31:
        got.add("total>2^31")
    if cap == 1:
        got.add("cap=1")
    for u, v, x in case["calls"]:
        D = len(u)
        if D in (0, 1, 1023, 1024, 1025, 5000):
            got.add("D=%d" % D)
        ok = (u >= 0) & (v >= 0) & (x >= 0) & (x <= 256)
        kept = int((ok & (x > 0)).sum())
        if D:
            got.add("kept<cap" if kept < cap else "kept=cap" if kept == cap else "kept>cap")
        if (ok & (x == 0)).any():
            got.add("deletes")
        if (~ok).any():
            got.add("invalid")
        if len(case["calls"]) > 1 and total // cap != (total + kept) // cap and total % cap:
            got.add("wraps")
        total += kept
    return got


# ---- all cases ----------------------------------------------------------------------------------------------------------
REQUIRED = {
    "online_draw": {"B=1", "B=128", "B=129", "B=1000", "nnz=0", "empty_first", "empty_mid", "empty_last",
                    "every_position", "W=0", "W<cap", "wrapped", "cap=1", "thresh=0", "thresh=2^31", "thresh=2^32",
                    "thresh=key_hi", "window_present", "window_changed", "window_deleted", "window_outside",
                    "ahead=0", "ahead=1", "step~2^63", "pid>2^31"},
    "append": {"D=0", "D=1", "D=1023", "D=1024", "D=1025", "D=5000", "kept<cap", "kept=cap", "kept>cap", "deletes",
               "invalid", "total>2^31", "wraps", "cap=1"},
}

REGIMES = {"online_draw": draw_regimes, "append": append_regimes}


@functools.lru_cache(None)
def all_cases():
    return tuple(draw_cases() + append_cases())
