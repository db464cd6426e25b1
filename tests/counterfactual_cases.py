"""Cases for the counterfactual kernels (csrc/counterfactual.cu), and their brute-force enumerations.

The references are written from the contracts in include/igmc_b200.h in plain Python, not taken from the host twins in
igmc_b200/recommend.py:
  igmc_counterfactual_pairs   position p of [cursor, cursor + B): trial p >> 1 of the last query q with offsets[q] <=
                              p >> 1 (a linear scan), side p & 1; positions past 2T repeat the last one with tag -1; the
                              trial row is sorted(set(range(deg)) - R - {candidate}), the candidate (step > 0) the c-th
                              entry of sorted(set(range(deg)) - R); ids outside G give the pair (0, 0)
  igmc_counterfactual_select  the trial chosen is a Python min over the key (not flipped, margin is NaN, margin, item),
                              flipped meaning ranks_before(s(u, Y), Y, s(u, X), X) restated from csrc/topk_merge.cuh
                              and the margin the fp32 difference s(u, X) - s(u, Y)
Every case claims the regimes it is built to reach; ``REGIMES[kernel](case)`` re-derives them from the case's data
alone, so a case that silently stops reaching one fails."""
import functools
import math

import numpy as np

PAIR_THREADS = 512     # csrc/counterfactual.cu: one chunk of k_cf_pairs' scan
ROW_THREADS = 256      # csrc/counterfactual.cu: one stride of a k_cf_rows row
SELECT_THREADS = 256   # csrc/counterfactual.cu: one stride of k_cf_select's trials, and its reduction tree
CONSTANTS = {("counterfactual.cu", "PAIR_THREADS"): PAIR_THREADS, ("counterfactual.cu", "ROW_THREADS"): ROW_THREADS,
             ("counterfactual.cu", "SELECT_THREADS"): SELECT_THREADS}

ERR_CANDIDATES = 7     # IGMC_ERR_CANDIDATES (csrc/common.cuh)
CF_MAX = 256           # IGMC_COUNTERFACTUAL_MAX
S32, SF = -9, -7.5     # the sentinels the select state starts from where the kernel must not write

# ---- the rating graph: users by degree ------------------------------------------------------------------------------
NI = 5000
DEGREES = (0, 1, 2, 3, 10, 40, 257, 600, 5, 300)
U0, U1, U2, U3, U10, U40, U257, U600 = range(8)
NU = len(DEGREES)


@functools.lru_cache(None)
def graph():
    """(row_ptr int32 [NU + 1], col_idx int32, rating uint8): ascending distinct items per row"""
    rng = np.random.default_rng(31)
    rows = [np.sort(rng.choice(NI, d, replace=False)) for d in DEGREES]
    row_ptr = np.concatenate([[0], np.cumsum(DEGREES)]).astype(np.int32)
    col = np.concatenate(rows).astype(np.int32)
    return row_ptr, col, rng.integers(0, 5, len(col)).astype(np.uint8)


def deg(u):
    rp = graph()[0]
    return int(rp[u + 1] - rp[u])


def free_positions(u, R):
    return sorted(set(range(deg(u))) - set(int(r) for r in R))


def offsets_of(count):
    off = [0]
    for c in count:
        off.append(off[-1] + int(c))
    return np.asarray(off, np.int64)


def _queries(spec, M, step):
    """spec: (user, X, Y, R, count or None = deg - |R| at step > 0, 1 at step 0)"""
    Q = len(spec)
    users = np.asarray([s[0] for s in spec], np.int64)
    items = np.asarray([s[1] for s in spec], np.int64)
    rivals = np.asarray([s[2] for s in spec], np.int64)
    size = np.asarray([len(s[3]) for s in spec], np.int32)
    removed = np.full((Q, M), S32, np.int32)
    count = []
    for q, (u, _, _, R, n) in enumerate(spec):
        removed[q, :len(R)] = sorted(R)
        count.append(n if n is not None else (1 if step == 0 else deg(u) - len(R)))
    return dict(users=users, items=items, rivals=rivals, size=size, removed=removed, M=M, step=step,
                offsets=offsets_of(count))


# ---- igmc_counterfactual_pairs ----------------------------------------------------------------------------------------
R255 = sorted({1, 3, 597} | set(np.random.default_rng(5).choice(np.arange(4, 597), 252, replace=False).tolist()))
WALK = [(U600, 11, 12, R255, None), (U40, 13, 14, [], 0), (U257, 15, 16, [128], None), (U10, 17, 18, [], None)]
STEP0 = [(U0, 1, 2, [], None), (U600, 3, 4, [], None), (U40, 5, 6, [], 0), (U257, 7, 8, [], None),
         (U3, 9, 10, [], None)]
WALK_CLAIMS = {"step>0", "across_query", "past_2T", "zero_trial_between", "deg=257", "deg=600", "R=0", "R=1",
               "R=255", "cand_first", "cand_last", "cand_next_to_removed"}


def pairs_cases():
    cases = []
    for B in (513, 512, 511):
        cases.append(dict(kernel="cf_pairs", name="walk B=%d" % B, B=B, cursors=[0, B, 2 * B], row_cap=None,
                          claims=WALK_CLAIMS | {"B=%d" % B} | ({"chunks>1"} if B > PAIR_THREADS else set()),
                          **_queries(WALK, CF_MAX, 1)))
    cases[0]["cursors"].append(689)
    cases[0]["claims"].add("cursor_odd")
    cases.append(dict(kernel="cf_pairs", name="B=1 step>0", B=1, cursors=[0, 1, 689, 690, 1221, 1222], row_cap=None,
                      claims={"B=1", "step>0", "cursor_odd", "past_2T", "R=255", "R=1", "cand_first", "deg=600",
                              "deg=257"}, **_queries(WALK, CF_MAX, 1)))
    cases.append(dict(kernel="cf_pairs", name="step 0 B>2T exact cap", B=64, cursors=[0], row_cap="exact",
                      claims={"step=0", "B>2T", "past_2T", "deg=0", "deg=600", "deg=257", "zero_trial_between",
                              "row_cap=total", "R=0"}, **_queries(STEP0, 4, 0)))
    cases.append(dict(kernel="cf_pairs", name="row_cap one short", B=64, cursors=[0], row_cap="short",
                      claims={"step=0", "row_cap=total-1"}, **_queries(STEP0, 4, 0)))
    cases.append(dict(kernel="cf_pairs", name="invalid ids", B=16, cursors=[0], row_cap=None,
                      claims={"step=0", "invalid_id"},
                      **_queries([(U10, 1, 2, [], None), (NU, 3, 4, [], None), (U10, 5, -1, [], None),
                                  (U3, NI, 6, [], None), (U40, 7, 8, [], None)], 4, 0)))
    cases.append(dict(kernel="cf_pairs", name="candidate past the row", B=128, cursors=[0], row_cap=None,
                      claims={"step>0", "cand_past_row"},
                      **_queries([(U40, 1, 2, [0], None), (U10, 3, 4, [2, 5], 9)], 4, 1)))
    return cases


def owner(offsets, trial):
    """the last q with offsets[q] <= trial, by a linear scan"""
    q = 0
    for j in range(len(offsets) - 1):
        if offsets[j] <= trial:
            q = j
    return q


def pairs_slots(case, pos):
    """per slot of the batch at ``pos``: dict(p, real, q, u, v, cand, bad, past) by the contract"""
    rp = graph()[0]
    off = case["offsets"]
    P2 = 2 * int(off[-1])
    out = []
    for i in range(case["B"]):
        p = pos + i
        real = p < P2
        p = p if real else P2 - 1
        trial = p >> 1
        q = owner(off, trial)
        u, v = int(case["users"][q]), int(case["rivals"][q] if p & 1 else case["items"][q])
        bad = not (0 <= u < NU and 0 <= v < NI)
        R = case["removed"][q, :case["size"][q]].tolist()
        cand, past = None, False
        if not bad and case["step"] > 0:
            free = free_positions(u, R)
            c = trial - int(off[q])
            past = c >= len(free)
            cand = None if past else free[c]
        out.append(dict(p=p, real=real, q=q, u=0 if bad else u, v=0 if bad else v, cand=cand, bad=bad, past=past,
                        R=R))
    return out


def pairs_reference(case, pos, row_cap=None):
    """(u, v, pair_id, tag, row_users [B], row_ptr [B + 1], row_col, row_rating, err, rows_defined); rows_defined is
    False where the contract leaves the rows open (ids outside G, a candidate past the row)"""
    rp, col, rat = graph()
    slots = pairs_slots(case, pos)
    u = np.asarray([s["u"] for s in slots], np.int64)
    v = np.asarray([s["v"] for s in slots], np.int64)
    tag = np.asarray([s["p"] if s["real"] else -1 for s in slots], np.int64)
    cols, rats, lens = [], [], []
    for s in slots:
        keep = set(free_positions(s["u"], s["R"])) - {s["cand"]}
        k = sorted(keep)
        cols += [int(col[rp[s["u"]] + x]) for x in k]
        rats += [int(rat[rp[s["u"]] + x]) for x in k]
        lens.append(len(k))
    row_ptr = offsets_of(lens).astype(np.int32)
    bad = any(s["bad"] for s in slots)
    past = any(s["past"] for s in slots)
    err = ERR_CANDIDATES if bad or past or (row_cap is not None and int(row_ptr[-1]) > row_cap) else 0
    return (u, v, u * NI + v, tag, u.astype(np.int32), row_ptr, np.asarray(cols, np.int32), np.asarray(rats, np.uint8),
            err, not (bad or past))


def row_cap_of(case, pos):
    total = int(pairs_reference(case, pos)[5][-1])
    if case["row_cap"] == "exact":
        return total
    if case["row_cap"] == "short":
        return total - 1
    return case["B"] * max(DEGREES)


def pairs_regimes(case):
    B, off = case["B"], case["offsets"]
    P2 = 2 * int(off[-1])
    counts = np.diff(off)
    got = {"step=0" if case["step"] == 0 else "step>0"}
    if B in (1, 511, 512, 513):
        got.add("B=%d" % B)
    if B > P2:
        got.add("B>2T")
    if B > PAIR_THREADS:
        got.add("chunks>1")
    nz = np.flatnonzero(counts > 0)
    if len(nz) and any(counts[q] == 0 for q in range(nz[0] + 1, nz[-1])):
        got.add("zero_trial_between")
    for pos in case["cursors"]:
        if pos % 2 and pos < P2:
            got.add("cursor_odd")
        slots = pairs_slots(case, pos)
        if len({s["q"] for s in slots if s["real"]}) > 1:
            got.add("across_query")
        if any(not s["real"] for s in slots):
            got.add("past_2T")
        for s in slots:
            if s["bad"]:
                got.add("invalid_id")
            if s["past"]:
                got.add("cand_past_row")
            if not s["real"] or s["bad"]:
                continue
            d = deg(s["u"])
            if d in (0, 257, 600):
                got.add("deg=%d" % d)
            if len(s["R"]) in (0, 1, 255):
                got.add("R=%d" % len(s["R"]))
            c = s["cand"]
            if c is not None:
                if c == 0:
                    got.add("cand_first")
                if c == d - 1:
                    got.add("cand_last")
                if c - 1 in s["R"] or c + 1 in s["R"]:
                    got.add("cand_next_to_removed")
        ref = pairs_reference(case, pos)
        total = int(ref[5][-1])
        if case["row_cap"] == "exact" and ref[8] == 0:
            got.add("row_cap=total")
        if case["row_cap"] == "short" and total > 0:
            got.add("row_cap=total-1")
    return got


# ---- igmc_counterfactual_select ---------------------------------------------------------------------------------------
def ranks_before(a_s, a_i, b_s, b_i):
    """csrc/topk_merge.cuh ranks_before at sign 1: score descending, NaN after every number (NaNs by id), id ascending"""
    an, bn = math.isnan(a_s), math.isnan(b_s)
    if an or bn:
        return a_i < b_i if (an and bn) else bn
    return a_s > b_s or (a_s == b_s and a_i < b_i)


def _select_case(name, spec, M, step, scores_of, claims):
    c = dict(kernel="cf_select", name=name, claims=claims, **_queries(spec, M, step))
    T = int(c["offsets"][-1])
    sc = np.zeros(2 * T, np.float32)
    for q in range(len(spec)):
        o, n = int(c["offsets"][q]), int(c["offsets"][q + 1] - c["offsets"][q])
        if n:
            sx, sy = scores_of(q, n)
            sc[2 * o:2 * (o + n):2], sc[2 * o + 1:2 * (o + n):2] = sx, sy
    c["scores"] = sc
    return c


def _few(seed):
    rng = np.random.default_rng(seed)
    vals = np.float32([0.25, 0.5, 0.5, 1.0, 1.5])
    return lambda q, n: (rng.choice(vals, n), rng.choice(vals, n))


def _flip_at(u, R, at):
    """no trial flips (X = 1 < Y = 2, s(X) = 1 > s(Y) = 0) except the one removing row position ``at``"""
    free = free_positions(u, R)

    def scores(q, n):
        sx, sy = np.ones(n, np.float32), np.zeros(n, np.float32)
        c = free.index(at[q])
        sx[c], sy[c] = 0.0, 1.0
        return sx, sy
    return scores


def select_cases():
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    cases = [
        _select_case("trial counts", [(U2, 1, 2, [0], None), (U257, 3, 4, [3, 100], None), (U40, 5, 6, [], 0),
                                      (U257, 7, 8, [200], None), (U257, 9, 10, [], None), (U600, 11, 12, [], None),
                                      (U600, 13, 14, R255, None)], CF_MAX, 1, _few(1),
                     {"n=1", "n=255", "n=256", "n=257", "n=600", "no_trials", "several_flips", "equal_margin_item_tie"}),
    ]

    def ties(q, n):
        if q == 0:   # X < Y, s(X) >= s(Y): no flip; the least margins +0 and -0, decided by item
            sx, sy = np.full(n, 1.0, np.float32), np.full(n, 0.5, np.float32)
            sx[[3, 9, 20]], sy[[3, 9, 20]] = np.float32([0.5, -0.0, 0.0]), np.float32([0.5, 0.0, -0.0])
            return sx, sy
        sx, sy = np.full(n, 1.0, np.float32), np.full(n, 0.5, np.float32)   # flips, two at the least margin
        sx[[1, 4, 6]], sy[[1, 4, 6]] = np.float32([0.0, 0.25, 0.25]), np.float32([1.0, 1.5, 1.5])
        return sx, sy
    cases.append(_select_case("flips, equal and signed-zero margins", [(U40, 1, 2, [2, 7], None),
                                                                       (U10, 5, 6, [], None)], 8, 1, ties,
                              {"several_flips", "equal_margin_item_tie", "signed_zero_tie"}))

    def nans(q, n):
        if q == 0:   # NaN margins among numbers: the numbers first
            sx = np.where(np.arange(n) % 3 == 0, nan, np.float32(2.0)).astype(np.float32)
            return sx, np.full(n, 1.0, np.float32)
        if q == 1:   # inf - inf is NaN; one finite margin beats it
            sx, sy = np.full(n, inf, np.float32), np.full(n, inf, np.float32)
            sx[n - 1], sy[n - 1] = 3.0, 1.0
            return sx, sy
        return np.full(n, nan, np.float32), np.full(n, nan, np.float32)    # all NaN: by item
    cases.append(_select_case("NaN margins", [(U10, 1, 2, [], None), (U40, 3, 4, [0], None),
                                              (U257, 5, 6, [], None)], 8, 1, nans,
                              {"nan_margin", "inf-inf", "all_nan"}))

    def item_tie(q, n):   # X = 9 > Y = 2: equal scores put Y first, so the trial with s(X) == s(Y) alone flips
        sx, sy = np.full(n, 2.0, np.float32), np.full(n, 1.0, np.float32)
        sx[4], sy[4] = 1.25, 1.25
        return sx, sy
    cases.append(_select_case("flip by the item tie-break", [(U40, 9, 2, [], None)], 8, 1, item_tie,
                              {"flip_by_item"}))
    def no_flip(q, n):   # X < Y and s(X) > s(Y): no trial flips
        return np.linspace(1.0, 2.0, n).astype(np.float32), np.zeros(n, np.float32)
    cases.append(_select_case("stops", [(U10, 1, 2, [1, 4, 8], None), (U3, 3, 4, [0, 2], None)], 4, 1,
                              no_flip, {"stop_M", "stop_deg"}))

    def base(q, n):
        return [(np.float32([1.0]), np.float32([2.0])), (np.float32([2.0]), np.float32([1.0])),
                (np.float32([1.0]), np.float32([1.0])), (np.float32([1.0]), np.float32([1.0])),
                (np.float32([nan]), np.float32([1.0]))][q]
    cases.append(_select_case("step 0", [(U10, 1, 2, [], None), (U40, 3, 4, [], None), (U257, 9, 5, [], None),
                                         (U600, 5, 9, [], None), (U3, 6, 7, [], None), (U2, 1, 2, [], 0)],
                              4, 0, base, {"step=0 found", "step=0 not_found", "no_trials"}))
    cases.append(_select_case("insert positions", [(U40, 1, 2, [10, 20], None), (U40, 3, 4, [10, 20], None),
                                                   (U40, 5, 6, [10, 20], None)], 8, 1,
                              _flip_at(U40, [10, 20], [5, 15, 30]),
                              {"insert_before", "insert_between", "insert_after"}))
    cases.append(_select_case("not the plan's trials", [(U40, 1, 2, [3], 36), (U10, 3, 4, [0, 1, 2, 3], None),
                                                        (NU, 5, 6, [], 5), (U257, 7, 8, [], None)], 4, 1, _few(3),
                              {"error_n", "error_t>=M", "error_id"}))
    return cases


def select_reference(case):
    """(state, err): the select state (removed, size, count, found, items, ratings, score, rival_score) after the
    pass, starting from the sentinels, by the contract"""
    rp, col, rat = graph()
    Q, M, step = len(case["users"]), case["M"], case["step"]
    st = dict(removed=case["removed"].copy(), size=case["size"].copy(), count=np.full(Q, S32, np.int32),
              found=np.full(Q, 0xAB, np.uint8), items=np.full((Q, M), S32, np.int32),
              ratings=np.full((Q, M), S32, np.int32), score=np.full((Q, M + 1), SF, np.float32),
              rival_score=np.full((Q, M + 1), SF, np.float32))
    off, sc, err = case["offsets"], case["scores"], 0
    info = []
    for q in range(Q):
        o, n = int(off[q]), int(off[q + 1] - off[q])
        u, X, Y = int(case["users"][q]), int(case["items"][q]), int(case["rivals"][q])
        bad = not (0 <= u < NU and 0 <= X < NI and 0 <= Y < NI)
        t = int(case["size"][q])
        d = 0 if bad else deg(u)
        if n <= 0 or bad or (step > 0 and (t >= M or n != d - t)):
            if n > 0:
                err = ERR_CANDIDATES
            st["count"][q] = 0
            info.append(None)
            continue
        if step == 0:
            sx, sy = float(sc[2 * o]), float(sc[2 * o + 1])
            st["score"][q, 0], st["rival_score"][q, 0] = sx, sy
            behind = ranks_before(sy, Y, sx, X)
            st["found"][q] = behind
            st["count"][q] = 0 if behind else d
            info.append(dict(behind=behind))
            continue
        R = case["removed"][q, :t].tolist()
        free = free_positions(u, R)
        trials = []
        for c in range(n):
            sx, sy = sc[2 * (o + c)], sc[2 * (o + c) + 1]
            with np.errstate(invalid="ignore"):
                m = float(np.float32(sx) - np.float32(sy))
            flip = ranks_before(float(sy), Y, float(sx), X)
            trials.append(((not flip, math.isnan(m), 0.0 if math.isnan(m) else m, int(col[rp[u] + free[c]])), c,
                           flip, m, float(sx), float(sy)))
        key, c, flip, m, sx, sy = min(trials)
        pos = free[c]
        st["removed"][q, :t + 1] = sorted(R + [pos])
        st["items"][q, t], st["ratings"][q, t] = int(col[rp[u] + pos]), int(rat[rp[u] + pos])
        st["score"][q, t + 1], st["rival_score"][q, t + 1] = sx, sy
        st["size"][q], st["found"][q] = t + 1, flip
        st["count"][q] = 0 if (flip or t + 1 == M or d == t + 1) else d - t - 1
        info.append(dict(trials=trials, best=(key, c, flip, m, sx, sy), R=R, pos=pos, t=t, deg=d))
    return st, err, info


def select_regimes(case):
    _, _, info = select_reference(case)
    got = set()
    off, M = case["offsets"], case["M"]
    for q, inf in enumerate(info):
        n = int(off[q + 1] - off[q])
        if n == 0:
            got.add("no_trials")
        if inf is None:
            if n > 0:
                u, t = int(case["users"][q]), int(case["size"][q])
                if not 0 <= u < NU:
                    got.add("error_id")
                elif t >= M:
                    got.add("error_t>=M")
                else:
                    got.add("error_n")
            continue
        if "behind" in inf:
            got.add("step=0 found" if inf["behind"] else "step=0 not_found")
            continue
        if n in (1, 255, 256, 257, 600):
            got.add("n=%d" % n)
        trials, (key, c, flip, m, sx, sy) = inf["trials"], inf["best"]
        if sum(tr[2] for tr in trials) >= 2:
            got.add("several_flips")
        same = [tr for tr in trials if tr[0][:3] == key[:3]]
        if len(same) > 1:
            got.add("equal_margin_item_tie")
            zs = {math.copysign(1.0, tr[3]) for tr in same if tr[3] == 0.0}
            if zs == {1.0, -1.0}:
                got.add("signed_zero_tie")
        nans = [math.isnan(tr[3]) for tr in trials]
        if any(nans) and not all(nans):
            got.add("nan_margin")
        if all(nans):
            got.add("all_nan")
        if any(math.isinf(tr[4]) and tr[4] == tr[5] for tr in trials):
            got.add("inf-inf")
        if flip and sx == sy:
            got.add("flip_by_item")
        t, R, pos = inf["t"], inf["R"], inf["pos"]
        if not flip and t + 1 == M:
            got.add("stop_M")
        if not flip and inf["deg"] == t + 1 and t + 1 < M:
            got.add("stop_deg")
        if R and pos < R[0]:
            got.add("insert_before")
        if R and pos > R[-1]:
            got.add("insert_after")
        if len(R) >= 2 and R[0] < pos < R[-1]:
            got.add("insert_between")
    return got


# ---- all cases ----------------------------------------------------------------------------------------------------------
REQUIRED = {
    "cf_pairs": {"B=1", "B=511", "B=512", "B=513", "B>2T", "chunks>1", "cursor_odd", "across_query", "past_2T",
                 "step=0", "step>0", "zero_trial_between", "deg=0", "deg=257", "deg=600", "R=0", "R=1", "R=255",
                 "cand_first", "cand_last", "cand_next_to_removed", "row_cap=total", "row_cap=total-1",
                 "invalid_id", "cand_past_row"},
    "cf_select": {"step=0 found", "step=0 not_found", "n=1", "n=255", "n=256", "n=257", "n=600", "several_flips",
                  "equal_margin_item_tie", "signed_zero_tie", "nan_margin", "inf-inf", "all_nan", "flip_by_item",
                  "stop_M", "stop_deg", "error_n", "error_t>=M", "error_id", "insert_before", "insert_between",
                  "insert_after", "no_trials"},
}

REGIMES = {"cf_pairs": pairs_regimes, "cf_select": select_regimes}


@functools.lru_cache(None)
def all_cases():
    return tuple(pairs_cases() + select_cases())
