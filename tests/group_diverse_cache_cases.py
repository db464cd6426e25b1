"""Cases for the group (csrc/groups.cu), diversity (csrc/diverse.cu) and cached-list (csrc/recommend_cache.cu) kernels,
and their brute-force enumerations.

The references are written in plain Python from the contracts in include/igmc_b200.h, not taken from the host twins in
igmc_b200/recommend.py:
  igmc_group_rows       per group the union of its members' rows as a Python set; summed degrees (Python ints) beyond
                        cap drop every group from the first one that does not fit
  igmc_group_pairs      position by position: unit i // width, member slot i % width, the padding as unit 0, slot 0
  igmc_group_stats      mean = a Python-float sum in member order, one division, rounded to fp32 with struct; min / max
                        a first-strict scan; NaN when any member's x is
  igmc_item_union       a Python set of the valid ids
  igmc_cocount          c_ab = |col(a) & col(b)| by set intersection over the rows
  igmc_item_cosine      c / math.sqrt(da * db) in Python floats, rounded once to fp32
  igmc_diverse_select   the greedy loop with np.float32 products then differences and ranks_before's order
  igmc_diverse_ws_bytes the largest chunk whose bytes_of fits the bound, by a linear scan
  igmc_rescore_plan     the header's set formula per slot
  igmc_cache_invalidate / igmc_cache_settle  slot by slot
Every case claims the regimes it is built to reach; ``REGIMES[kernel](case)`` re-derives them from the case's data
alone, so a case that silently stops reaching one fails.  The launch constants those regimes depend on are restated
below and checked against the sources."""
import functools
import math
import struct

import numpy as np

from tests.ranking_cases import ckpt_mean

ROW_THREADS = 256     # csrc/groups.cu: one chunk of k_gr_offsets' group scan and of a group's entry scan
PAIR_THREADS = 256    # csrc/groups.cu: positions per k_gr_pairs block
STATS_THREADS = 128   # csrc/groups.cu: units per k_gr_stats block
SCAN_THREADS = 256    # csrc/diverse.cu: one chunk of k_dv_scan = 256 bitmap words = 8 192 items
COUNT_TILE = 1024     # csrc/diverse.cu: row entries per k_dv_count tile
SELECT_THREADS = 256  # csrc/diverse.cu: pool entries per k_dv_select CTA (8 warps); IGMC_TOPK_MAX there
MARK_THREADS = 256    # csrc/recommend_cache.cu: one stride of a k_rp_mark / k_rp_write row's words
RP_SCAN_THREADS = 1024  # csrc/recommend_cache.cu: SCAN_THREADS, one chunk of k_rp_scan / k_cache_settle / k_rp_candmask
SLOT_THREADS = 256    # csrc/recommend_cache.cu: slots per k_cache_invalidate block
CONSTANTS = {("groups.cu", "ROW_THREADS"): ROW_THREADS, ("groups.cu", "PAIR_THREADS"): PAIR_THREADS,
             ("groups.cu", "STATS_THREADS"): STATS_THREADS, ("diverse.cu", "SCAN_THREADS"): SCAN_THREADS,
             ("diverse.cu", "COUNT_TILE"): COUNT_TILE, ("recommend_cache.cu", "MARK_THREADS"): MARK_THREADS,
             ("recommend_cache.cu", "SCAN_THREADS"): RP_SCAN_THREADS,
             ("recommend_cache.cu", "SLOT_THREADS"): SLOT_THREADS, ("diverse.cu", "SELECT_THREADS"): SELECT_THREADS}
COUNT_GRID = 65535    # csrc/diverse.cu: k_dv_count's grid is min(num_users, 65535): a grid-stride loop past it

FLT_MAX = float(np.finfo(np.float32).max)
SUB = float(np.float32(1e-45))          # the least positive subnormal
BIG_DEG = 2 ** 25 + 1                   # 64 copies of a row this long sum past 2^31 - 1
DIVERSE_WS_DEFAULT = 256 << 20
ERR = 7                                 # IGMC_ERR_CANDIDATES


def f32(x):
    """x rounded to fp32, as a Python float"""
    return struct.unpack("f", struct.pack("f", x))[0]


def csr(rows):
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    ci = np.concatenate([np.asarray(r, np.int64) for r in rows] + [np.zeros(0, np.int64)])
    return rp.astype(np.int32), ci.astype(np.int32)


def columns(rp, ci, num_items):
    """col_ptr [num_items+1] and row_idx of the CSR rows (rows ascending within a column)"""
    rp, ci = np.asarray(rp, np.int64), np.asarray(ci, np.int64)
    u = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    o = np.lexsort((u, ci))
    cp = np.concatenate([[0], np.cumsum(np.bincount(ci, minlength=num_items))]).astype(np.int32)
    return cp, u[o].astype(np.int32)


def col_sets(rp, ci, items):
    """{item: set of the users who rated it} for the given items"""
    want = set(int(v) for v in items)
    out = {v: set() for v in want}
    rp = np.asarray(rp, np.int64)
    for u in range(len(rp) - 1):
        for v in ci[rp[u]:rp[u + 1]].tolist():
            if v in want:
                out[v].add(u)
    return out


def ranks_before(av, ai, bv, bi):
    """ranks_before (csrc/topk_merge.cuh) with sign +1: value descending, id ascending, NaN after every number, empty
    ids (< 0) last"""
    if ai < 0:
        return False
    if bi < 0:
        return True
    an, bn = math.isnan(av), math.isnan(bv)
    if an or bn:
        return ai < bi if (an and bn) else bn
    return av > bv or (av == bv and ai < bi)


# ======================================================================================================================
# groups.cu
# ======================================================================================================================
GROUP_NU, GROUP_NI = 40, 3000


@functools.lru_cache(None)
def group_graph():
    """40 users over 3 000 items: user 3 rated 700, user 5 300, user 7 nothing"""
    rng = np.random.default_rng(20)
    rows = [np.sort(rng.choice(GROUP_NI, int(rng.integers(0, 41)), replace=False)) for _ in range(GROUP_NU)]
    rows[3] = np.sort(rng.choice(GROUP_NI, 700, replace=False))
    rows[5] = np.sort(rng.choice(GROUP_NI, 300, replace=False))
    rows[7] = np.zeros(0, np.int64)
    return csr(rows)


@functools.lru_cache(None)
def big_degree_graph():
    """user 0 rated BIG_DEG items (64 copies of it sum to 2^31 + 64), users 1 and 2 a handful"""
    rows = [np.arange(BIG_DEG), np.array([3, 9, 12, 40, BIG_DEG - 1]), np.array([1, 9, 77, 500, 501, 502, 600])]
    return csr(rows)


def _members(rng, G, M, dup=True):
    out = np.full((G, M), -1, np.int32)
    for g in range(G):
        n = int(rng.integers(1, M + 1))
        out[g, :n] = rng.choice(GROUP_NU, n, replace=dup)
    return out


def _degree_sums(rp, members, num_users):
    d = np.diff(np.asarray(rp, np.int64))
    return [sum(int(d[m]) for m in row if 0 <= m < num_users) for row in np.asarray(members, np.int64)]


def group_rows_cases():
    rp, _ = group_graph()
    rng = np.random.default_rng(21)
    cases = []

    def add(name, members, cap, claims):
        cases.append(dict(kernel="group_rows", name=name, graph="groups", num_users=GROUP_NU, rp=rp,
                          members=np.asarray(members, np.int32), cap=cap, claims=claims))

    need = lambda m: sum(_degree_sums(rp, m, GROUP_NU))   # noqa: E731
    m = np.array([[3]], np.int32)
    add("G=1 M=1", m, need(m), {"G=1", "M=1", "union>256", "cap=need"})
    m = _members(rng, 256, 7)
    m[1] = [-1, 4, 5, 6, -1, -1, -1]                          # empty slots first, mid and last
    m[2] = [2, -1, 6, 6, 3, -1, -1]
    m[3] = [3, 5, 9, 9, 3, 1, 2]                              # every slot, duplicated members
    add("G=256 M=7", m, need(m), {"G=256", "M=7", "dup_member", "empty_first", "empty_mid", "empty_last", "union>256",
                                  "cap=need"})
    m = _members(rng, 257, 64)
    m[0] = [3] * 64                                           # one member 64 times
    m[1, :] = -1
    m[1, 40] = 5
    add("G=257 M=64", m, need(m), {"G=257", "M=64", "dup_member", "empty_first", "empty_last", "union>256",
                                   "cap=need"})
    m = _members(rng, 600, 7)
    m[599] = [5, 3, -1, -1, -1, -1, -1]
    add("G=600 cap=need-1", m, need(m) - 1, {"G=600", "M=7", "cap=need-1", "overflow_last"})
    m = np.array([[3, 5, -1], [1, 2, 4], [8, -1, -1], [0, 0, 6], [7, -1, -1]], np.int32)
    add("overflow first", m, int(_degree_sums(rp, m, GROUP_NU)[0]) - 1, {"overflow_first", "cap<need-1"})
    m = np.array([[1, 2, -1], [4, 6, 8], [3, -1, -1], [9, 10, 11], [5, 1, -1], [12, -1, -1]], np.int32)
    s = _degree_sums(rp, m, GROUP_NU)
    add("overflow mid", m, sum(s[:2]) + s[2] - 1, {"overflow_mid", "cap<need-1"})
    add("zero cap", np.array([[7, -1], [3, 5]], np.int32), 0, {"overflow_last", "cap<need-1"})
    m = np.array([[0, 2], [3, 99], [5, -3], [GROUP_NU, -1], [6, 1]], np.int32)
    add("bad member ids", m, need(np.where((m < -1) | (m >= GROUP_NU), -1, m)), {"bad_member", "cap=need"})
    big = np.full((3, 64), -1, np.int32)
    big[0, :2] = [1, 2]
    big[1, :] = 0                                             # 64 * (2^25 + 1) entries: past 2^31 - 1
    big[2, :3] = [2, 1, 2]
    cases.append(dict(kernel="group_rows", name="degree sum past 2^31", graph="big", num_users=3,
                      rp=big_degree_graph()[0], members=big, cap=4096, claims={"deg_sum>=2^31", "M=64",
                                                                               "overflow_mid"}))
    big1 = np.zeros((1, 64), np.int32)
    cases.append(dict(kernel="group_rows", name="one group past 2^31", graph="big", num_users=3,
                      rp=big_degree_graph()[0], members=big1, cap=4096,
                      claims={"deg_sum>=2^31", "M=64", "overflow_first", "G=1"}))
    return cases


def graph_of(case):
    return big_degree_graph() if case["graph"] == "big" else group_graph()


def group_rows_reference(case, rp=None, ci=None):
    """(row_ptr [G+1], col_idx, err): kept groups' unions as sorted Python sets"""
    if rp is None:
        rp, ci = graph_of(case)
    rp = np.asarray(rp, np.int64)
    nu, cap = case["num_users"], case["cap"]
    members = [[int(x) for x in row] for row in case["members"]]
    err = 0
    n, total = [], 0
    for row in members:
        s = 0
        for m in row:
            if m < -1 or m >= nu:
                err = ERR
            elif m >= 0:
                s += int(rp[m + 1] - rp[m])
        n.append(s)
    out_rp, out_ci, before = [0], [], 0
    for g, row in enumerate(members):
        union = set()
        if before + n[g] <= cap:
            for m in row:
                if 0 <= m < nu:
                    union |= set(ci[rp[m]:rp[m + 1]].tolist())
        before += n[g]
        out_ci += sorted(union)
        out_rp.append(len(out_ci))
    if before > cap:
        err = ERR
    return np.asarray(out_rp, np.int64), np.asarray(out_ci, np.int64), err


def group_rows_regimes(case):
    members, cap, nu = np.asarray(case["members"], np.int64), case["cap"], case["num_users"]
    G, M = members.shape
    got = {"G=%d" % G, "M=%d" % M}
    n = _degree_sums(case["rp"], members, nu)
    for row in members:
        real = [j for j in range(M) if 0 <= row[j] < nu]
        v = [int(row[j]) for j in real]
        if len(set(v)) < len(v):
            got.add("dup_member")
        if real and row[0] == -1:
            got.add("empty_first")
        if real and any(row[j] == -1 and j < max(real) for j in range(1, M - 1)):
            got.add("empty_mid")
        if real and row[M - 1] == -1:
            got.add("empty_last")
        if ((row < -1) | (row >= nu)).any():
            got.add("bad_member")
    need, before, first = sum(n), 0, None
    for g in range(G):
        if before + n[g] <= cap and n[g] > ROW_THREADS:
            got.add("union>256")
        if first is None and before + n[g] > cap:
            first = g
        before += n[g]
    if max(n) >= 2 ** 31:
        got.add("deg_sum>=2^31")
    got.add("cap=need" if cap == need else "cap=need-1" if cap == need - 1 else "cap<need-1" if cap < need else "")
    if first is not None:
        last = max(g for g in range(G) if n[g] > 0)
        got.add("overflow_first" if first == 0 else "overflow_last" if first == last else "overflow_mid")
    return got - {""}


# ---- igmc_group_pairs ---------------------------------------------------------------------------------------------------
def group_pairs_cases():
    rng = np.random.default_rng(22)
    NU, NI = 6, 500_000_000                                   # pair ids past 2^31
    spec = [  # (name, M, B, invalid, claims)
        ("B=M=7", 7, 7, None, {"B=M", "M=7"}),
        ("M=7 B=255", 7, 255, None, {"M=7", "B=255", "B%M!=0", "lead_empty", "pid>=2^31", "tag=-1"}),
        ("M=64 B=256", 64, 256, None, {"M=64", "B=256", "lead_empty"}),
        ("M=7 B=257", 7, 257, None, {"M=7", "B=257", "B%M!=0", "pid>=2^31"}),
        ("M=1 B=513", 1, 513, None, {"M=1", "B=513", "pid>=2^31", "tag=-1"}),
        ("M=64 B=513", 64, 513, None, {"M=64", "B=513", "B%M!=0", "lead_empty"}),
        ("bad group", 7, 257, "group", {"bad_group"}),
        ("bad item", 7, 257, "item", {"bad_item"}),
        ("bad member", 7, 257, "member", {"bad_member"}),
    ]
    cases = []
    for name, M, B, bad, claims in spec:
        G = 5
        members = np.full((G, M), -1, np.int32)
        for g in range(G):
            k = int(rng.integers(1, M + 1))
            members[g, :k] = rng.integers(0, NU, k)
        members[1, 0] = -1                                    # a group whose first slot is empty
        if M > 2:
            members[1, 1:3] = [-1, 4]
            members[1, 3:] = -1
        Gu = B // M
        ug = rng.integers(0, G, Gu).astype(np.int32)
        ug[Gu // 2] = 1
        uv = rng.integers(0, NI, Gu).astype(np.int32)
        ut = rng.permutation(Gu).astype(np.int64)
        if "tag=-1" in claims:
            ut[-1] = -1
        if bad == "group":
            ug[Gu // 3] = G
        elif bad == "item":
            uv[0] = NI
        elif bad == "member":
            members[ug[0], M - 1] = NU
        cases.append(dict(kernel="group_pairs", name=name, members=members, num_users=NU, num_items=NI, unit_g=ug,
                          unit_v=uv, unit_tag=ut, B=B, invalid=bad is not None, claims=claims))
    # B = width: one unit of 64 slots, the first empty
    m = np.full((2, 64), -1, np.int32)
    m[0, 5], m[0, 63], m[1, :3] = 2, 4, [1, 2, 3]
    cases.append(dict(kernel="group_pairs", name="B=M=64", members=m, num_users=NU, num_items=NI,
                      unit_g=np.array([0], np.int32), unit_v=np.array([NI - 1], np.int32),
                      unit_tag=np.array([3], np.int64), B=64, invalid=False, claims={"B=M", "M=64", "lead_empty",
                                                                                   "pid>=2^31"}))
    return cases


def group_pairs_reference(case):
    """(links_u, links_v, pair_id, tag) [B] and err, one position at a time"""
    members, M = case["members"], case["members"].shape[1]
    G, NU, NI, B = len(members), case["num_users"], case["num_items"], case["B"]
    Gu = B // M
    out, err = [[], [], [], []], 0
    for i in range(B):
        real = i < Gu * M
        u0, j = (i // M, i % M) if real else (0, 0)
        g, v = int(case["unit_g"][u0]), int(case["unit_v"][u0])
        if not (0 <= g < G and 0 <= v < NI):
            err, g, v = ERR, 0, 0
        m = int(members[g][j])
        if m < -1 or m >= NU:
            err, m = ERR, -1
        lead = int(members[g][0])
        lead = lead if 0 <= lead < NU else -1
        u = m if m >= 0 else (lead if lead >= 0 else 0)
        for r, x in enumerate((u, v, u * NI + v, int(case["unit_tag"][u0]) if real and m >= 0 else -1)):
            out[r].append(x)
    return [np.asarray(x, np.int64) for x in out], err


def group_pairs_regimes(case):
    members, B = np.asarray(case["members"], np.int64), case["B"]
    G, M = members.shape
    Gu = B // M
    got = {"M=%d" % M}
    if B == M:
        got.add("B=M")
    if B in (255, 256, 257, 513):
        got.add("B=%d" % B)
    if B % M:
        got.add("B%M!=0")
    ug, uv = np.asarray(case["unit_g"][:Gu], np.int64), np.asarray(case["unit_v"][:Gu], np.int64)
    if ((ug < 0) | (ug >= G)).any():
        got.add("bad_group")
    if ((uv < 0) | (uv >= case["num_items"])).any():
        got.add("bad_item")
    okg = ug[(ug >= 0) & (ug < G)]
    if ((members[okg] < -1) | (members[okg] >= case["num_users"])).any():
        got.add("bad_member")
    if (members[okg, 0] == -1).any():
        got.add("lead_empty")
    if (np.asarray(case["unit_tag"][:Gu]) < 0).any():
        got.add("tag=-1")
    if (members.max() * case["num_items"] + uv.max()) >= 2 ** 31:
        got.add("pid>=2^31")
    return got


# ---- igmc_group_stats ---------------------------------------------------------------------------------------------------
def _stats_case(name, K, Gu, M, pad, rng, specials, claims):
    B = Gu * M + pad
    x = np.round(rng.normal(3, 1, (K, B)) * 8) / 8                # ties
    preds = x.astype(np.float32)
    tag = np.full(B, -1, np.int64)
    for u in range(Gu):
        n = int(rng.integers(0, M + 1)) if u % 5 else M
        slots = sorted(rng.choice(M, n, replace=False).tolist())
        tag[[u * M + j for j in slots]] = u
    for u, vals in specials:                                   # unit u's members take the values as given (K = 1)
        tag[u * M:(u + 1) * M] = -1
        for j, v in enumerate(vals):
            if v is not None:
                preds[:, u * M + j] = v
                tag[u * M + j] = u
    return dict(kernel="group_stats", name=name, preds=preds, K=K, B=B, M=M, tag=tag, claims=claims)


def group_stats_cases():
    rng = np.random.default_rng(23)
    nan, inf = float("nan"), float("inf")
    cases = [_stats_case("Gu=127 M=1 K=1", 1, 127, 1, 0, rng, [(3, [0.0]), (4, [-0.0]), (5, [None])],
                         {"Gu=127", "M=1", "K=1", "x:-0", "no_real"}),
             _stats_case("Gu=128 M=7 K=3", 3, 128, 7, 3, rng, [], {"Gu=128", "M=7", "K=3", "padding"}),
             _stats_case("Gu=129 M=7 K=7", 7, 129, 7, 6, rng, [], {"Gu=129", "Gu>128", "M=7", "K=7", "padding",
                                                                    "fp32_sum_differs"})]
    specials = [
        (0, [FLT_MAX] * 64),                                    # 64 x FLT_MAX: an fp32 sum would overflow
        (1, [1e8, 1.0, -1e8]),                                  # cancellation: an fp32 sum gives 0
        (2, [1.0, 2.0 ** -24, 2.0 ** -24]),                     # an fp32 sum rounds the small terms away
        (3, [0.0, -0.0, 0.0]), (4, [-0.0, 0.0]),                # signed zeros: the first is kept by min / max
        (5, [2.0, nan, 1.0]), (6, [inf, 1.0, -2.0]), (7, [-inf, 3.0]), (8, [inf, -inf]),
        (9, [SUB, 3 * SUB, -SUB]), (10, [SUB, None, SUB, None]),  # subnormals
        (11, [None] * 64),                                      # no real position: key 0
        (12, [None, 5.0, None, 5.0, -FLT_MAX, FLT_MAX]),        # empty slots first and between; ties
        (13, [1.5] * 64),
    ]
    cases.append(_stats_case("Gu=300 M=64 K=1 specials", 1, 300, 64, 0, rng, specials,
                             {"Gu=300", "Gu>128", "M=64", "K=1", "x:nan", "x:+inf", "x:-inf", "x:subnormal",
                              "x:FLT_MAX", "x:-0", "64xFLT_MAX", "cancellation", "fp32_sum_differs", "no_real",
                              "signed_zero_tie"}))
    return cases


def group_x(case):
    return ckpt_mean(np.asarray(case["preds"], np.float32).reshape(case["K"], case["B"]))


def group_stats_reference(case, aggregate):
    """per unit (key, [x_j or None], tag) with the key a Python float rounded to fp32 (0.0 for a unit without real
    positions)"""
    x = [float(v) for v in group_x(case)]
    M, B, tag = case["M"], case["B"], case["tag"]
    out = []
    for u in range(B // M):
        real = [j for j in range(M) if tag[u * M + j] >= 0]
        xs = [x[u * M + j] for j in real]
        t = int(tag[u * M + real[-1]]) if real else -1
        if not real:
            k = 0.0
        elif any(v != v for v in xs):
            k = float("nan")
        elif aggregate == "mean":
            s = 0.0
            for v in xs:
                s = s + v
            k = f32(s / len(xs))
        else:
            k = xs[0]
            for v in xs[1:]:
                if (v < k) if aggregate == "min" else (v > k):
                    k = v
        out.append((k, [x[u * M + j] if tag[u * M + j] >= 0 else None for j in range(M)], t))
    return out


def group_stats_regimes(case):
    M, B, K, tag = case["M"], case["B"], case["K"], np.asarray(case["tag"])
    Gu = B // M
    got = {"M=%d" % M, "K=%d" % K, "Gu=%d" % Gu}
    if Gu > STATS_THREADS:
        got.add("Gu>128")
    if B % M:
        got.add("padding")
    x = group_x(case)
    for u in range(Gu):
        real = [j for j in range(M) if tag[u * M + j] >= 0]
        xs = x[[u * M + j for j in real]]
        if not real:
            got.add("no_real")
            continue
        bits = xs.view(np.uint32)
        for name, hit in (("x:nan", np.isnan(xs)), ("x:+inf", xs == np.inf), ("x:-inf", xs == -np.inf),
                          ("x:-0", bits == 0x80000000), ("x:FLT_MAX", np.abs(xs) == FLT_MAX),
                          ("x:subnormal", (xs != 0) & (np.abs(xs) < np.finfo(np.float32).tiny))):
            if hit.any():
                got.add(name)
        if len(real) == 64 and (xs == FLT_MAX).all():
            got.add("64xFLT_MAX")
        if (bits == 0x80000000).any() and (bits == 0).any():
            got.add("signed_zero_tie")
        vals = [float(v) for v in xs]
        if any(vals[i:i + 3] == [f32(1e8), 1.0, -f32(1e8)] for i in range(len(vals))):
            got.add("cancellation")
        if np.isfinite(xs).all():
            s32 = np.float32(0)
            with np.errstate(over="ignore"):
                for v in xs:
                    s32 = np.float32(s32 + v)
            s64 = 0.0
            for v in vals:
                s64 += v
            if np.float32(s32 / np.float32(len(vals))) != f32(s64 / len(vals)):
                got.add("fp32_sum_differs")
    return got


# ======================================================================================================================
# diverse.cu
# ======================================================================================================================
def item_union_cases():
    rng = np.random.default_rng(30)
    cases = []
    for ni, n, claims in ((1, 3, {"ni=1", "repeats"}), (31, 40, {"ni=31", "last_word_partial", "repeats"}),
                          (32, 40, {"ni=32", "repeats"}), (33, 40, {"ni=33", "last_word_partial"}),
                          (8191, 3000, {"ni=8191", "last_word_partial"}), (8192, 3000, {"ni=8192"}),
                          (8193, 3000, {"ni=8193", "bits_past_8192", "last_word_partial"}),
                          (2 ** 20 + 5, 20000, {"ni=2^20+5", "bits_past_8192", "last_word_partial"})):
        items = rng.integers(-1, ni, n).astype(np.int64)
        items[:2] = ni - 1                                    # the last item, twice
        items[2] = 0
        cases.append(dict(kernel="item_union", name="ni=%d" % ni, items=items, num_items=ni, claims=claims))
    cases.append(dict(kernel="item_union", name="n=0", items=np.zeros(0, np.int64), num_items=33, claims={"n=0"}))
    cases.append(dict(kernel="item_union", name="all padding", items=np.full(500, -1, np.int64), num_items=8193,
                      claims={"all_padding"}))
    cases.append(dict(kernel="item_union", name="bad ids", items=np.array([4, -1, 9000, 9, -2, 8500, 4], np.int64),
                      num_items=9000, claims={"bad_id", "bits_past_8192"}))
    return cases


def item_union_reference(case):
    """(map [ni], list, err)"""
    ni = case["num_items"]
    s, err = set(), 0
    for v in case["items"].tolist():
        if v < -1 or v >= ni:
            err = ERR
        elif v >= 0:
            s.add(v)
    lst = sorted(s)
    mp = np.full(ni, -1, np.int64)
    mp[lst] = np.arange(len(lst))
    return mp, np.asarray(lst, np.int64), err


def item_union_regimes(case):
    ni, items = case["num_items"], np.asarray(case["items"], np.int64)
    got = {"ni=2^20+5" if ni == 2 ** 20 + 5 else "ni=%d" % ni}
    ok = items[(items >= 0) & (items < ni)]
    if len(items) == 0:
        got.add("n=0")
    elif (items == -1).all():
        got.add("all_padding")
    if ((items < -1) | (items >= ni)).any():
        got.add("bad_id")
    if (ok >= SCAN_THREADS * 32).any() and (ok < SCAN_THREADS * 32).any():
        got.add("bits_past_8192")
    if ni % 32 and (ok >= ni // 32 * 32).any():
        got.add("last_word_partial")
    if len(np.unique(ok)) < len(ok):
        got.add("repeats")
    return got


# ---- igmc_cocount -------------------------------------------------------------------------------------------------------
COUNT_NU, COUNT_NI = 70000, 4000
LONG_ROWS = {65540: (0, 2048), 66000: (1024, 3072), 67000: (1024, 2047), 68000: (1024, 2048), 69000: (1024, 2049),
             69999: (0, 3073)}                                # user: the items range(lo, hi) it rated


@functools.lru_cache(None)
def count_graph():
    """70 000 users (past the count kernel's 65 535-CTA grid) over 4 000 items, with rows of 1 023 .. 3 073 entries
    among the users the grid-stride loop reaches"""
    rng = np.random.default_rng(31)
    deg = rng.integers(0, 4, COUNT_NU)
    rows = [np.unique(rng.integers(0, COUNT_NI, int(d))) for d in deg]
    for u, (lo, hi) in LONG_ROWS.items():
        rows[u] = np.arange(lo, hi)
    rows[2] = np.arange(1024, 1100)                           # a row below the grid with many union entries
    return csr(rows)


def count_union():
    """items of [1024, 2048) and [3072, 4000) only: rows range(0, 2048) and range(0, 3073) start with an empty tile,
    range(1024, 3072) ends with one"""
    rng = np.random.default_rng(32)
    return np.sort(np.r_[rng.choice(np.arange(1024, 2048), 150, replace=False), 3072,
                         rng.choice(np.arange(3073, 4000), 50, replace=False)])


def cocount_cases():
    u = count_union()
    cases = [dict(kernel="cocount", name="Nu=0", union=np.zeros(0, np.int64), cap=0, claims={"Nu=0"}),
             dict(kernel="cocount", name="Nu=1", union=np.array([1500]), cap=0, claims={"Nu=1"}),
             dict(kernel="cocount", name="Nu=2", union=np.array([1030, 1031]), cap=1, claims={"Nu=2", "users>65535"}),
             dict(kernel="cocount", name="Nu=2 cap=need-1", union=np.array([1030, 1031]), cap=0,
                  claims={"cap=need-1"}),
             dict(kernel="cocount", name="tiles", union=u, cap=len(u) * (len(u) - 1) // 2,
                  claims={"row=1023", "row=1024", "row=1025", "row=2048", "row=3073", "empty_first_tile",
                          "empty_last_tile", "users>65535", "empty_row"}),
             dict(kernel="cocount", name="tiles cap=need-1", union=u, cap=len(u) * (len(u) - 1) // 2 - 1,
                  claims={"cap=need-1"})]
    return cases


def cocount_reference(case):
    """(the upper triangle as a list of counts, return code)"""
    u = [int(x) for x in case["union"]]
    nu = len(u)
    need = nu * (nu - 1) // 2
    if need > case["cap"]:
        return None, -2
    rp, ci = count_graph()
    cols = col_sets(rp, ci, u)
    return [len(cols[u[i]] & cols[u[j]]) for i in range(nu) for j in range(i + 1, nu)], 0


def cocount_regimes(case):
    u = np.asarray(case["union"], np.int64)
    nu = len(u)
    need = nu * (nu - 1) // 2
    got = {"Nu=%d" % nu} if nu < 3 else set()
    if case["cap"] == need - 1:
        got.add("cap=need-1")
    if case["cap"] < need:
        return got
    rp, ci = count_graph()
    inu = np.zeros(COUNT_NI, bool)
    inu[u] = True
    for w in range(len(rp) - 1):
        row = ci[rp[w]:rp[w + 1]]
        hit = inu[row]
        if len(row) == 0:
            got.add("empty_row")
        if hit.sum() < 2:
            continue
        if w >= COUNT_GRID:
            got.add("users>65535")
        if len(row) in (1023, 1024, 1025, 2048, 3073):
            got.add("row=%d" % len(row))
        tiles = [hit[t:t + COUNT_TILE].any() for t in range(0, len(row), COUNT_TILE)]
        if len(tiles) > 1 and not tiles[0]:
            got.add("empty_first_tile")
        if len(tiles) > 1 and not tiles[-1]:
            got.add("empty_last_tile")
    return got


# the Nu >= 65 537 table (8.6 GB): run on the GPU only, when it fits
HUGE_NU = 65537
HUGE_ROWS = [[0, 1, 65535, 65536], [65534, 65536], [2, 65534, 65535, 65536], [1, 2], [65536]]
HUGE_ITEMS = [0, 1, 2, 65534, 65535, 65536, 65536]            # union indices whose int32 t(i, j) would wrap


def huge_reference():
    """{table index: count} of the nonzero entries and the cosine of HUGE_ITEMS"""
    cols = {}
    for w, r in enumerate(HUGE_ROWS):
        for v in r:
            cols.setdefault(v, set()).add(w)
    nz = {}
    for r in HUGE_ROWS:
        for a in range(len(r)):
            for b in range(a + 1, len(r)):
                t = r[a] * (2 * HUGE_NU - r[a] - 1) // 2 + r[b] - r[a] - 1
                nz[t] = nz.get(t, 0) + 1
    cos = [[cosine(len(cols.get(a, set()) & cols.get(b, set())), len(cols.get(a, ())), len(cols.get(b, ())))
            for b in HUGE_ITEMS] for a in HUGE_ITEMS]
    return nz, np.asarray(cos, np.float32)


# ---- igmc_diverse_select / igmc_item_cosine -----------------------------------------------------------------------------
SEL_NU, SEL_NI = 300, 3000


@functools.lru_cache(None)
def select_graph():
    """300 users over 3 000 items; items 2 990.. unrated; users 0-9 rated the same 120 items (heavy co-rating)"""
    rng = np.random.default_rng(33)
    rows = [np.sort(rng.choice(SEL_NI - 10, int(rng.integers(0, 60)), replace=False)) for _ in range(SEL_NU)]
    common = rng.choice(SEL_NI - 10, 120, replace=False)
    for u in range(10):
        rows[u] = np.union1d(rows[u], common)
    return csr(rows)


def cosine(c, da, db):
    if da == 0 or db == 0:
        return 0.0
    return f32(float(c) / math.sqrt(float(da) * float(db)))


def select_cases():
    rng = np.random.default_rng(34)
    rp, ci = select_graph()
    deg = np.bincount(ci, minlength=SEL_NI)
    rated = np.flatnonzero(deg >= 2)
    common = np.intersect1d(ci[rp[0]:rp[1]], ci[rp[1]:rp[2]])
    spec = [  # (name, P, k, penalty, claims)
        ("P=1 k=1", 1, 1, 0.75, {"P=1", "k=1", "k=P"}),
        ("P=31 k=P", 31, 31, 0.0, {"P=31", "k=P", "penalty=0", "padding"}),
        ("P=32 k=1", 32, 1, 1e30, {"P=32", "k=1", "penalty=1e30"}),
        ("P=33 k=P", 33, 33, 1.0, {"P=33", "k=P", "winner_warp>0", "tie_across_warps", "unrated"}),
        ("P=255 k=1", 255, 1, SUB, {"P=255", "k=1", "penalty=subnormal", "winner_warp>0", "tie_across_warps"}),
        ("P=255 k=P", 255, 255, 2.0, {"P=255", "k=P", "winner_warp>0", "tie_across_warps", "score:nan",
                                      "score:+inf", "score:-inf"}),
        ("P=256 k=P", 256, 256, 0.5, {"P=256", "k=P", "tie_across_warps", "winner_warp>0", "padding", "unrated"}),
        ("P=256 k=1 subnormal", 256, 1, SUB, {"P=256", "k=1", "penalty=subnormal"}),
        ("P=33 k=1 1e30", 33, 1, 1e30, {"P=33", "k=1", "penalty=1e30"}),
    ]
    cases = []
    for name, P, k, pen, claims in spec:
        Q = 3
        pi = np.full((Q, P), -1, np.int64)
        ps = np.full((Q, P), -np.inf, np.float32)
        for q in range(Q):
            n = P if q != 1 or "padding" not in claims else max(P - 7, 1)
            src = common if q == 2 and len(common) >= n else rated
            pi[q, :n] = rng.choice(src, n, replace=False)
            ps[q, :n] = np.round(rng.uniform(1, 5, n) * 2) / 2            # exact ties
        if P > 32:
            ps[0, :] = 1.0                                     # every other key equal: the order is the position
            ps[0, min(40, P - 1)], ps[0, P - 1] = 9.0, 9.0     # the winner in warp 1, tied with the last warp's
            ps[1, 5] = 7.0                                     # a tie of warp 0 and the last warp
            ps[1, P - 1 if "padding" not in claims else P - 8] = 7.0
            ps[2, 3], ps[2, 70 % P] = 0.0, -0.0                  # signed zeros
        if "unrated" in claims:
            pi[1, 1] = SEL_NI - 1
        if "score:nan" in claims:
            ps[1, 10], ps[1, 200], ps[2, 0], ps[2, 100], ps[2, 101] = np.nan, np.nan, np.inf, np.inf, -np.inf
        if pen == SUB:
            ps[1, :] = np.where(pi[1] >= 0, 0.0, -np.inf)      # keys -0 and -subnormal
        cases.append(dict(kernel="select", name=name, pool_item=pi, pool_score=ps.astype(np.float32), k=k,
                          penalty=float(np.float32(pen)), claims=claims))
    bad = np.array([[4, 5, 6], [4, SEL_NI, 6], [4, -3, 6], [8, 9, -1]], np.int64)
    cases.append(dict(kernel="select", name="bad pools", pool_item=bad, pool_score=np.ones((4, 3), np.float32), k=2,
                      penalty=1.0, claims={"bad_id", "padding"}))
    return cases


def select_union(case):
    """the union list a run over this case builds (every valid pool item)"""
    it = np.asarray(case["pool_item"], np.int64).reshape(-1)
    return np.unique(it[(it >= 0) & (it < SEL_NI)])


def select_reference(case, union=None, table_of=None):
    """(items [Q, k], scores [Q, k], keys [Q, k], err): the greedy loop with np.float32 fmul then fsub"""
    rp, ci = select_graph()
    deg = np.bincount(ci, minlength=SEL_NI)
    union = select_union(case) if union is None else union
    inu = set(int(x) for x in union)
    cols = col_sets(rp, ci, union)
    pen = np.float32(case["penalty"])
    pi, ps, k = case["pool_item"], case["pool_score"], case["k"]
    Q, P = pi.shape
    oi, os_, ok = np.full((Q, k), -1, np.int64), np.full((Q, k), -np.inf, np.float32), np.full((Q, k), -np.inf,
                                                                                                 np.float32)
    err = 0
    for q in range(Q):
        items = [int(v) for v in pi[q]]
        if any(v < -1 or v >= SEL_NI or (v >= 0 and v not in inu) for v in items):
            err = ERR
            continue
        live = [v >= 0 for v in items]
        m = [np.float32(0)] * P
        for s in range(k):
            keys = [np.float32(ps[q, j] - np.float32(pen * m[j])) for j in range(P)]
            best = -1
            for j in range(P):
                if live[j] and (best < 0 or ranks_before(float(keys[j]), j, float(keys[best]), best)):
                    best = j
            if best < 0:
                break
            c = items[best]
            oi[q, s], os_[q, s], ok[q, s] = c, ps[q, best], keys[best]
            live[best] = False
            for j in range(P):
                if live[j]:
                    v = items[j]
                    cnt = int(deg[v]) if v == c else len(cols[v] & cols[c])
                    sim = np.float32(cosine(cnt, int(deg[v]), int(deg[c])))
                    m[j] = sim if sim > m[j] else m[j]
    return oi, os_, ok, err


def select_regimes(case):
    pi, ps, k, pen = case["pool_item"], case["pool_score"], case["k"], case["penalty"]
    Q, P = pi.shape
    got = set()
    if P in (1, 31, 32, 33, 255, 256):
        got.add("P=%d" % P)
    if k == 1:
        got.add("k=1")
    if k == P:
        got.add("k=P")
    if pen == 0:
        got.add("penalty=0")
    elif pen < np.finfo(np.float32).tiny:
        got.add("penalty=subnormal")
    elif pen >= 1e30:
        got.add("penalty=1e30")
    _, ci = select_graph()
    deg = np.bincount(ci, minlength=SEL_NI)
    for q in range(Q):
        it, sc = pi[q], ps[q]
        if ((it < -1) | (it >= SEL_NI)).any():
            got.add("bad_id")
            continue
        live = it >= 0
        if (~live).any():
            got.add("padding")
        if (live & (deg[np.clip(it, 0, SEL_NI - 1)] == 0)).any():
            got.add("unrated")
        for name, hit in (("score:nan", np.isnan(sc)), ("score:+inf", sc == np.inf), ("score:-inf", sc == -np.inf)):
            if (hit & live).any():
                got.add(name)
        v = np.where(live & ~np.isnan(sc), sc, -np.inf)
        if live.any() and np.isfinite(v.max()) or (v == np.inf).any():
            top = np.flatnonzero(live & (v == v.max()))
            if len(top) and top[0] >= 32:
                got.add("winner_warp>0")
            if len(set(top // 32)) > 1:
                got.add("tie_across_warps")
    return got


def cosine_cases():
    rng = np.random.default_rng(35)
    _, ci = select_graph()
    cases = []
    for Q in (1, 255, 256, 257):
        items = rng.choice(SEL_NI, Q).astype(np.int64)
        if Q > 1:
            items[:3] = [SEL_NI - 1, 5, 5]                     # an unrated item, a repeat
            items[3:13] = np.unique(ci)[:10]
        cases.append(dict(kernel="cosine", name="Q=%d" % Q, items=items, claims={"Q=%d" % Q} |
                          ({"repeats", "unrated"} if Q > 1 else set())))
    return cases


def cosine_reference(case):
    rp, ci = select_graph()
    deg = np.bincount(ci, minlength=SEL_NI)
    items = [int(v) for v in case["items"]]
    cols = col_sets(rp, ci, items)
    return np.asarray([[cosine(len(cols[a] & cols[b]), int(deg[a]), int(deg[b])) for b in items] for a in items],
                      np.float32)


def cosine_regimes(case):
    items = np.asarray(case["items"], np.int64)
    _, ci = select_graph()
    deg = np.bincount(ci, minlength=SEL_NI)
    got = {"Q=%d" % len(items)}
    if len(np.unique(items)) < len(items):
        got.add("repeats")
    if (deg[items] == 0).any():
        got.add("unrated")
    return got


# ---- igmc_diverse_ws_bytes ----------------------------------------------------------------------------------------------
def _bytes_of(users, pool, ni):
    nu = min(users * pool, ni)
    return nu * (nu - 1) // 2 * 4


def ws_cases():
    out = []
    for name, args, claims in (
            ("default bound, fits", (40, 50, 3706, 0), {"default", "all_fit"}),
            ("bound = bytes_of(7)", (40, 50, 100000, _bytes_of(7, 50, 100000)), {"bound=bytes_of(c)"}),
            ("bound = bytes_of(7) - 1", (40, 50, 100000, _bytes_of(7, 50, 100000) - 1), {"bound=bytes_of(c)-1"}),
            ("union capped by num_items", (40, 50, 300, 0), {"default", "all_fit", "capped_by_items"}),
            ("chunked, bound one below", (40, 50, 420, _bytes_of(8, 50, 420) - 1), {"chunked",
                                                                                    "bound=bytes_of(c)-1"}),
            ("below one query", (40, 50, 100000, 100), {"floor_one"}),
            ("default bound, chunked", (4000, 256, 2 ** 20, -5), {"default", "chunked"})):
        out.append(dict(kernel="ws_bytes", name=name, args=args, claims=claims))
    return out


def ws_reference(case):
    """(table_bytes, chunk) by a linear scan over the chunk sizes"""
    q, pool, ni, bound = case["args"]
    cap = bound if bound > 0 else DIVERSE_WS_DEFAULT
    c = q
    while c > 1 and _bytes_of(c, pool, ni) > cap:
        c -= 1
    return _bytes_of(c, pool, ni), c


def ws_regimes(case):
    q, pool, ni, bound = case["args"]
    cap = bound if bound > 0 else DIVERSE_WS_DEFAULT
    got = {"default"} if bound <= 0 else set()
    fits = [c for c in range(1, q + 1) if _bytes_of(c, pool, ni) <= cap]
    c = fits[-1] if fits else 1
    if len(fits) == q:
        got.add("all_fit")
    elif fits:
        got.add("chunked")
        if cap == _bytes_of(c, pool, ni):
            got.add("bound=bytes_of(c)")
        if cap == _bytes_of(c + 1, pool, ni) - 1:
            got.add("bound=bytes_of(c)-1")
    else:
        got.add("floor_one")
    if c * pool > ni:
        got.add("capped_by_items")
    return got


# ======================================================================================================================
# recommend_cache.cu
# ======================================================================================================================
CACHE_NU = 220


@functools.lru_cache(None)
def cache_graph(ni):
    """220 users over ni items; user 11 rated 100 of them (an edit row longer than a warp), user 12 nothing"""
    rng = np.random.default_rng(40 + ni)
    rows = [np.sort(rng.choice(ni, int(rng.integers(0, min(ni, 25))), replace=False)) for _ in range(CACHE_NU)]
    rows[11] = np.sort(rng.choice(ni, min(ni, 100), replace=False))
    rows[12] = np.zeros(0, np.int64)
    return csr(rows)


def plan_ws_bytes(ni, chunk):
    """the workspace bytes that hold exactly `chunk` slots: align256(4 W) + 512 + chunk * (4 W + 8)"""
    W = (ni + 31) // 32
    return (4 * W + 255) // 256 * 256 + 512 + chunk * (4 * W + 8)


def rescore_cases():
    rng = np.random.default_rng(41)
    cases = []

    def add(name, ni, U, chunks, edits, cand, exclude, claims, bad_user=False, out_caps=("total", "total-1")):
        rp, ci = cache_graph(ni)
        users = rng.integers(0, CACHE_NU, U).astype(np.int64)
        users[0] = 11
        if U > 3:
            users[1], users[2] = users[3], 12
        if bad_user:
            users[U // 2] = CACHE_NU
        eu, ev = edits(users, rp, ci, ni)
        cases.append(dict(kernel="rescore", name=name, num_items=ni, users=users, edit_u=np.asarray(eu, np.int64),
                          edit_v=np.asarray(ev, np.int64), cand=cand, exclude=exclude, chunks=chunks,
                          out_caps=out_caps, claims=claims))

    def typical(users, rp, ci, ni, bad=False):
        eu = list(rng.integers(0, CACHE_NU, 6))
        ev = list(rng.integers(0, ni, 6))
        r11 = ci[rp[11]:rp[12]]
        u = int(users[-1])                                     # an edit rated by a slot user through user 11's row
        ru = ci[rp[u]:rp[u + 1]]
        eu += [11, 11]
        ev += [int(ru[0]) if len(ru) else 0, int(r11[0])]
        eu += [eu[0], eu[0]]                                   # duplicated edits
        ev += [ev[0], ev[0]]
        eu.append(int(users[1]))                               # an edit by a slot's own user
        ev.append(1)
        if bad:
            eu += [CACHE_NU, -1, 3]
            ev += [0, 0, 10 ** 6]
        return eu, ev

    add("U=1 chunk=1", 33, 1, (1,), lambda us, rp, ci, ni: ([11, 4], [int(ci[rp[11]]), 2]), None, 1,
        {"U=1", "chunk=U=1", "ni=33", "cand:all", "exclude:1", "edit:own"})
    add("U=3000 ni=32", 32, 3000, (3000, 1, 1025), typical, None, 1,
        {"U=3000", "chunk=1", "chunk=1025", "chunk>1024", "multi_chunk", "ni=32", "cand:all", "edit:own",
         "edit:dup", "exclude:1", "out_cap=total", "out_cap=total-1"})
    cand = np.sort(np.r_[rng.choice(8193, 300, replace=False), 8192, 8192, 5, 5])
    add("U=1100 ni=8193 shared", 8193, 1100, (1100, 1025, 7), typical, cand, 0,
        {"ni=8193", "cand:shared", "cand:dup", "chunk>1024", "chunk=1025", "multi_chunk", "edit:own", "edit:dup",
         "edit_row>32",
         "exclude:0", "out_cap=total", "out_cap=total-1"})
    add("U=40 ni=32769", 32769, 40, (40, 3), typical, None, 1,
        {"ni=32769", "cand:all", "multi_chunk", "edit:own", "edit_row>32", "exclude:1", "out_cap=total",
         "out_cap=total-1"})
    add("U=1025 ni=33 shared", 33, 1025, (1025, 1024), typical, np.array([0, 1, 1, 5, 31, 32, 32]), 1,
        {"ni=33", "cand:shared", "cand:dup", "chunk=1025", "chunk>1024", "multi_chunk", "edit_row>32", "exclude:1"})
    add("bad ids", 33, 50, (50, 7), lambda us, rp, ci, ni: typical(us, rp, ci, ni, bad=True), np.array([0, 2, 40, -1, 9]), 1,
        {"edit:bad", "slot_user:bad", "cand:bad", "multi_chunk"}, bad_user=True)
    return cases


def rescore_reference(case):
    """(user_off [U+1], items, full [U], totals (2), err): per slot the header's set formula"""
    ni = case["num_items"]
    rp, ci = cache_graph(ni)
    rp = np.asarray(rp, np.int64)
    nu = len(rp) - 1
    err = 0
    if case["cand"] is None:
        cands = set(range(ni))
    else:
        cands = set()
        for v in case["cand"].tolist():
            if 0 <= v < ni:
                cands.add(v)
            else:
                err = ERR
    edits = []
    for a, b in zip(case["edit_u"].tolist(), case["edit_v"].tolist()):
        if 0 <= a < nu and 0 <= b < ni:
            edits.append((a, b))
        else:
            err = ERR
    off, items, full, total = [0], [], [], 0
    for u in case["users"].tolist():
        if not 0 <= u < nu:
            err = ERR
            off.append(off[-1])
            full.append(1)
            continue
        row = set(ci[rp[u]:rp[u + 1]].tolist())
        affected = set()
        for a, b in edits:
            if a == u:
                affected = set(range(ni))
                break
            affected.add(b)
            if b in row:
                affected |= set(ci[rp[a]:rp[a + 1]].tolist() if a < nu else [])
        c = cands - row if case["exclude"] else cands
        plan = sorted(affected & c)
        items += plan
        off.append(len(items))
        full.append(int(len(plan) == len(c)))
        total += len(c)
    return (np.asarray(off, np.int64), np.asarray(items, np.int64), np.asarray(full, np.uint8),
            (off[-1], total), err)


def rescore_regimes(case):
    ni, users, U = case["num_items"], case["users"], len(case["users"])
    rp, ci = cache_graph(ni)
    nu = len(rp) - 1
    got = {"ni=%d" % ni, "exclude:%d" % case["exclude"]}
    if U in (1, 3000):
        got.add("U=%d" % U)
    for c in case["chunks"]:
        if c == 1 == U:
            got.add("chunk=U=1")
        elif c == 1:
            got.add("chunk=1")
        if c == 1025:
            got.add("chunk=1025")
        if c > RP_SCAN_THREADS and c <= U:
            got.add("chunk>1024")
        if c < U:
            got.add("multi_chunk")
    cand = case["cand"]
    if cand is None:
        got.add("cand:all")
    else:
        got.add("cand:shared")
        if len(np.unique(cand)) < len(cand):
            got.add("cand:dup")
        if ((cand < 0) | (cand >= ni)).any():
            got.add("cand:bad")
    eu, ev = case["edit_u"], case["edit_v"]
    ok = (eu >= 0) & (eu < nu) & (ev >= 0) & (ev < ni)
    if (~ok).any():
        got.add("edit:bad")
    if ((users < 0) | (users >= nu)).any():
        got.add("slot_user:bad")
    if np.isin(eu[ok], users).any():
        got.add("edit:own")
    pairs = list(zip(eu[ok].tolist(), ev[ok].tolist()))
    if len(set(pairs)) < len(pairs):
        got.add("edit:dup")
    deg = np.diff(np.asarray(rp, np.int64))
    for a, b in pairs:
        if deg[a] > 32 and any(0 <= u < nu and u != a and b in ci[rp[u]:rp[u + 1]] for u in users.tolist()):
            got.add("edit_row>32")
            break
    for oc in case["out_caps"]:
        got.add("out_cap=" + oc)
    return got


# ---- igmc_cache_invalidate / igmc_cache_settle ---------------------------------------------------------------------------
def _lists(rng, U, D, fill_all=False):
    """U lists of D entries: a prefix of distinct items with quantised scores (ties), descending, then padding"""
    top_s, top_i = np.full((U, D), -np.inf, np.float32), np.full((U, D), -1, np.int64)
    for j in range(U):
        n = D if fill_all or j % 3 == 0 else int(rng.integers(0, D + 1))
        items = rng.choice(max(2 * D, 40), n, replace=False)
        sc = np.round(rng.normal(3, 1, n) * 2) / 2
        o = np.lexsort((items, -sc))
        top_s[j, :n], top_i[j, :n] = sc[o], items[o]
    return top_s, top_i


def invalidate_cases():
    rng = np.random.default_rng(50)
    cases = []
    for name, U, D, claims in (("U=300 D=256", 300, 256, {"D=256", "full_prefix", "U>256", "full", "complete",
                                                           "empty_prefix", "rescored_hit"}),
                               ("U=1025 D=10", 1025, 10, {"U>256", "full", "complete", "empty_prefix",
                                                          "rescored_hit", "full_prefix"})):
        top_s, top_i = _lists(rng, U, D, fill_all=D == 256)
        if D == 256:
            top_s[5:9], top_i[5:9] = -np.inf, -1              # a few empty prefixes among the full ones
        resc, full, complete = [], np.zeros(U, np.uint8), np.zeros(U, np.uint8)
        for j in range(U):
            n = int((top_i[j] >= 0).sum())
            pick = rng.choice(top_i[j, :n], min(n, int(rng.integers(0, 4))), replace=False) if n else []
            extra = rng.choice(np.arange(1000, 1100), int(rng.integers(0, 3)), replace=False)
            resc.append(np.unique(np.r_[pick, extra]).astype(np.int64))
            full[j] = j % 11 == 0
            complete[j] = j % 7 == 0
        user_off = np.concatenate([[0], np.cumsum([len(r) for r in resc])]).astype(np.int64)
        cases.append(dict(kernel="invalidate", name=name, top_s=top_s, top_i=top_i, user_off=user_off,
                          resc=np.concatenate(resc).astype(np.int32), full=full, complete=complete, claims=claims))
    return cases


def invalidate_reference(case):
    """(top_s, top_i, thr_s, thr_i), slot by slot"""
    top_s, top_i = case["top_s"].copy(), case["top_i"].copy()
    U, D = top_i.shape
    thr_s, thr_i = np.full(U, -np.inf, np.float32), np.full(U, -1, np.int64)
    for j in range(U):
        n = 0
        while n < D and top_i[j, n] >= 0:
            n += 1
        if case["complete"][j] or case["full"][j]:
            thr_i[j], thr_s[j] = -1, -np.inf
        elif n == 0:
            thr_i[j], thr_s[j] = -2, -np.inf
        else:
            thr_i[j], thr_s[j] = top_i[j, n - 1], top_s[j, n - 1]
        gone = set(case["resc"][case["user_off"][j]:case["user_off"][j + 1]].tolist())
        keep = [] if case["full"][j] else [(top_s[j, e], top_i[j, e]) for e in range(n) if int(top_i[j, e]) not in gone]
        top_s[j], top_i[j] = -np.inf, -1
        for e, (s, i) in enumerate(keep):
            top_s[j, e], top_i[j, e] = s, i
    return top_s, top_i, thr_s, thr_i


def invalidate_regimes(case):
    top_i, full, complete = case["top_i"], case["full"], case["complete"]
    U, D = top_i.shape
    got = {"D=%d" % D} if D == 256 else set()
    if U > SLOT_THREADS:
        got.add("U>256")
    n = (top_i >= 0).sum(1)
    if (n == D).any():
        got.add("full_prefix")
    if full.any():
        got.add("full")
    if complete.any():
        got.add("complete")
    if ((n == 0) & (full == 0) & (complete == 0)).any():
        got.add("empty_prefix")
    for j in range(U):
        if (full[j] == 0) and np.isin(top_i[j, :n[j]], case["resc"][case["user_off"][j]:case["user_off"][j + 1]]).any():
            got.add("rescored_hit")
            break
    return got


def settle_cases():
    rng = np.random.default_rng(51)
    cases = []
    for name, U, D, k, claims in (("U=1024 D=10 k=3", 1024, 10, 3, {"U=1024", "thr=-1", "thr=-2", "tie_before",
                                                                     "tie_after", "redo", "complete", "thr:nan"}),
                                  ("U=1025 D=256 k=256", 1025, 256, 256, {"U=1025", "D=256", "full_prefix", "redo",
                                                                         "thr=-1", "thr=-2"}),
                                  ("U=3000 D=20 k=5", 3000, 20, 5, {"U=3000", "thr=-1", "thr=-2", "tie_before",
                                                                    "tie_after", "redo", "complete", "thr:nan",
                                                                    "nan_entry"})):
        top_s, top_i = _lists(rng, U, D, fill_all=D == 256)
        thr_s, thr_i = np.full(U, -np.inf, np.float32), np.full(U, -1, np.int64)
        for j in range(U):
            n = int((top_i[j] >= 0).sum())
            r = j % 6
            if r == 1:
                thr_i[j] = -2
            elif r >= 2 and n:
                e = int(rng.integers(0, n))
                thr_s[j] = top_s[j, e]                         # a tie with entry e: its id decides
                thr_i[j] = top_i[j, e] + (1 if r == 2 else -1 if r == 3 and top_i[j, e] > 0 else 0)
                if r == 4:
                    thr_s[j] = np.float32(rng.normal(3, 1))
                if r == 5 and j % 12 == 5:
                    thr_s[j] = np.nan                          # a NaN threshold: every number ranks before it
            if j % 50 == 17 and n > 1:
                top_s[j, n - 1] = np.nan                        # a NaN entry at the end of a merged list
        cases.append(dict(kernel="settle", name=name, k=k, top_s=top_s, top_i=top_i, thr_s=thr_s, thr_i=thr_i,
                          claims=claims))
    return cases


def settle_reference(case):
    """(top_s, top_i, complete, redo), slot by slot"""
    top_s, top_i = case["top_s"].copy(), case["top_i"].copy()
    U, D = top_i.shape
    complete, redo = np.zeros(U, np.uint8), []
    for j in range(U):
        ti, ts = int(case["thr_i"][j]), float(case["thr_s"][j])
        d = 0
        if ti != -2:
            while d < D and top_i[j, d] >= 0 and (ti == -1 or not ranks_before(ts, ti, float(top_s[j, d]),
                                                                              int(top_i[j, d]))):
                d += 1
        top_s[j, d:], top_i[j, d:] = -np.inf, -1
        complete[j] = int(ti == -1 and d < D)
        if ti != -1 and d < case["k"]:
            redo.append(j)
    return top_s, top_i, complete, np.asarray(redo, np.int64)


def settle_regimes(case):
    top_s, top_i, thr_s, thr_i = case["top_s"], case["top_i"], case["thr_s"], case["thr_i"]
    U, D = top_i.shape
    got = {"U=%d" % U} if U in (1024, 1025, 3000) else set()
    if D == 256:
        got.add("D=256")
    n = (top_i >= 0).sum(1)
    if (n == D).any():
        got.add("full_prefix")
    if (thr_i == -1).any():
        got.add("thr=-1")
    if (thr_i == -2).any():
        got.add("thr=-2")
    if np.isnan(thr_s[thr_i >= 0]).any():
        got.add("thr:nan")
    if np.isnan(top_s).any():
        got.add("nan_entry")
    _, _, complete, redo = settle_reference(case)
    if len(redo):
        got.add("redo")
    if complete.any():
        got.add("complete")
    for j in np.flatnonzero(thr_i >= 0):
        tie = (top_s[j, :n[j]] == thr_s[j])
        if (tie & (top_i[j, :n[j]] < thr_i[j])).any():
            got.add("tie_before")
        if (tie & (top_i[j, :n[j]] > thr_i[j])).any():
            got.add("tie_after")
    return got


# ---- all cases ----------------------------------------------------------------------------------------------------------
REQUIRED = {
    "group_rows": {"G=1", "G=256", "G=257", "G=600", "M=1", "M=7", "M=64", "dup_member", "empty_first", "empty_mid",
                   "empty_last", "union>256", "cap=need", "cap=need-1", "overflow_first", "overflow_mid",
                   "overflow_last", "bad_member", "deg_sum>=2^31"},
    "group_pairs": {"B=M", "B=255", "B=256", "B=257", "B=513", "B%M!=0", "M=1", "M=7", "M=64", "pid>=2^31",
                    "lead_empty", "tag=-1", "bad_group", "bad_item", "bad_member"},
    "group_stats": {"Gu=127", "Gu=128", "Gu=129", "Gu=300", "Gu>128", "M=1", "M=7", "M=64", "K=1", "K=3", "K=7",
                    "padding", "x:nan", "x:+inf", "x:-inf", "x:subnormal", "x:FLT_MAX", "x:-0", "64xFLT_MAX",
                    "cancellation", "fp32_sum_differs", "no_real", "signed_zero_tie"},
    "item_union": {"ni=1", "ni=31", "ni=32", "ni=33", "ni=8191", "ni=8192", "ni=8193", "ni=2^20+5", "n=0",
                   "all_padding", "bits_past_8192", "last_word_partial", "repeats", "bad_id"},
    "cocount": {"Nu=0", "Nu=1", "Nu=2", "cap=need-1", "row=1023", "row=1024", "row=1025", "row=2048", "row=3073",
                "empty_first_tile", "empty_last_tile", "users>65535", "empty_row"},
    "select": {"P=1", "P=31", "P=32", "P=33", "P=255", "P=256", "k=1", "k=P", "penalty=0", "penalty=subnormal",
               "penalty=1e30", "winner_warp>0", "tie_across_warps", "unrated", "padding", "score:nan", "score:+inf",
               "score:-inf", "bad_id"},
    "cosine": {"Q=1", "Q=255", "Q=256", "Q=257", "repeats", "unrated"},
    "ws_bytes": {"default", "all_fit", "chunked", "bound=bytes_of(c)", "bound=bytes_of(c)-1", "capped_by_items",
                 "floor_one"},
    "rescore": {"U=1", "U=3000", "chunk=U=1", "chunk=1", "chunk=1025", "chunk>1024", "multi_chunk", "ni=32", "ni=33",
                "ni=8193", "ni=32769", "cand:all", "cand:shared", "cand:dup", "cand:bad", "edit:own", "edit:dup",
                "edit:bad", "slot_user:bad", "edit_row>32", "out_cap=total", "out_cap=total-1", "exclude:0",
                "exclude:1"},
    "invalidate": {"D=256", "full_prefix", "U>256", "full", "complete", "empty_prefix", "rescored_hit"},
    "settle": {"U=1024", "U=1025", "U=3000", "D=256", "full_prefix", "thr=-1", "thr=-2", "thr:nan", "nan_entry",
               "tie_before", "tie_after", "redo", "complete"},
}

REGIMES = {"group_rows": group_rows_regimes, "group_pairs": group_pairs_regimes, "group_stats": group_stats_regimes,
           "item_union": item_union_regimes, "cocount": cocount_regimes, "select": select_regimes,
           "cosine": cosine_regimes, "ws_bytes": ws_regimes, "rescore": rescore_regimes,
           "invalidate": invalidate_regimes, "settle": settle_regimes}


@functools.lru_cache(None)
def all_cases():
    return tuple(group_rows_cases() + group_pairs_cases() + group_stats_cases() + item_union_cases() +
                 cocount_cases() + select_cases() + cosine_cases() + ws_cases() + rescore_cases() +
                 invalidate_cases() + settle_cases())
