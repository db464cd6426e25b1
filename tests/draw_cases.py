"""Cases for the Monte-Carlo-dropout draw kernels (csrc/draws.cu), and their brute-force enumerations.

The references are written from the contracts in include/igmc_b200.h in plain Python, not taken from the host twins in
igmc_b200/recommend.py:
  igmc_draws_expand  position i < G*S: pair i // S, draw i % S; positions G*S..B-1: pair 0, tag -1, draw 0
  igmc_draws_mask    edge e of graph g kept iff the high 32 bits of splitmix64(draw state + (e - edge_ptr[g])) reach
                     keep_thresh(adj_dropout), and never at adj_dropout >= 1 (kept with probability 1 - adj_dropout);
                     hidden unit o likewise at 0.5; a graph with tag < 0 keeps everything.  splitmix64, sample_state and
                     keep_thresh are restated from csrc/common.cuh / csrc/lists.cuh on Python integers
  igmc_draws_stats   the draws are ranking_cases.ckpt_mean of the checkpoint predictions; mean, std and key in Python
                     floats (IEEE fp64, in draw order, no fma), each rounded once with np.float32
Every case claims the regimes it is built to reach; ``REGIMES[kernel](case)`` re-derives them from the case's data
alone, so a case that silently stops reaching one fails.  The launch constants those regimes depend on are restated
below and checked against the sources."""
import functools
import math

import numpy as np

from tests.ranking_cases import ckpt_mean, f32_bits

EXPAND_THREADS = 256   # csrc/draws.cu: one block of k_draws_expand
MASK_THREADS = 128     # csrc/draws.cu: one stride of a k_draws_mask graph's edges
STATS_THREADS = 128    # csrc/draws.cu: pairs per k_draws_stats block
DRAWS_HOP_TAG = 4      # csrc/draws.cu: sample_state's hop slot of the draw streams
CONSTANTS = {("draws.cu", "EXPAND_THREADS"): EXPAND_THREADS, ("draws.cu", "MASK_THREADS"): MASK_THREADS,
             ("draws.cu", "STATS_THREADS"): STATS_THREADS, ("draws.cu", "DRAWS_HOP_TAG"): DRAWS_HOP_TAG}

DRAWS_MAX = 256        # IGMC_DRAWS_MAX
LIN1_OUT = 128         # IGMC_LIN1_OUT: hidden units per graph
M64 = (1 << 64) - 1
FLT_MAX = float(np.finfo(np.float32).max)


# ---- the counter hashes, restated on Python integers ----------------------------------------------------------------
def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def _unxorshift(y, s):
    x = y
    for _ in range(64 // s + 1):
        x = y ^ (x >> s)
    return x & M64


def unsplitmix64(z):
    """the inverse of splitmix64 (each step is a bijection of 64-bit words)"""
    z = _unxorshift(z, 31)
    z = (z * pow(0x94D049BB133111EB, -1, 1 << 64)) & M64
    z = _unxorshift(z, 27)
    z = (z * pow(0xBF58476D1CE4E5B9, -1, 1 << 64)) & M64
    z = _unxorshift(z, 30)
    return (z - 0x9E3779B97F4A7C15) & M64


def sample_state(seed, pid, side, hop):
    """csrc/common.cuh: splitmix64(seed ^ splitmix64(pid * 16 + hop * 2 + side)), pid an int64 read as uint64"""
    return splitmix64((seed & M64) ^ splitmix64((pid * 16 + hop * 2 + side) & M64))


def keep_thresh(p):
    """csrc/lists.cuh: p (as the kernel sees it, fp32) * 2^32 in fp64, 0xFFFFFFFF from 2^32 - 1 up"""
    t = float(np.float32(p)) * 4294967296.0
    return 0xFFFFFFFF if t >= 4294967295.0 else int(t)


def draw_state(seed, pid, s, side):
    return splitmix64((sample_state(seed, pid, side, DRAWS_HOP_TAG) + (s & 0xFFFFFFFF)) & M64)


def hash_hi(state, index):
    return splitmix64((state + index) & M64) >> 32


def keeps(state, index, p):
    """a unit is kept with probability 1 - p: never at p >= 1, else iff its hash reaches keep_thresh(p)"""
    return float(np.float32(p)) < 1.0 and hash_hi(state, index) >= keep_thresh(p)


def seed_for(pid, s, e, high):
    """the draw_seed under which edge e of draw s of pair pid hashes to the high word ``high`` (low word 0)"""
    se = (unsplitmix64(high << 32) - e) & M64
    st = (unsplitmix64(se) - s) & M64
    return unsplitmix64(st) ^ splitmix64((pid * 16 + DRAWS_HOP_TAG * 2) & M64)


# ---- igmc_draws_expand ------------------------------------------------------------------------------------------------
def _pairs(G, rng, big=False):
    u = rng.integers(0, 2 ** 31 - 1, G)
    v = rng.integers(0, 2 ** 31 - 1, G)
    pid = rng.integers(2 ** 31, 2 ** 62, G) if big else rng.integers(0, 2 ** 31, G)
    return u.astype(np.int64), v.astype(np.int64), pid.astype(np.int64), rng.permutation(G).astype(np.int64)


def expand_cases():
    spec = [  # (S, B, pair tags of -1 at, big pair ids, claims)
        (1, 1, (), False, {"S=1", "S=B", "B=1"}),
        (1, 600, (5, 300), True, {"S=1", "B>256", "pid>2^31"}),
        (7, 600, (10,), False, {"padding", "B>256", "pair_across_blocks"}),
        (256, 256, (), True, {"S=256", "S=B", "S=256,B=256"}),
        (256, 600, (), False, {"S=256", "padding", "S=256,B=600", "B>256"}),
        (3, 257, (40,), True, {"padding", "B>256", "tag=-1_mid"}),
    ]
    cases = []
    for k, (S, B, neg, big, claims) in enumerate(spec):
        G = B // S
        u, v, pid, tag = _pairs(G, np.random.default_rng(100 + k), big)
        tag[list(neg)] = -1
        cases.append(dict(kernel="expand", name="S=%d B=%d" % (S, B), S=S, B=B, pair_u=u, pair_v=v, pair_pid=pid,
                          pair_tag=tag, claims=claims))
    return cases


def expand_reference(case):
    """(links_u, links_v, pair_id, tag, draw) [B] int64 by the position rule"""
    S, B = case["S"], case["B"]
    G = B // S
    out = np.zeros((5, B), np.int64)
    for i in range(B):
        if i < G * S:
            g = i // S
            out[:, i] = (case["pair_u"][g], case["pair_v"][g], case["pair_pid"][g], case["pair_tag"][g], i - g * S)
        else:
            out[:, i] = (case["pair_u"][0], case["pair_v"][0], case["pair_pid"][0], -1, 0)
    return out


def expand_regimes(case):
    S, B = case["S"], case["B"]
    G = B // S
    got = set()
    if B == 1:
        got.add("B=1")
    if any(g * S // EXPAND_THREADS != ((g + 1) * S - 1) // EXPAND_THREADS for g in range(G)):
        got.add("pair_across_blocks")
    if S == 1:
        got.add("S=1")
    if S == B:
        got.add("S=B")
    if S == DRAWS_MAX:
        got.add("S=256")
        if B in (256, 600):
            got.add("S=256,B=%d" % B)
    if B % S:
        got.add("padding")
    if B > EXPAND_THREADS:
        got.add("B>256")
    if (np.asarray(case["pair_tag"][:max(G - 1, 0)]) == -1).any():
        got.add("tag=-1_mid")
    if (np.asarray(case["pair_pid"]) > 2 ** 31).any():
        got.add("pid>2^31")
    return got


# ---- igmc_draws_mask -------------------------------------------------------------------------------------------------
# the constructed hashes: edge 3 of draw 0 of pair 45 750 587 hashes to 0xFFFFFFFF (all 32 high bits set) under this
# seed, so it is the one edge a threshold compare alone would keep at adj_dropout = 1
P1_PID, P1_EDGE, P1_SEED = 45750587, 3, 0x3f0d2d8aa7a78368
AT_PID, AT_DRAW, AT_EDGE = 2 ** 40 + 12345, 7, 5
P_DECIMAL = 0.1        # fp32 0.100000001490116...: keep_thresh 429496736, not the decimal's 429496729


def _mask_case(name, counts, p, seed, pid, tag, draw, claims):
    return dict(kernel="mask", name=name, edge_ptr=np.concatenate([[0], np.cumsum(counts)]).astype(np.int64),
                pair_id=np.asarray(pid, np.int64), tag=np.asarray(tag, np.int64), draw=np.asarray(draw, np.int64),
                p=p, seed=seed, claims=claims)


def mask_cases():
    sizes = [0, 127, 128, 129, 300, 6, 2]
    rng = np.random.default_rng(7)
    pid = [int(x) for x in rng.integers(0, 2 ** 62, len(sizes))]
    pid[1] = 12345
    tag, draw = [0, 1, 2, 3, 4, -1, 6], [0, 3, 255, 1, 2, 0, 255]
    base = {"E=0", "E=127", "E=128", "E=129", "E>256", "padding", "draw=255", "pid>2^31"}
    cases = [
        _mask_case("sizes p=0.2 seed 0", sizes, 0.2, 0, pid, tag, draw, base | {"seed=0"}),
        _mask_case("sizes p=0 seed 2^64-1", sizes, 0.0, M64, pid, tag, draw, base | {"p=0", "seed=2^64-1"}),
        _mask_case("sizes p=1", sizes, 1.0, 99, pid, tag, draw, base | {"p=1"}),
        _mask_case("p=1 all-ones hash", [10, 6, 4], 1.0, P1_SEED, [P1_PID, 5, 6], [0, 1, -1], [0, 0, 0],
                   {"hash=0xFFFFFFFF at p=1", "padding"}),
    ]
    th = keep_thresh(P_DECIMAL)
    for name, high, claim in (("at", th, "hash=thresh kept"), ("one below", th - 1, "hash=thresh-1 dropped")):
        cases.append(_mask_case("hash %s keep_thresh(0.1)" % name, [12, 129], P_DECIMAL,
                                seed_for(AT_PID, AT_DRAW, AT_EDGE, high), [AT_PID, 77], [3, 0], [AT_DRAW, 255],
                                {claim, "p!=decimal", "E=129", "draw=255", "pid>2^31"}))
    return cases


def mask_reference(case):
    """(edge_keep [E], hidden_keep [B * 128]) uint8 by the hash rule, graph by graph"""
    ep = case["edge_ptr"]
    B = len(ep) - 1
    ek, hk = np.zeros(int(ep[-1]), np.uint8), np.zeros(B * LIN1_OUT, np.uint8)
    for g in range(B):
        pid, s = int(case["pair_id"][g]), int(case["draw"][g])
        pad = case["tag"][g] < 0
        se, sh = draw_state(case["seed"], pid, s, 0), draw_state(case["seed"], pid, s, 1)
        for e in range(int(ep[g]), int(ep[g + 1])):
            ek[e] = pad or keeps(se, e - int(ep[g]), case["p"])
        for o in range(LIN1_OUT):
            hk[g * LIN1_OUT + o] = pad or keeps(sh, o, 0.5)
    return ek, hk


def mask_regimes(case):
    ep, p = case["edge_ptr"], case["p"]
    got = set()
    p32 = float(np.float32(p))
    if p32 == 0.0:
        got.add("p=0")
    if p32 == 1.0:
        got.add("p=1")
    if p32 != p:
        got.add("p!=decimal")
    if case["seed"] == 0:
        got.add("seed=0")
    if case["seed"] == M64:
        got.add("seed=2^64-1")
    th = keep_thresh(p)
    for g in range(len(ep) - 1):
        n = int(ep[g + 1] - ep[g])
        got.add("E>256" if n > 2 * MASK_THREADS else "E=%d" % n)
        if case["tag"][g] < 0:
            got.add("padding")
            continue
        if case["draw"][g] == DRAWS_MAX - 1:
            got.add("draw=255")
        if case["pair_id"][g] > 2 ** 31:
            got.add("pid>2^31")
        se = draw_state(case["seed"], int(case["pair_id"][g]), int(case["draw"][g]), 0)
        hs = [hash_hi(se, e) for e in range(n)]
        if p32 < 1.0 and th in hs:
            got.add("hash=thresh kept")
        if p32 < 1.0 and th - 1 in hs:
            got.add("hash=thresh-1 dropped")
        if p32 >= 1.0 and 0xFFFFFFFF in hs:
            got.add("hash=0xFFFFFFFF at p=1")
    return got


# ---- igmc_draws_stats ------------------------------------------------------------------------------------------------
SPECIALS = np.float32([np.nan, np.inf, -np.inf, -0.0, 0.0, FLT_MAX, -FLT_MAX, 1.0, -2.5]).tolist() + \
    f32_bits([1, 0x80000003, 0x007fffff]).tolist()


def _stats_preds(K, B, S, rng, special):
    preds = rng.normal(3.0, 1.0, (K, B)).astype(np.float32)
    if special:
        x = np.asarray(SPECIALS, np.float32)
        preds[0, :] = rng.choice(x, B)
        if S == 2:   # pairs of specials side by side: inf - inf, FLT_MAX + FLT_MAX, -0 + -0, subnormal pairs
            preds[0, :20] = f32_bits([0x7f800000, 0xff800000, 0x7f7fffff, 0x7f7fffff, 0x80000000, 0x80000000,
                                      1, 3, 0x7f7fffff, 0xff7fffff, 0x7fc00000, 0x3f800000, 0x80000001,
                                      0x80000001, 0xff7fffff, 0xff7fffff, 0x3f800000, 0x3f800000, 0, 0x80000000])
    return preds


def stats_cases():
    spec = [  # (name, K, B, S, beta, mode, specials, tags -1 at pairs, claims)
        ("S=1 G=300 key", 1, 300, 1, 0.0, "key", True, (4,),
         {"S=1", "K=1", "G>128", "beta=0", "mode:key", "draw:nan", "draw:+inf", "draw:-inf", "draw:-0",
          "draw:subnormal", "draw:+FLT_MAX", "draw:-FLT_MAX"}),
        ("S=1 G=300 values", 3, 300, 1, 0.0, "values", False, (0, 7, 299),
         {"S=1", "K=3", "G>128", "mode:values", "tag=-1"}),
        ("S=2 specials key beta=-0", 1, 300, 2, -0.0, "key", True, (),
         {"S=2", "K=1", "G>128", "beta=-0", "mode:key", "draw:nan", "draw:+inf", "draw:-inf", "draw:-0",
          "draw:subnormal", "draw:+FLT_MAX", "draw:-FLT_MAX"}),
        ("S=2 specials values", 1, 41, 2, 0.0, "values", True, (3,),
         {"S=2", "K=1", "mode:values", "tag=-1", "values:nan", "draw:nan", "draw:+inf", "draw:-inf", "draw:-0", "draw:subnormal",
          "draw:+FLT_MAX", "draw:-FLT_MAX"}),
        ("S=2 K=3 beta<0", 3, 64, 2, -2.5, "key", True, (), {"S=2", "beta<0", "mode:key"}),
        ("S=256 B=600 values", 1, 600, 256, 0.0, "values", False, (1,), {"S=256", "K=1", "mode:values", "padding"}),
        ("S=256 B=256 key", 3, 256, 256, 1.0, "key", False, (), {"S=256", "G=1", "mode:key"}),
        ("S=3 G=133 key beta=1e300", 1, 400, 3, 1e300, "key", True, (2,), {"G>128", "beta=1e300", "mode:key"}),
    ]
    cases = []
    for k, (name, K, B, S, beta, mode, special, neg, claims) in enumerate(spec):
        rng = np.random.default_rng(200 + k)
        G = B // S
        ptag = rng.permutation(G).astype(np.int64)
        ptag[list(neg)] = -1
        tag = np.full(B, -1, np.int64)
        tag[:G * S] = np.repeat(ptag, S)
        cases.append(dict(kernel="stats", name=name, K=K, B=B, S=S, beta=beta, mode=mode, tag=tag,
                          preds=_stats_preds(K, B, S, rng, special), claims=claims))
    return cases


def stats_reference(case):
    """(x [G, S], mean [G], std [G], key [G]) fp32: each pair's statistics in Python floats, rounded once"""
    S, B = case["S"], case["B"]
    G = B // S
    x = ckpt_mean(case["preds"])[:G * S].reshape(G, S)
    out = np.zeros((3, G), np.float32)
    with np.errstate(over="ignore"):
        for g in range(G):
            total = 0.0
            for s in range(S):
                total = total + float(x[g, s])
            mean = total / S
            sd = 0.0
            if S > 1:
                ss = 0.0
                for s in range(S):
                    d = float(x[g, s]) - mean
                    ss = ss + d * d
                sd = math.sqrt(ss / (S - 1))
            out[:, g] = (np.float32(mean), np.float32(sd), np.float32(mean + case["beta"] * sd))
    return x, out[0], out[1], out[2]


def stats_outputs(case, fill):
    """what igmc_draws_stats writes: key [G], or (value [P * S], mean [P], std [P]) with P = the largest tag + 1 and
    the entries of no pair left at ``fill``"""
    S, B = case["S"], case["B"]
    G = B // S
    x, mean, sd, key = stats_reference(case)
    if case["mode"] == "key":
        return key
    P = int(case["tag"].max()) + 1
    value, mo, so = np.full(P * S, fill, np.float32), np.full(P, fill, np.float32), np.full(P, fill, np.float32)
    for g in range(G):
        t = int(case["tag"][g * S])
        if t >= 0:
            value[t * S:(t + 1) * S], mo[t], so[t] = x[g], mean[g], sd[g]
    return value, mo, so


def stats_regimes(case):
    S, B, beta = case["S"], case["B"], case["beta"]
    G = B // S
    got = {"S=%d" % S, "K=%d" % case["K"], "mode:" + case["mode"]}
    if G > STATS_THREADS:
        got.add("G>128")
    if G == 1:
        got.add("G=1")
    if B % S:
        got.add("padding")
    if beta == 0.0:
        got.add("beta=-0" if math.copysign(1.0, beta) < 0 else "beta=0")
    elif beta < 0:
        got.add("beta<0")
    elif beta >= 1e300:
        got.add("beta=1e300")
    if case["mode"] == "values" and (case["tag"][:G * S:S] < 0).any():
        got.add("tag=-1")
    x = ckpt_mean(case["preds"])[:G * S]
    bits = x.view(np.uint32)
    for name, hit in (("nan", np.isnan(x)), ("+inf", x == np.inf), ("-inf", x == -np.inf),
                      ("-0", bits == 0x80000000), ("subnormal", (x != 0) & (np.abs(x) < np.finfo(np.float32).tiny)),
                      ("+FLT_MAX", x == FLT_MAX), ("-FLT_MAX", x == -FLT_MAX)):
        if hit.any():
            got.add("draw:" + name)
    if case["mode"] == "values" and np.isnan(x).any():
        got.add("values:nan")
    return got


# ---- all cases ----------------------------------------------------------------------------------------------------------
REQUIRED = {
    "expand": {"B=1", "pair_across_blocks", "S=1", "S=B", "S=256", "S=256,B=256", "S=256,B=600", "padding", "B>256", "tag=-1_mid", "pid>2^31"},
    "mask": {"E=0", "E=127", "E=128", "E=129", "E>256", "padding", "p=0", "p=1", "p!=decimal", "hash=thresh kept",
             "hash=thresh-1 dropped", "hash=0xFFFFFFFF at p=1", "seed=0", "seed=2^64-1", "draw=255", "pid>2^31"},
    "stats": {"S=1", "S=2", "S=256", "K=1", "K=3", "draw:nan", "draw:+inf", "draw:-inf", "draw:-0", "draw:subnormal",
              "draw:+FLT_MAX", "draw:-FLT_MAX", "beta=0", "beta=-0", "beta<0", "beta=1e300", "mode:key",
              "mode:values", "tag=-1", "G>128", "G=1", "padding", "values:nan"},
}

REGIMES = {"expand": expand_regimes, "mask": mask_regimes, "stats": stats_regimes}


@functools.lru_cache(None)
def all_cases():
    return tuple(expand_cases() + mask_cases() + stats_cases())
