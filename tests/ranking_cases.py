"""Adversarial cases for the inference path's ranking and selection kernels, and their brute-force orders.

The orders are written here from the contracts in include/igmc_b200.h, not taken from the host twins in
igmc_b200/recommend.py:
  igmc_topk_merge, igmc_score_scatter   s = fp32 sum of the K checkpoint predictions in checkpoint order, then / K;
                                        score descending, item ascending, NaN after every number, empty slots last
  igmc_influence_topk                   pro: value descending, con: value ascending; index ascending; NaN last;
                                        empty slots (-1, -inf) / (-1, +inf)
  igmc_occlusion_order                  delta = fp32(occluded - score); |delta| descending, NaN last, ties by j;
                                        top-m rows padded with -1 / delta 0
  igmc_corated_items, _sessions         w = A r, w[u] = 0, paths = w^T A in int64; paths descending, item ascending,
                                        items without a bridge never returned
Every case claims the regimes it is built to reach; ``*_regimes`` re-derive them from the case's data alone, so a
case that silently stops reaching its regime fails (tests/test_ranking_cases.py on the host, and the GPU test before
it compares).  Scores use palettes of ties, signed zeros, infinities, NaN payloads, subnormals, neighbouring floats,
all-equal and all-NaN values next to a distinct-random control; ids come shuffled and include 2^31 - 1."""
import functools

import numpy as np
import scipy.sparse as ssp

MERGE_THREADS = 256          # csrc/recommend.cu: threads of one k_topk_merge CTA (and of one k_infl_topk CTA)
SMEM_DEFAULT = 48 * 1024     # dynamic shared memory a launch gets without opting in
SMEM_MAX = 227 * 1024        # what one CTA may opt in to on sm_90
MERGE_HEAD = 16              # csrc/topk_merge.cuh: the head ahead of the lists (k_topk_merge's segment-end word)
RETRIEVE_CHUNK = 512         # csrc/retrieve.cu: threads of a k_corated CTA = items per chunk of its tie scan
RETRIEVE_SMEM = 200 * 1024   # csrc/retrieve.cu: histograms up to this size live in shared memory
ID_MAX = 2 ** 31 - 1

PALETTES = ("few", "signed_zero", "inf", "nan", "subnormal", "near_one", "equal", "all_nan", "random")
NAN_BITS = (0x7fc00000, 0xffc00000, 0x7fc00001, 0x7f800001, 0xffffffff, 0x7fd23456)


def f32_bits(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def palette(name, n, rng):
    """n fp32 values of the named palette"""
    one_up, one_down = np.nextafter(np.float32(1), np.float32(2)), np.nextafter(np.float32(1), np.float32(0))
    nans = f32_bits(NAN_BITS)
    if name == "few":
        return rng.choice(np.float32([0.25, 0.5, 1.5, 3.0]), n)
    if name == "signed_zero":
        return rng.choice(np.float32([0.0, -0.0, 0.0, -0.0, 1.0, -1.0]), n)
    if name == "inf":
        return rng.choice(np.float32([np.inf, -np.inf, 0.5, -0.5]), n)
    if name == "nan":
        return np.where(rng.random(n) < 0.4, rng.choice(nans, n), rng.choice(np.float32([0.5, 1.0, -2.0]), n))
    if name == "subnormal":
        return rng.choice(f32_bits([1, 2, 3, 0x007fffff, 0x00800000, 0x80000001, 0x80000002, 0]), n)
    if name == "near_one":
        return rng.choice(np.float32([1.0, one_up, one_down]), n)
    if name == "equal":
        return np.full(n, 0.75, np.float32)
    if name == "all_nan":
        return rng.choice(nans, n)
    if name == "random":
        v = np.unique(rng.standard_normal(2 * n + 16).astype(np.float32))
        return rng.permutation(v)[:n]
    raise ValueError(name)


def shuffled_ids(n, rng, hi=ID_MAX):
    """n distinct ids in [0, hi], shuffled, hi among them when n > 0"""
    if n == 0:
        return np.zeros(0, np.int64)
    pool = np.unique(rng.integers(0, hi, 2 * n + 8))
    ids = np.concatenate([rng.permutation(pool)[:n - 1], [hi]])
    return rng.permutation(ids).astype(np.int64)


# ---- fp32 comparison: bit for bit through the int32 view, NaN only as NaN unless its payload must survive ---------------
def same_f32(got, want, keep_nan_bits=False):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    if got.shape != want.shape:
        return False
    eq = got.view(np.int32) == want.view(np.int32)
    if not keep_nan_bits:
        eq |= np.isnan(got) & np.isnan(want)
    return bool(eq.all())


# ---- brute-force orders ---------------------------------------------------------------------------------------------------
def order_desc(values, ids):
    """positions of values by value descending (-0 == +0), NaN after every number, then id ascending"""
    v = np.asarray(values, np.float32)
    nan = np.isnan(v)
    return np.lexsort((np.asarray(ids, np.int64), -np.where(nan, 0, v).astype(np.float64), nan))


def order_asc(values, ids):
    v = np.asarray(values, np.float32)
    nan = np.isnan(v)
    return np.lexsort((np.asarray(ids, np.int64), np.where(nan, 0, v).astype(np.float64), nan))


def top_list(values, ids, k, order, pad):
    o = order(values, ids)[:k]
    tv, ti = np.full(k, pad, np.float32), np.full(k, -1, np.int64)
    tv[:len(o)], ti[:len(o)] = np.asarray(values, np.float32)[o], np.asarray(ids, np.int64)[o]
    return tv, ti


def ckpt_mean(preds):
    """preds [K, n] -> the fp32 mean summed q = 0 .. K-1, then / K (K = 1: the values as they are)"""
    preds = np.asarray(preds, np.float32)
    with np.errstate(all="ignore"):
        a = preds[0].copy()
        for q in range(1, len(preds)):
            a = (a + preds[q]).astype(np.float32)
        return a if len(preds) == 1 else (a / np.float32(len(preds))).astype(np.float32)


def ckpt_mean_reversed(preds):
    preds = np.asarray(preds, np.float32)
    return ckpt_mean(preds[::-1]) if len(preds) > 1 else preds[0]


def ties_at(values, ids, k):
    """the k-th and (k+1)-th entries of the order have the same key (NaN counts as one key)"""
    v = np.asarray(values, np.float32)
    if len(v) <= k:
        return False
    o = order_desc(v, ids)
    a, b = v[o[k - 1]], v[o[k]]
    return bool((np.isnan(a) and np.isnan(b)) or a == b)


# ---- igmc_topk_merge / igmc_score_scatter ---------------------------------------------------------------------------------
# A stream is one run's candidates in batch order: per query slot a contiguous run of (item, preds[K]); `cuts` are the
# real entries of each call; `pad` entries of tag -1 follow the last call's.
MIXED_SEGS = (1, 1, 1, 255, 256, 257, 600, 1, 40)          # the 600-run continues over three calls of MIXED_CUTS
MIXED_CUTS = ((3, 500, 512, 300, 97), (700, 712), (1, 2, 1409))


def merge_cases():
    cases = []
    ks = (1, 2, 7, 255, 256)
    for pi, pal in enumerate(PALETTES):
        for kj, k in enumerate(ks):
            K = (1, 2, 3, 4)[(pi + kj) % 4]
            claims = {"long_segment"}
            if pal in ("few", "signed_zero", "equal", "all_nan", "near_one", "subnormal") or (pal == "inf" and k < 7):
                claims.add("ties_at_k")
            if pal in ("nan", "all_nan"):
                claims.add("nan")
            if K >= 3:
                claims.add("sum_order")
            cases.append(dict(kernel="merge", name="%s k=%d K=%d" % (pal, k, K), palette=pal, k=k, K=K,
                              segs=MIXED_SEGS, cuts=MIXED_CUTS, pad=30, seed=100 * pi + kj, claims=claims))
    # batch sizes at k = 256 around the 48 KB and 227 KB shared-memory limits; one user spans each big batch
    for B, segs, claims in ((1, (2, 3), set()), (50, (20, 1, 29), set()),
                            (3838, (3838,), {"ties_at_k", "long_segment"}),
                            (3839, (3839,), {"ties_at_k", "long_segment", "smem_over_48k"}),
                            (19113, (9000, 10113), {"ties_at_k", "long_segment", "smem_over_48k", "nan"})):
        total = sum(segs)
        cuts = (tuple([B] * (total // B) + ([total % B] if total % B else [])),)
        pal = "nan" if B == 19113 else "few"
        cases.append(dict(kernel="merge", name="B=%d" % B, palette=pal, k=256, K=2 if B == 19113 else 1,
                          segs=segs, cuts=cuts, pad=0, seed=7 + B, claims=claims))
    return cases


def merge_stream(case):
    """(slot [n], item [n], preds [K, n]) of the case's stream"""
    rng = np.random.default_rng(case["seed"])
    segs, K = case["segs"], case["K"]
    slot = np.concatenate([np.full(s, j, np.int64) for j, s in enumerate(segs)])
    item = np.concatenate([shuffled_ids(s, rng) for s in segs])
    preds = np.stack([palette(case["palette"], len(slot), rng) for _ in range(K)])
    if K >= 3:   # entries whose mean depends on the summation order: (1 + 2^25) - 2^25 = 0, (-2^25 + 2^25) + 1 = 1
        preds[:, :4] = 0
        preds[:3, :4] = np.float32([[1], [2 ** 25], [-2 ** 25]])
    return slot, item, preds


def merge_calls(case, cuts):
    """per call (preds [K, B], tag [B], items [B]) with the padding after the last call's real entries"""
    slot, item, preds = merge_stream(case)
    calls, pos = [], 0
    for c, n in enumerate(cuts):
        pad = case["pad"] if c == len(cuts) - 1 else 0
        tag = np.concatenate([slot[pos:pos + n], np.full(pad, -1, np.int64)])
        it = np.concatenate([item[pos:pos + n], np.zeros(pad, np.int64)]).astype(np.int32)
        pr = np.concatenate([preds[:, pos:pos + n], np.full((case["K"], pad), np.nan, np.float32)], axis=1)
        calls.append((np.ascontiguousarray(pr), tag, it, (pos, pos + n)))
        pos += n
    assert pos == len(slot)
    return calls


def merge_reference(case, upto):
    """the running lists [slots, k] after the stream's first `upto` entries"""
    slot, item, preds = merge_stream(case)
    s = ckpt_mean(preds)
    k, n_slots = case["k"], len(case["segs"])
    ts, ti = np.full((n_slots, k), -np.inf, np.float32), np.full((n_slots, k), -1, np.int64)
    for j in range(n_slots):
        sel = np.nonzero(slot[:upto] == j)[0]
        ts[j], ti[j] = top_list(s[sel], item[sel], k, order_desc, -np.inf)
    return ts, ti


def merge_regimes(case):
    slot, item, preds = merge_stream(case)
    s, k = ckpt_mean(preds), case["k"]
    got = set()
    if any(ties_at(s[slot == j], item[slot == j], k) for j in range(len(case["segs"]))):
        got.add("ties_at_k")
    if np.isnan(s).any():
        got.add("nan")
    if case["K"] >= 2 and not same_f32(ckpt_mean_reversed(preds), s):
        got.add("sum_order")
    for cuts in case["cuts"]:
        pos = 0
        for c, n in enumerate(cuts):
            B = n + (case["pad"] if c == len(cuts) - 1 else 0)
            runs = np.diff(np.flatnonzero(np.diff(np.concatenate([[-2], slot[pos:pos + n], [-3]]))))
            if runs.max() > MERGE_THREADS:
                got.add("long_segment")
            if MERGE_HEAD + (k + B) * 12 > SMEM_DEFAULT:
                got.add("smem_over_48k")
            pos += n
    return got


def scatter_cases():
    return [dict(kernel="scatter", name="%s K=%d" % (pal, K), palette=pal, K=K, n=700, B=300, seed=11 * i + K,
                 claims={"nan"} if pal in ("nan", "all_nan") else ({"sum_order"} if K >= 3 else set()))
            for i, pal in enumerate(PALETTES) for K in (1, 2, 3, 4)]


def scatter_data(case):
    """(preds [K, B], tag [B]: a permutation of n pair indices cut to B with -1 tags spread in, n)"""
    rng = np.random.default_rng(case["seed"])
    K, B, n = case["K"], case["B"], case["n"]
    preds = np.stack([palette(case["palette"], B, rng) for _ in range(K)])
    if K >= 3:
        preds[:, :4] = 0
        preds[:3, :4] = np.float32([[1], [2 ** 25], [-2 ** 25]])
    tag = rng.permutation(n)[:B].astype(np.int64)
    tag[rng.random(B) < 0.2] = -1
    return preds, tag, n


def scatter_regimes(case):
    preds, tag, _ = scatter_data(case)
    got = set()
    if np.isnan(ckpt_mean(preds)[tag >= 0]).any():
        got.add("nan")
    if case["K"] >= 2 and not same_f32(ckpt_mean_reversed(preds)[tag >= 0], ckpt_mean(preds)[tag >= 0]):
        got.add("sum_order")
    return got


# ---- igmc_influence_topk ---------------------------------------------------------------------------------------------------
def influence_cases():
    return [
        dict(kernel="influence", name="T=1 k=1 small batches", T=1, k=1, cuts=((5, 5, 3), (13,)), seed=12,
             claims={"ties_at_k", "nan"}),
        dict(kernel="influence", name="T=3 k=256", T=3, k=256, cuts=((300, 280, 400), (980,), (1, 979)), seed=2,
             claims={"ties_at_k", "nan", "long_segment"}),
        dict(kernel="influence", name="T=1024 k=256", T=1024, k=256, cuts=((600, 500), (1100,)), seed=3,
             claims={"ties_at_k", "nan", "long_segment"}),
        dict(kernel="influence", name="T=3 k=256 past 48 KB", T=3, k=256, cuts=((3836, 3000), (6836,)), seed=21,
             claims={"ties_at_k", "nan", "long_segment", "smem_over_48k"}),
        dict(kernel="influence", name="T=3 k=256 at 227 KB", T=3, k=256, cuts=((19108, 5000), (5000, 19108)), seed=5,
             claims={"ties_at_k", "nan", "long_segment", "smem_over_48k"}),
        dict(kernel="influence", name="T=1 k=1 at 227 KB", T=1, k=1, cuts=((19363,),), seed=6,
             claims={"ties_at_k", "long_segment", "smem_over_48k"}),
    ]


def influence_stream(case):
    """(index [N] shuffled, values [N, T]): column t from palette (t + seed) mod 9"""
    rng = np.random.default_rng(case["seed"])
    N, T = sum(case["cuts"][0]), case["T"]
    idx = shuffled_ids(N, rng)
    vals = np.stack([palette(PALETTES[(t + case["seed"]) % len(PALETTES)], N, rng) for t in range(T)], 1)
    return idx, np.ascontiguousarray(vals)


def influence_calls(case, cuts):
    """per call (S [B, T], tag [B], (start, end)): negative tags (-1 and -7) inside the batch and at its tail"""
    idx, vals = influence_stream(case)
    rng = np.random.default_rng(case["seed"] + 1000)
    calls, pos = [], 0
    for n in cuts:
        holes = min(3, n)
        at = np.sort(rng.integers(0, n + 1, holes))
        tag = np.insert(idx[pos:pos + n], at, -1)
        tag[np.flatnonzero(tag < 0)[:1]] = -7
        tag = np.concatenate([tag, [-1, -1]])
        S = np.insert(vals[pos:pos + n], at, np.float32(np.nan), axis=0)
        S = np.concatenate([S, np.full((2, case["T"]), -np.inf, np.float32)])
        calls.append((np.ascontiguousarray(S, np.float32), tag.astype(np.int64), (pos, pos + n)))
        pos += n
    return calls


def influence_reference(case, upto):
    """(pro_v, pro_i, con_v, con_i) [T, k] after the stream's first `upto` training pairs"""
    idx, vals = influence_stream(case)
    T, k = case["T"], case["k"]
    out = [np.zeros((T, k), np.float32), np.zeros((T, k), np.int64), np.zeros((T, k), np.float32),
           np.zeros((T, k), np.int64)]
    for t in range(T):
        out[0][t], out[1][t] = top_list(vals[:upto, t], idx[:upto], k, order_desc, -np.inf)
        out[2][t], out[3][t] = top_list(vals[:upto, t], idx[:upto], k, order_asc, np.inf)
    return out


def influence_regimes(case):
    idx, vals = influence_stream(case)
    k = case["k"]
    got = set()
    for t in range(case["T"]):
        if ties_at(vals[:, t], idx, k) or ties_at(-vals[:, t], idx, k):
            got.add("ties_at_k")
    if np.isnan(vals).any():
        got.add("nan")
    for cuts in case["cuts"]:
        for n in cuts:
            B = n + min(3, n) + 2
            if B > MERGE_THREADS:
                got.add("long_segment")
            if MERGE_HEAD + (k + B) * 12 > SMEM_DEFAULT:
                got.add("smem_over_48k")
    return got


# ---- igmc_occlusion_order ---------------------------------------------------------------------------------------------------
# chosen (score, occluded) segments: inf - inf = NaN, -0 - +0 = -0, differences that round to one value, subnormals,
# NaN next to zero
CHOSEN = (
    (np.inf, [np.inf, 1.0, -np.inf, np.inf, 2.0]),
    (0.0, [-0.0, 0.0, -0.0, 1e-45, -1e-45, 2e-45, 1.1754942e-38]),
    (1e8, [0.5, 1.0, 2.0, -3.0, 1e8, 1.5]),
    (1.0, [1.0000001, 0.99999994, 1.0, 1.0000001, 1.0]),
    (1.1754944e-38, [1.1754945e-38, 1.1754942e-38, 1.1754944e-38, 1.1754945e-38]),
    (0.0, [np.nan, 0.5, 0.0, np.nan, -0.0]),            # NaN after zero: NaN's key must not collide with |0|'s
)


def occlusion_cases():
    cases = []
    big = (0, 1, 0, 2 ** 16 + 3, 7, 0, 1_000_003, 0)
    for m, with_score in ((0, True), (1, False), (3, True), (256, False)):
        cases.append(dict(kernel="occlusion", name="big m=%d score=%s" % (m, with_score), lengths=big, m=m,
                          with_score=with_score, chosen=False, seed=m * 2 + with_score,
                          claims={"ties_at_k", "nan"} if m else {"nan"}))
    chosen_len = tuple([0] + [len(o) for _, o in CHOSEN[:2]] + [0] + [len(o) for _, o in CHOSEN[2:]] + [0])
    for m in (0, 1, 3, 256):
        for with_score in (True, False):
            cases.append(dict(kernel="occlusion", name="chosen m=%d score=%s" % (m, with_score), lengths=chosen_len,
                              m=m, with_score=with_score, chosen=True, seed=50 + m,
                              claims={"nan"} | ({"ties_at_k"} if m in (1, 3) else set())))
    for m in (1, 3, 256):
        cases.append(dict(kernel="occlusion", name="T=0 m=%d" % m, lengths=(0, 0, 0), m=m, with_score=True,
                          chosen=False, seed=9, claims=set()))
    return cases


def occlusion_data(case):
    """(score [P] or None, occluded [T], offsets [P+1], user, item, rating [T] distinct random per position)"""
    if case["name"] not in _OCCLUSION:
        _OCCLUSION.clear()
        _OCCLUSION[case["name"]] = _occlusion_data(case)
    return _OCCLUSION[case["name"]]


_OCCLUSION = {}


def _occlusion_data(case):
    rng = np.random.default_rng(case["seed"])
    lengths = np.asarray(case["lengths"], np.int64)
    offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    P, T = len(lengths), int(offsets[-1])
    if case["chosen"]:
        sc, occ = [], []
        it = iter(CHOSEN)
        for n in lengths:
            if n == 0:
                sc.append(np.float32(0.5))
            else:
                s, o = next(it)
                sc.append(s)
                occ += o
        score, occluded = np.float32(sc), np.float32(occ)
    else:
        score = palette("random", P, rng)
        occluded = np.concatenate([palette(PALETTES[i % len(PALETTES)], int(c), rng)
                                   for i, c in enumerate(np.full(9, T // 9) + (np.arange(9) < T % 9))])
        occluded = rng.permutation(occluded) if T else np.zeros(0, np.float32)
        if T:
            occluded[offsets[3]:offsets[3] + 40] = score[3] + np.float32(0.25)   # ties among equal deltas
    user, item, rating = (shuffled_ids(T, rng).astype(np.int32) for _ in range(3))
    return (score if case["with_score"] else None), occluded.astype(np.float32), offsets, user, item, rating


def occlusion_delta(score, occluded, offsets):
    q = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets))
    if score is None:
        return occluded.copy()
    with np.errstate(all="ignore"):
        return (occluded - score[q]).astype(np.float32)


def occlusion_reference(case):
    """(positions in output order: [T] for m = 0, else [P, m] padded with -1; delta [T])"""
    score, occluded, offsets, _, _, _ = occlusion_data(case)
    d = occlusion_delta(score, occluded, offsets)
    P, T = len(offsets) - 1, int(offsets[-1])
    q = np.repeat(np.arange(P), np.diff(offsets))
    j = np.arange(T) - offsets[q]
    nan = np.isnan(d)
    order = np.lexsort((j, -np.abs(np.where(nan, 0, d)).astype(np.float64), nan, q))
    if case["m"] == 0:
        return order, d
    top = np.full((P, case["m"]), -1, np.int64)
    for p in range(P):
        seg = order[offsets[p]:offsets[p + 1]][:case["m"]]
        top[p, :len(seg)] = seg
    return top, d


def occlusion_regimes(case):
    score, occluded, offsets, _, _, _ = occlusion_data(case)
    d = occlusion_delta(score, occluded, offsets)
    got = set()
    if np.isnan(d).any():
        got.add("nan")
    m = case["m"]
    for p in range(len(offsets) - 1):
        seg = np.abs(d[offsets[p]:offsets[p + 1]])
        if m and ties_at(seg, np.arange(len(seg)), m):
            got.add("ties_at_k")
    return got


# ---- igmc_corated_items / igmc_corated_sessions ------------------------------------------------------------------------------
def _graph(pairs, nu, ni):
    u, v = np.asarray(pairs, np.int64).T if len(pairs) else (np.zeros(0, np.int64), np.zeros(0, np.int64))
    return ssp.csr_matrix((np.ones(len(u), np.float32), (u, v)), shape=(nu, ni))


def graph_chunk_ties():
    """user 0 rates item 0, as do users 1 and 2; users 1 and 2 rate items 1..9 (2 bridges each), user 1 alone items
    10..2999 (1 bridge each: 2990 ties); user 4 rates item 3999, which nobody else rated; user 5 rates items 3997 and
    3998, user 6 item 3998 and items 3990..3995 (user 5's 6 bridged items, one bridge each); users 3 and 7.. rate
    nothing"""
    pairs = [(0, 0), (1, 0), (2, 0)] + [(u, i) for u in (1, 2) for i in range(1, 10)]
    pairs += [(1, i) for i in range(10, 3000)] + [(4, 3999)]
    pairs += [(5, 3997), (5, 3998), (6, 3998)] + [(6, i) for i in range(3990, 3996)]
    return _graph(pairs, 40, 4000)


def graph_bytes(nu=65600):
    """user 0 and users 1..65538 rate item 0 (one shared item each: w = 1); item v_c is rated by the first c of them,
    c in COUNTS: bridge counts around 255/256 and 65535/65536.  65600 users: the histograms leave shared memory"""
    pairs = [(u, 0) for u in range(0, 65539)]
    for j, c in enumerate(BYTE_COUNTS):
        pairs += [(u, 1 + j) for u in range(1, 1 + c)]
    return _graph(pairs, nu, 64)


BYTE_COUNTS = (255, 256, 257, 65535, 65536, 65537, 1, 511, 512, 256)


def graph_top_byte():
    """user 0 and 4096 users rate items 0..4096 (w = 4097 each); items 4097 and 4098 are rated by all 4096 (paths
    4096 * 4097 = 2^24 + 4096), items 4099 and 4100 by 4095 (2^24 - 1), item 4101 by one: about 17 M ratings"""
    a, n = 4097, 4096
    users = np.arange(1, n + 1)
    blocks = [np.stack([np.zeros(a, np.int64), np.arange(a)], 1),
              np.stack([np.repeat(users, a), np.tile(np.arange(a), n)], 1)]
    for it, cnt in ((4097, n), (4098, n), (4099, n - 1), (4100, n - 1), (4101, 1)):
        blocks.append(np.stack([users[:cnt], np.full(cnt, it)], 1))
    u, v = np.concatenate(blocks).T
    return ssp.csr_matrix((np.ones(len(u), np.float32), (u, v)), shape=(n + 1, 4102))


GRAPHS = {"chunk_ties": graph_chunk_ties, "bytes": graph_bytes, "top_byte": functools.lru_cache(1)(graph_top_byte)}


def corated_cases():
    cases = []
    q_ties = (0, 0, 3, 4, 1, 2, 5)   # duplicates, a user with no ratings, one whose item has no co-raters
    for m in (1200, 5, 6, 7, 600, 2999, 4000):   # user 5 has m + 1, m and m - 1 bridged items at m = 5, 6, 7
        for exclude in (True, False):
            cases.append(dict(kernel="corated", name="chunk ties m=%d exclude=%s" % (m, exclude), graph="chunk_ties",
                              users=q_ties + (40,), m=m, exclude=exclude,
                              claims={"retriever_shared"} | ({"ties_span_chunks", "ties_at_k"} if m == 1200 else set())))
    rng = np.random.default_rng(3)
    q_bytes = tuple([0] + rng.choice(np.arange(1, 65539), 299, replace=False).tolist() + [65590, 70000])
    for m in (1, 2, 3, 4, 5, 6, 7, 10):
        cases.append(dict(kernel="corated", name="byte straddle m=%d" % m, graph="bytes", users=q_bytes, m=m,
                          exclude=True, claims={"retriever_global"} | ({"ties_at_k"} if m == 7 else set())))
    for m, exclude in ((3, True), (2, True), (5, True), (6, False)):
        cases.append(dict(kernel="corated", name="2^24 m=%d exclude=%s" % (m, exclude), graph="top_byte",
                          users=(0, 0), m=m, exclude=exclude,
                          claims={"retriever_shared", "radix_top_byte"} | ({"ties_at_k"} if m in (3, 6) else set())
                          | ({"ties_span_chunks"} if not exclude else set())))
    # histograms and keys of 48 896 bytes: with the kernel's static shared words past the 48 KB a launch gets unasked
    cases.append(dict(kernel="corated", name="row at 48 KB m=2048", graph="at_48k", users=(5, 6, 3, 4), m=2048,
                      exclude=True, claims={"retriever_shared"}))
    # one query, m a power of two with the threshold's ties spread over chunks: a selection that takes one tie too
    # many writes a sort key past the CTA's workspace row
    cases.append(dict(kernel="corated", name="global ties m=1024", graph="bytes_ties", users=(0,), m=1024,
                      exclude=True, claims={"retriever_global", "ties_span_chunks", "ties_at_k"}))
    return cases


def graph_bytes_ties():
    """graph_chunk_ties' bridges on 60 000 users: the histograms live in global memory"""
    A = graph_chunk_ties().tocoo()
    return ssp.csr_matrix((A.data, (A.row, A.col)), shape=(60000, 4000))


GRAPHS["bytes_ties"] = graph_bytes_ties


def graph_at_48k():
    """graph_chunk_ties on 4096 users: row_bytes(4096, 4000, 2048) = 48 896"""
    A = graph_chunk_ties().tocoo()
    return ssp.csr_matrix((A.data, (A.row, A.col)), shape=(4096, 4000))


GRAPHS["at_48k"] = graph_at_48k


def row_bytes(nu, ni, m):
    def a256(x):
        return (x + 255) // 256 * 256
    return a256(nu * 4) + a256(ni * 4) + (1 << max(0, int(m - 1).bit_length())) * 8


def retriever_shared(nu, ni, m):
    return row_bytes(nu, ni, m) <= RETRIEVE_SMEM


def corated_paths(A, rows, users):
    """paths [U, ni] int64 for query rows `rows` (item arrays) of users `users` (ids outside A: no w[u] to clear):
    w = A r, w[u] = 0, paths = w^T A"""
    nu, ni = A.shape
    A = ssp.csr_matrix((np.ones(A.nnz, np.int64), A.indices, A.indptr), shape=A.shape)
    R = ssp.csr_matrix((np.ones(sum(len(r) for r in rows), np.int64),
                        np.concatenate([np.asarray(r, np.int64) for r in rows] + [np.zeros(0, np.int64)]),
                        np.concatenate([[0], np.cumsum([len(r) for r in rows])])), shape=(len(rows), ni))
    W = (R @ A.T).tocsr()
    P = np.asarray((W @ A).todense(), np.int64)
    for j, u in enumerate(users):
        if 0 <= u < nu and W[j, u]:
            P[j] -= int(W[j, u]) * A[u].toarray()[0]
    return P


def corated_select(paths, rows, m, exclude):
    """(items [U, m], paths [U, m]) int32 by the contract, and per query the threshold count and its tie items"""
    U = len(paths)
    items, out = np.full((U, m), -1, np.int32), np.zeros((U, m), np.int32)
    thresholds = []
    for j in range(U):
        p = paths[j].copy()
        if exclude:
            p[np.asarray(rows[j], np.int64)] = 0
        o = np.lexsort((np.arange(len(p)), -p))
        o = o[p[o] > 0][:m]
        items[j, :len(o)], out[j, :len(o)] = o, p[o]
        thr = int(p[o[-1]]) if len(o) == m else 0
        tie_items = np.flatnonzero(p == thr) if thr else np.zeros(0, np.int64)
        thresholds.append((thr, tie_items, bool(thr) and int((p >= thr).sum()) > m))
    return items, out, thresholds


def corated_rows(A, users):
    nu = A.shape[0]
    return [A.indices[A.indptr[u]:A.indptr[u + 1]] if 0 <= u < nu else np.zeros(0, np.int32) for u in users]


def corated_reference(case, A=None):
    A = GRAPHS[case["graph"]]() if A is None else A
    users = list(case["users"])
    rows = corated_rows(A, users)
    items, paths, thr = corated_select(corated_paths(A, rows, users), rows, case["m"], case["exclude"])
    return items, paths, thr


def corated_regimes(case, A=None):
    A = GRAPHS[case["graph"]]() if A is None else A
    nu, ni = A.shape
    m = case["m"]
    got = {"retriever_shared" if retriever_shared(nu, ni, m) else "retriever_global"}
    items, paths, thr = corated_reference(case, A)
    if (paths >> 24).any():
        got.add("radix_top_byte")
    for t, tie_items, straddle in thr:
        if straddle:
            got.add("ties_at_k")
            if len(tie_items) > 1500 and len(np.unique(tie_items // RETRIEVE_CHUNK)) >= 3:
                got.add("ties_span_chunks")
    return got


# sessions on graph_chunk_ties: (users, session, items, values); value = label + 1, 0 deletes
SESSIONS = dict(users=(45, 0, 1, 2, 77),
                session=(0, 2, 2, 3, 3, 3),
                items=(0, 5, 10, 1, 3, 200),
                values=(3, 0, 0, 0, 2, 4))


def session_rows(A):
    """the session rows by their definition: the user's graph row (new ids: empty) with the edits applied"""
    nu = A.shape[0]
    rows = []
    for s, u in enumerate(SESSIONS["users"]):
        r = set(A.indices[A.indptr[u]:A.indptr[u + 1]].tolist()) if u < nu else set()
        for ss, it, val in zip(SESSIONS["session"], SESSIONS["items"], SESSIONS["values"]):
            if ss == s:
                (r.add if val else r.discard)(it)
        rows.append(np.array(sorted(r), np.int64))
    return rows


# the regimes every kernel's cases must reach between them
REQUIRED = {
    "merge": {"ties_at_k", "nan", "long_segment", "smem_over_48k", "sum_order"},
    "scatter": {"nan", "sum_order"},
    "influence": {"ties_at_k", "nan", "long_segment", "smem_over_48k"},
    "occlusion": {"ties_at_k", "nan"},
    "corated": {"retriever_shared", "retriever_global", "radix_top_byte", "ties_span_chunks", "ties_at_k"},
}


def all_cases():
    return merge_cases() + scatter_cases() + influence_cases() + occlusion_cases() + corated_cases()


REGIMES = {"merge": merge_regimes, "scatter": scatter_regimes, "influence": influence_regimes,
           "occlusion": occlusion_regimes, "corated": corated_regimes}
