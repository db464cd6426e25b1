"""The subgraph extractors (csrc/extract.cu) in every regime they branch on, bit for bit against the numpy oracle.

Each case builds a rating matrix and pairs that put at least one subgraph into its regime, asserts from host quantities
that they did (``SubgraphExtractor.plan``, the extractor's ``cap`` and, per pair from the oracle's batch, the edge count
m, the user-row entries D the one-launch kernel scans and its tile count), then extracts with the one-launch path
allowed (``fast=True``) and with the generic two-launch kernels forced (``fast=False``) and compares both with
``oracle/extract_np`` under the same hash sampler on every array the model kernels read: the public arrays, the graph
offsets, ``graph_nu``, ``node_gid`` and the message-passing lists.

The regimes (constants restated from csrc/extract.cu; tests/test_extract_regime_plans.py checks without a GPU that
every case sits on the side it claims):
  - the one-launch path's shared-memory limit (110 KB) at R = 5 (1 000 and 3 706 items) and R = 12;
  - canonical edges kept in shared memory up to FX_CANO = 12 288 per subgraph, spilled to global memory above;
  - the tile table: the host admits the one-launch path only while cap * longest row <= 128 * 2 048;
  - the ballot split by rating (one lane per class): R = 1, R = 32 (every lane) and R = 33 (generic path);
  - the (item, rating) bitmaps of ceil(cap / 32) words around the word boundaries;
  - the generic path's own limits: the h = 1 item table and the h = 2 visited / candidate bitmaps (one above each
    raises, no launch);
  - sampling edges, target kinds, batch sizes, and rating sessions on both paths."""
import functools

import numpy as np
import pytest
import scipy.sparse as ssp

from oracle import extract_np
from tests.helpers import batch_equal

pytestmark = pytest.mark.gpu

FX_TILE, FX_TCAP, FX_CANO = 128, 2048, 12288
SEED = 11


# ---- rating matrices -------------------------------------------------------------------------------------------------
def _csr(u, v, lab, shape):
    """values = label + 1; the first of duplicate cells is kept"""
    u, v, lab = (np.asarray(a, np.int64) for a in (u, v, lab))
    _, first = np.unique(u * shape[1] + v, return_index=True)
    return ssp.csr_matrix(((lab[first] + 1).astype(np.float32), (u[first], v[first])), shape=shape)


def _block(rng, u0, v0, nu, nv, R, holes=()):
    """every cell of users u0.. x items v0.. except the local (a, b) in ``holes``"""
    a, b = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    keep = np.ones((nu, nv), bool)
    for h in holes:
        keep[h] = False
    a, b = a[keep], b[keep]
    return u0 + a, v0 + b, rng.integers(0, R, len(a))


def _sparse(rng, users, items, n, R):
    return rng.choice(users, n), rng.choice(items, n), rng.integers(0, R, n)


def _cat(*parts):
    return [np.concatenate([p[k] for p in parts]) for k in range(3)]


def _pairs(A, pu, pv):
    """(u, v, label) with the label of a rated target, 0 for an unrated one"""
    pu, pv = np.asarray(pu, np.int64), np.asarray(pv, np.int64)
    lab = np.asarray(A[pu, pv]).ravel()
    return pu, pv, np.where(lab > 0, lab - 1, 0).astype(np.int64)


@functools.lru_cache(maxsize=None)
def g_dense(n, R, items):
    """an n x n block (items 0..n-1; targets (i, i), i < 8, unrated) beside 100 sparse users on the other items: the
    block's columns set cap = 1 + min(n, mnph)"""
    rng = np.random.default_rng(n * 100 + R)
    blk = _block(rng, 0, 0, n, n, R, holes=[(i, i) for i in range(8)])
    sp = _sparse(rng, np.arange(n, n + 100), np.arange(n, items), 3000, R)
    A = _csr(*_cat(blk, sp), (n + 100, items))
    pu = np.r_[np.arange(8), np.arange(8), rng.integers(n, n + 100, 12)]
    pv = np.r_[np.arange(8), np.arange(1, 9), rng.integers(n, items, 12)]
    return A, _pairs(A, pu, pv), np.arange(1, R + 1, dtype=np.float32)


# g_mixed: the canonical-spill blocks beside a sparse region, cold and low-degree users / items
MIX_B1, MIX_B2, MIX_B3 = 0, 112, 224            # first user = first item of each block
MIX_SP_U, MIX_SP_V = 344, 344                    # sparse users 344..443 x items 344..643
MIX_COLD_U, MIX_COLD_V = 444, 644                # no ratings
MIX_LOW_U, MIX_LOW_V = 445, 645                  # 2 ratings / 3 raters
MIX_D20_U, MIX_D21_U, MIX_D20_V, MIX_D21_V = 446, 447, 646, 647   # 21 / 22 ratings, 21 / 22 raters
MIX_SHAPE = (448, 648)


@functools.lru_cache(maxsize=None)
def g_mixed():
    """B1: 112 x 112 with 255 holes off its first row and column, so that the pair at its corner has exactly 12 288
    edges; B2: the same with 254 holes (12 289); B3: 120 x 120 fully rated (14 399)"""
    rng = np.random.default_rng(7)

    def holes(k):
        cells = rng.choice(111 * 111, k, replace=False)
        return [(1 + c // 111, 1 + c % 111) for c in cells]
    sp_u, sp_v = np.arange(MIX_SP_U, MIX_SP_U + 100), np.arange(MIX_SP_V, MIX_SP_V + 300)
    parts = [_block(rng, MIX_B1, MIX_B1, 112, 112, 5, holes(255)), _block(rng, MIX_B2, MIX_B2, 112, 112, 5, holes(254)),
             _block(rng, MIX_B3, MIX_B3, 120, 120, 5), _sparse(rng, sp_u, sp_v, 3000, 5),
             ([MIX_LOW_U] * 2, sp_v[:2], [1, 2]), (sp_u[:3], [MIX_LOW_V] * 3, [0, 3, 4]),
             ([MIX_D20_U] * 21, sp_v[:21], rng.integers(0, 5, 21)), ([MIX_D21_U] * 22, sp_v[:22], rng.integers(0, 5, 22)),
             (sp_u[:21], [MIX_D20_V] * 21, rng.integers(0, 5, 21)), (sp_u[:22], [MIX_D21_V] * 22, rng.integers(0, 5, 22))]
    A = _csr(*_cat(*[tuple(np.asarray(x) for x in p) for p in parts]), MIX_SHAPE)
    return A, np.arange(1, 6, dtype=np.float32)


def mixed_pairs(kind, rng=None):
    A, _ = g_mixed()
    sp = lambda k, r: (r.integers(MIX_SP_U, MIX_SP_U + 100, k), r.integers(MIX_SP_V, MIX_SP_V + 300, k))  # noqa: E731
    r = np.random.default_rng(3)
    if kind == "spill":   # spilled and unspilled CTAs in one launch, in a mixed order
        su, sv = sp(12, r)
        pu = np.r_[su[:3], MIX_B1, su[3:5], MIX_B2, su[5:7], MIX_B3, MIX_B1 + 5, MIX_B2 + 18, MIX_B3 + 26, su[7:]]
        pv = np.r_[sv[:3], MIX_B1, sv[3:5], MIX_B2, sv[5:7], MIX_B3, MIX_B1 + 7, MIX_B2 + 28, MIX_B3 + 36, sv[7:]]
    elif kind == "targets":   # rated, unrated, cold user, cold item, isolated pair
        su, sv = sp(8, r)
        rows = A[su[:4]]
        rated_v = np.array([rows[k].indices[0] for k in range(4)])
        pu = np.r_[su[:4], su[4:], MIX_COLD_U, su[0], MIX_COLD_U, MIX_B1 + 3, MIX_LOW_U]
        pv = np.r_[rated_v, sv[4:], sv[0], MIX_COLD_V, MIX_COLD_V, MIX_B2 + 4, MIX_LOW_V]
    elif kind == "sampling":   # candidate counts 1..3 (ratio 0.3 keeps none), exactly mnph and mnph + 1 (mnph 20)
        pu = np.r_[MIX_LOW_U, MIX_SP_U, MIX_D20_U, MIX_D21_U, MIX_SP_U, MIX_SP_U + 1, MIX_B1, MIX_B3 + 2]
        pv = np.r_[MIX_SP_V, MIX_LOW_V, MIX_SP_V, MIX_SP_V, MIX_D20_V, MIX_D21_V, MIX_B1 + 1, MIX_B3 + 9]
    else:   # "b256": every kind above, blocks and sparse pairs in one batch
        rr = rng or np.random.default_rng(5)
        parts_u, parts_v = [], []
        for k in ("spill", "targets", "sampling"):
            u, v, _ = mixed_pairs(k)
            parts_u.append(u)
            parts_v.append(v)
        n = 256 - sum(len(u) for u in parts_u)
        blk = rr.choice([MIX_B1, MIX_B2, MIX_B3], n // 2)
        parts_u.append(blk + rr.integers(0, 112, n // 2))
        parts_v.append(blk + rr.integers(0, 112, n // 2))
        su, sv = sp(n - n // 2, rr)
        parts_u.append(su)
        parts_v.append(sv)
        perm = rr.permutation(256)
        pu, pv = np.concatenate(parts_u)[perm], np.concatenate(parts_v)[perm]
    return _pairs(A, pu, pv)


@functools.lru_cache(maxsize=None)
def g_tile(extra):
    """222 users x 1 200 items, every user rates items 0..19 and 1 160 others (rows of 1 180); ``extra``: user 0 rates
    one more (1 181).  mnph 221 gives cap 222: cap * 1 180 = 261 960 <= 262 144 < cap * 1 181"""
    rng = np.random.default_rng(22)
    u, v = [], []
    for a in range(222):
        row = np.r_[np.arange(20), 20 + rng.choice(1180, 1160 + (extra if a == 0 else 0), replace=False)]
        u.append(np.full(len(row), a))
        v.append(row)
    u, v = np.concatenate(u), np.concatenate(v)
    A = _csr(u, v, rng.integers(0, 5, len(u)), (222, 1200))
    unrated = [int(np.setdiff1d(np.arange(1200), A[a].indices)[0]) for a in (1, 2)]
    return A, _pairs(A, np.r_[0, 1, 2, 3, 100, 221, 1, 2], np.r_[0, 0, 1, 5, 19, 3, unrated]), \
        np.arange(1, 6, dtype=np.float32)


@functools.lru_cache(maxsize=None)
def g_classes(R):
    """80 x 60 at density 0.5, labels uniform over 0..R-1"""
    rng = np.random.default_rng(R)
    keep = rng.random((80, 60)) < 0.5
    u, v = np.nonzero(keep)
    A = _csr(u, v, rng.integers(0, R, len(u)), (80, 60))
    pu, pv = rng.integers(0, 80, 16), rng.integers(0, 60, 16)
    return A, _pairs(A, pu, pv), np.arange(1, R + 1, dtype=np.float32)


@functools.lru_cache(maxsize=None)
def g_words(n):
    """n x n without its diagonal: every degree is n - 1, cap = n; the unrated pair (0, 0) has n nodes per side"""
    rng = np.random.default_rng(n)
    A = _csr(*_block(rng, 0, 0, n, n, 5, holes=[(i, i) for i in range(n)]), (n, n))
    return A, _pairs(A, [0, 1, n - 1, 3], [0, 2, n - 1, 5]), np.arange(1, 6, dtype=np.float32)


@functools.lru_cache(maxsize=None)
def g_items(items):
    """30 users over ``items`` items: user 0 rates 200 (cap 201), the others 20 each"""
    rng = np.random.default_rng(items % 1000)
    u = np.r_[np.zeros(200, np.int64), np.repeat(np.arange(1, 30), 20)]
    v = np.r_[np.arange(200), rng.integers(0, items, 29 * 20)]
    v[200:220] = np.arange(20)          # user 1 shares items with user 0
    A = _csr(u, v, rng.integers(0, 5, len(u)), (30, items))
    return A, _pairs(A, [0, 0, 1, 2, 5, 0, 29, 1], [5, 199, 3, v[240], 7, items - 1, v[-1], items - 1]), \
        np.arange(1, 6, dtype=np.float32)


@functools.lru_cache(maxsize=None)
def g_h2(N):
    """N users x N items, 3 N sparse ratings; user 0 rates items 0..14 and item 0 is rated by users 0..14, so that
    mnph 10 gives cap 1 + 10 + 10 = 21 at h = 2"""
    rng = np.random.default_rng(N)
    u = np.r_[np.zeros(15, np.int64), np.arange(15), rng.integers(0, N, 3 * N)]
    v = np.r_[np.arange(15), np.zeros(15, np.int64), rng.integers(0, N, 3 * N)]
    A = _csr(u, v, rng.integers(0, 5, len(u)), (N, N))
    k = rng.integers(30, len(u), 10)
    return A, _pairs(A, np.r_[0, 3, u[k]], np.r_[0, 7, v[k]]), np.arange(1, 6, dtype=np.float32)


@functools.lru_cache(maxsize=None)
def g_long(long_row):
    """item 0 rated by users 0..4 999 (5 000 candidates), every user ~3 more ratings; ``long_row``: user 0 also rates
    4 500 items (cap 101 * 4 500 > 262 144: the generic path)"""
    rng = np.random.default_rng(4096 + long_row)
    items = 5000 if long_row else 300
    u = np.r_[np.arange(5000), rng.integers(0, 5200, 15600)]
    v = np.r_[np.zeros(5000, np.int64), rng.integers(1, items, 15600)]
    if long_row:
        u, v = np.r_[u, np.zeros(4500, np.int64)], np.r_[v, np.arange(1, 4501)]
    A = _csr(u, v, rng.integers(0, 5, len(u)), (5200, items))
    return A, _pairs(A, [0, 17, 4999, 5100, 0, 3], [0, 0, 0, 0, items - 1, 1]), np.arange(1, 6, dtype=np.float32)


# ---- cases ---------------------------------------------------------------------------------------------------------
# build: () -> (A, (pu, pv, labels), class_values); path: what a fast=True extractor takes ("fast", "generic" or
# "none" = refused); cap: the extractor's; claim(st): the regime, from the per-pair quantities of ``pair_stats``.
def _spill_claim(st):
    m = st["m"]
    assert (m == FX_CANO).any() and (m == FX_CANO + 1).any() and (m >= 14399).any()
    assert ((m > 0) & (m <= FX_CANO)).any()


def _tile_claim(st):
    assert st["T"].max() >= 2040 and st["T"].max() <= FX_TCAP and (st["m"] > FX_CANO).any()


def _fills_cap(st):
    assert (st["nu"] == st["cap"]).any() and (st["nv"] == st["cap"]).any()


def _words_claim(n):
    def claim(st):
        assert st["words"] == (n + 31) // 32 and st["nu"][0] == n and st["nv"][0] == n and st["nu"][1] == n - 1
    return claim


def _classes_claim(R):
    def claim(st):
        assert any(len(np.unique(s["r"])) == R for s in st["subs"]), "a subgraph holding every rating class"
    return claim


def _targets_claim(st):
    assert (st["m"] == 0).any() and (st["nu"] == 1).any() and (st["nv"] == 1).any()
    assert st["rated"].any() and (~st["rated"]).any()


def _sampling_claim(st):
    # hop-1 candidates per side: the target excluded
    du, dv = st["du"], st["dv"]
    assert ((du >= 1) & (du <= 3) & (st["nu"] == 1)).any() and ((dv >= 1) & (dv <= 3) & (st["nv"] == 1)).any()


def _mnph_claim(st):
    du, dv = st["du"], st["dv"]
    assert ((dv == 20) & (st["nv"] == 21)).any() and ((dv == 21) & (st["nv"] == 21)).any()
    assert ((du == 20) & (st["nu"] == 21)).any() and ((du == 21) & (st["nu"] == 21)).any()


def _long_claim(st):
    assert (st["du"] >= 4096).any() and (st["nu"] == 101).any()


def _long_row_claim(st):
    _long_claim(st)
    assert (st["dv"] >= 4096).any() and (st["nv"] == 101).any()


def _none(st):
    pass


CASES = {
    # shared-memory limit of the one-launch path
    "smem_r5_items1000_cap224": dict(build=lambda: g_dense(230, 5, 1000), mnph=223, cap=224, path="fast",
                                     claim=_fills_cap),
    "smem_r5_items1000_cap225": dict(build=lambda: g_dense(230, 5, 1000), mnph=224, cap=225, path="generic",
                                     claim=_fills_cap),
    "smem_r12_cap140": dict(build=lambda: g_dense(150, 12, 1000), mnph=139, cap=140, path="fast", claim=_fills_cap),
    "smem_r12_cap141": dict(build=lambda: g_dense(150, 12, 1000), mnph=140, cap=141, path="generic", claim=_fills_cap),
    "smem_r5_ml1m_items_cap206": dict(build=lambda: g_dense(215, 5, 3706), mnph=205, cap=206, path="fast",
                                      claim=_fills_cap),
    "smem_r5_ml1m_items_cap207": dict(build=lambda: g_dense(215, 5, 3706), mnph=206, cap=207, path="generic",
                                      claim=_fills_cap),
    # canonical edges: 12 288 in shared memory, 12 289 and 14 399 spilled, small subgraphs around them
    "canonical_spill": dict(build=lambda: (g_mixed()[0], mixed_pairs("spill"), g_mixed()[1]), mnph=None, cap=121,
                            path="fast", claim=_spill_claim),
    # tile table: cap * longest row just under / over 128 * 2 048
    "tile_table_under": dict(build=lambda: g_tile(0), mnph=221, cap=222, path="fast", claim=_tile_claim),
    "tile_table_over": dict(build=lambda: g_tile(1), mnph=221, cap=222, path="generic", claim=_tile_claim),
    # ballot split by rating
    "classes_r1": dict(build=lambda: g_classes(1), mnph=None, cap=None, path="fast", claim=_classes_claim(1)),
    "classes_r32": dict(build=lambda: g_classes(32), mnph=None, cap=None, path="fast", claim=_classes_claim(32)),
    "classes_r33": dict(build=lambda: g_classes(33), mnph=None, cap=None, path="generic", claim=_classes_claim(33)),
    # catalogue limits of the generic path
    "items_h1_111836": dict(build=lambda: g_items(111836), mnph=None, cap=201, path="generic", claim=_none),
    "items_h1_111837": dict(build=lambda: g_items(111837), mnph=None, cap=201, path="none", claim=_none),
    "h2_35324": dict(build=lambda: g_h2(35324), mnph=10, h=2, cap=21, path="generic", claim=_none),
    "h2_35325": dict(build=lambda: g_h2(35325), mnph=10, h=2, cap=21, path="none", claim=_none),
    # sampling
    "sampling_ratio_zero": dict(build=lambda: (g_mixed()[0], mixed_pairs("sampling"), g_mixed()[1]), mnph=None,
                                ratio=0.3, cap=121, path="fast", claim=_sampling_claim),
    "sampling_mnph_edges": dict(build=lambda: (g_mixed()[0], mixed_pairs("sampling"), g_mixed()[1]), mnph=20,
                                cap=21, path="fast", claim=_mnph_claim),
    "sampling_long_column": dict(build=lambda: g_long(False), mnph=100, cap=101, path="fast", claim=_long_claim),
    "sampling_long_row": dict(build=lambda: g_long(True), mnph=100, cap=101, path="generic", claim=_long_row_claim),
    # targets
    "targets": dict(build=lambda: (g_mixed()[0], mixed_pairs("targets"), g_mixed()[1]), mnph=None, cap=121,
                    path="fast", claim=_targets_claim),
    "b256_every_kind": dict(build=lambda: (g_mixed()[0], mixed_pairs("b256"), g_mixed()[1]), mnph=None, cap=121,
                            path="fast", claim=lambda st: (_spill_claim(st), _targets_claim(st))),
}
for _n in (31, 32, 33, 64, 65):
    CASES["words_%d" % _n] = dict(build=functools.partial(g_words, _n), mnph=None, cap=_n, path="fast",
                                  claim=_words_claim(_n))


def case_args(c):
    return c.get("h", 1), c.get("ratio", 1.0), c["mnph"]


# ---- rating sessions -----------------------------------------------------------------------------------------------
def _session_tile(longest):
    """tile-table graph: a new user with an empty row and user 5 as it is; ``longest``: user 3 rates one more item
    (1 181: past the tile table, the batch moves to the generic path)"""
    A, _, cv = g_tile(0)
    users = [222, 5, 3] if longest else [222, 5]
    extra = int(np.setdiff1d(np.arange(1200), A[3].indices)[0])
    edits = ([2], [extra], [3]) if longest else ((), (), ())
    pairs = [(0, 0), (0, 7), (1, 0), (1, 30)] + ([(2, 0), (2, extra), (2, 1)] if longest else [])
    return A, cv, users, edits, pairs


def _session_spill():
    """spill graph: a new user with an empty row, and B1's corner user rating 38 sparse items more (a row of 150, the
    longest: cap 121 -> 151) - its pair at the block corner has 12 326 edges"""
    A, cv = g_mixed()
    add = np.arange(MIX_SP_V, MIX_SP_V + 38)
    users = [MIX_SHAPE[0], MIX_B1, MIX_SP_U]
    edits = (np.ones(38, np.int64), add, np.full(38, 2))
    pairs = [(0, MIX_B1), (0, MIX_SP_V), (1, MIX_B1), (1, MIX_SP_V + 3), (1, MIX_B1 + 9), (2, MIX_SP_V + 1),
             (2, MIX_B2)]
    return A, cv, users, edits, pairs


SESSION_CASES = {
    "session_tile_table_under": dict(build=lambda: _session_tile(False), mnph=221, cap=222, row_deg=1180, path="fast"),
    "session_tile_table_over": dict(build=lambda: _session_tile(True), mnph=221, cap=222, row_deg=1181,
                                    path="generic"),
    "session_spill": dict(build=_session_spill, mnph=None, cap=151, row_deg=150, path="fast"),
}


def session_rows(A, users, edits):
    """per session the dict item -> value (label + 1) of its user's row after its edits"""
    A = ssp.csr_matrix(A)
    out = []
    for s, u in enumerate(users):
        d = {}
        if u < A.shape[0]:
            d = {int(c): int(round(x)) for c, x in zip(A[u].indices, A[u].data)}
        for ss, it, x in zip(*edits):
            if ss == s:
                if x > 0:
                    d[int(it)] = int(x)
                else:
                    d.pop(int(it), None)
        out.append(d)
    return out


def graph_with_row(A, u, row):
    """A with user u's row replaced by ``row`` (item -> value), grown to hold u"""
    coo = ssp.coo_matrix(A)
    keep = coo.row != u
    r = np.r_[coo.row[keep], np.full(len(row), u)]
    c = np.r_[coo.col[keep], np.array(list(row.keys()), np.int64)]
    d = np.r_[coo.data[keep], np.array(list(row.values()), np.float64)]
    return ssp.csr_matrix((d.astype(np.float32), (r, c)), shape=(max(A.shape[0], u + 1), A.shape[1]))


# ---- the oracle and the comparison ---------------------------------------------------------------------------------
def oracle_batch(graphs, pu, pv, pl, cv, h, ratio, mnph, pids):
    """``extract_np.extract_batch`` with the hash sampler; ``graphs``: one RatingCSR, or one per pair (sessions: the
    graph with that pair's session applied)"""
    if isinstance(graphs, extract_np.RatingCSR):
        ob = extract_np.extract_batch(graphs, pu, pv, pl, cv, h, ratio, mnph, seed=SEED, pair_ids=pids)
        graphs = [graphs] * len(pu)
    else:
        subs, gs = [], []
        for k in range(len(pu)):
            sub = extract_np.extract_subgraph(graphs[k], pu[k], pv[k], h, ratio, mnph, seed=SEED,
                                              pair_id=int(pids[k]))
            subs.append(sub)
            gs.append(extract_np.construct_graph(sub, cv[int(pl[k])], h))
        ob = extract_np.collate(gs)
        ob["subs"] = subs
    ob["graphs"] = graphs
    return ob


def pair_stats(ob, pu, pv, cap):
    """per pair: m (edges), the user-row entries D of its user nodes and the tile count ceil(D / 128), side sizes,
    hop-1 candidates per side (target excluded) and whether the target is rated; cap and bitmap words"""
    st = dict(m=[], D=[], nu=[], nv=[], du=[], dv=[], rated=[], subs=ob["subs"], cap=cap, words=(cap + 31) // 32)
    for k, s in enumerate(ob["subs"]):
        g = ob["graphs"][k]
        rows, rated = g.row(int(pu[k]))[0], int(pv[k]) in set(g.row(int(pu[k]))[0].tolist())
        st["m"].append(len(s["u"]))
        st["D"].append(int(np.diff(g.indptr)[s["u_nodes"]].sum()))
        st["nu"].append(len(s["u_nodes"]))
        st["nv"].append(len(s["v_nodes"]))
        st["du"].append(len(g.col(int(pv[k]))) - rated)
        st["dv"].append(len(rows) - rated)
        st["rated"].append(rated)
    for k in ("m", "D", "nu", "nv", "du", "dv", "rated"):
        st[k] = np.asarray(st[k])
    st["T"] = (st["D"] + FX_TILE - 1) // FX_TILE
    return st


def expected_private(ob):
    """graph offsets, counts, graph_nu, node_gid and the message-passing lists of the oracle's batch: every node's
    in-edges sorted by (rating, local source), packed src | rating << 16, ``adj_eid`` = the edge's position in the
    batch, ``adj_in_ptr`` global (the layout of the static store)"""
    subs = ob["subs"]
    n = np.array([len(s["u_nodes"]) + len(s["v_nodes"]) for s in subs], np.int64)
    e = np.array([2 * len(s["u"]) for s in subs], np.int64)
    node_ptr, edge_ptr = np.r_[0, np.cumsum(n)], np.r_[0, np.cumsum(e)]
    N, E = int(node_ptr[-1]), int(edge_ptr[-1])
    src, dst = ob["edge_index"]
    et = ob["edge_type"]
    loc = src - node_ptr[ob["batch"][src]] if E else src
    order = np.lexsort((loc, et, dst))
    return dict(counts=np.array([N, E]), node_ptr=node_ptr, edge_ptr=edge_ptr,
                graph_nu=np.array([len(s["u_nodes"]) for s in subs]),
                node_gid=np.concatenate([np.r_[s["u_nodes"], s["v_nodes"]] for s in subs]),
                adj_in_ptr=np.r_[0, np.cumsum(np.bincount(dst, minlength=N))],
                adj_in=loc[order] | (et[order] << 16), adj_eid=order)


def assert_batch_matches(b, ob, tag):
    b.check()
    res = batch_equal(b, ob)
    assert all(res.values()), (tag, res)
    want = expected_private(ob)
    B = len(ob["subs"])
    N, E = (int(x) for x in want["counts"])
    p, adj = b._priv, b._adj[1]
    got = dict(counts=p["counts"], node_ptr=p["node_ptr"][:B + 1], edge_ptr=p["edge_ptr"][:B + 1],
               graph_nu=p["graph_nu"][:B], node_gid=b.node_gid, adj_in_ptr=adj["adj_in_ptr"][:N + 1],
               adj_in=adj["adj_in"][:E], adj_eid=adj["adj_eid"][:E])
    for k, w in want.items():
        g = got[k].cpu().numpy().astype(np.int64)
        assert np.array_equal(g, w), (tag, k, int(np.argmax(g != w)) if g.shape == w.shape else (g.shape, w.shape))


def _side(plan):
    return "fast" if plan > 0 else "generic" if plan == 0 else "none"


# ---- the tests -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_regime_vs_oracle(name):
    from igmc_b200.util_functions import RatingGraph, SubgraphExtractor
    c = CASES[name]
    A, (pu, pv, pl), cv = c["build"]()
    h, ratio, mnph = case_args(c)
    B = len(pu)
    G = RatingGraph(A)
    og = extract_np.RatingCSR(A)
    ob = None
    for fast in (True, False):
        ex = SubgraphExtractor(G, pu, pv, pl, cv, h, ratio, mnph, max_batch=B, seed=SEED, fast=fast)
        if c["cap"] is not None:
            assert ex.cap == c["cap"], (name, ex.cap)
        plan = ex.plan(B)
        want = c["path"] if fast or c["path"] == "none" else "generic"
        assert _side(plan) == want, (name, fast, plan)
        if want == "none":
            with pytest.raises(RuntimeError, match="code -3"):
                ex.extract(idx=np.arange(B))
            assert int(ex.err.item()) == 0
            continue
        if ob is None:
            ob = oracle_batch(og, pu, pv, pl, cv, h, ratio, mnph, np.arange(B))
            c["claim"](pair_stats(ob, pu, pv, ex.cap))
        assert_batch_matches(ex.extract(idx=np.arange(B)), ob, (name, fast))


@pytest.mark.parametrize("fast", [True, False])
def test_batch_sizes_through_one_workspace(fast):
    """B = 1 and ragged batch sizes through one workspace (the one-launch flags re-armed between launches), then
    B = 256 mixing every subgraph kind of the mixed graph"""
    from igmc_b200.util_functions import RatingGraph, SubgraphExtractor
    A, cv = g_mixed()
    og = extract_np.RatingCSR(A)
    pu, pv, pl = mixed_pairs("b256")
    ex = SubgraphExtractor(RatingGraph(A), pu, pv, pl, cv, 1, 1.0, None, max_batch=64, seed=SEED, fast=fast)
    for lo, nb in ((0, 1), (1, 3), (4, 64), (68, 17), (85, 1), (86, 256 - 86)):
        idx = np.arange(lo, lo + nb)
        assert _side(ex.plan(nb)) == ("fast" if fast else "generic")
        ob = oracle_batch(og, pu[idx], pv[idx], pl[idx], cv, 1, 1.0, None, idx)
        assert_batch_matches(ex.extract(idx=idx), ob, (fast, lo, nb))
    ob = oracle_batch(og, pu, pv, pl, cv, 1, 1.0, None, np.arange(256))
    _spill_claim(pair_stats(ob, pu, pv, ex.cap))
    assert_batch_matches(ex.extract(idx=np.arange(256)), ob, (fast, 256))


@pytest.mark.parametrize("name", sorted(SESSION_CASES))
def test_session_regime_vs_oracle(name):
    """session mode on both paths: an empty session row, and a session row that is the longest row (it moves cap and
    the plan through serve_sessions); the oracle runs on the graph with each session's edits applied"""
    import torch
    from igmc_b200 import recommend as rc
    from igmc_b200.util_functions import RatingGraph, SubgraphExtractor
    c = SESSION_CASES[name]
    A, cv, users, edits, pairs = c["build"]()
    G = RatingGraph(A)
    sess = rc.RatingSessions(G, users, *edits)
    rows = session_rows(A, users, edits)
    assert sess.max_row_deg == c["row_deg"] == max(len(r) for r in rows)
    assert any(len(r) == 0 for r in rows)
    s_of = np.array([p[0] for p in pairs], np.int32)
    pu = np.array([users[s] for s in s_of], np.int64)
    pv = np.array([p[1] for p in pairs], np.int64)
    As = [graph_with_row(A, u, r) for u, r in zip(users, rows)]
    ogs = [extract_np.RatingCSR(a) for a in As]
    lab = np.array([max(int(round(As[s][u, v])) - 1, 0) for s, u, v in zip(s_of, pu, pv)], np.int64)
    pid = pu * A.shape[1] + pv
    ob = oracle_batch([ogs[s] for s in s_of], pu, pv, lab, cv, 1, 1.0, c["mnph"], pid)
    B = len(pu)
    for fast in (True, False):
        ex = SubgraphExtractor(G, [0], [0], [0], cv, 1, 1.0, c["mnph"], max_batch=B, seed=SEED, fast=fast)
        before = ex.plan(B)
        ex.serve_sessions(sess.max_row_deg)
        plan = ex.plan(B)
        assert ex.cap == c["cap"], (name, ex.cap)
        assert _side(plan) == (c["path"] if fast else "generic"), (name, fast, plan)
        if fast:
            assert before > 0
            if c["row_deg"] > G.max_row_deg:
                assert plan != before     # the session row moved cap or the path
            st = pair_stats(ob, pu, pv, ex.cap)
            if "spill" in name:
                assert (st["m"] > FX_CANO).any() and st["nv"].max() == 150
            else:
                assert st["T"].max() >= 2040
        b = ex.extract(pairs=(pu, pv, lab), pair_ids=pid, sessions=sess, sess=torch.as_tensor(s_of))
        assert_batch_matches(b, ob, (name, fast))
