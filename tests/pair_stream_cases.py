"""Cases for the inference path's pair-stream kernels, and their brute-force enumerations.

The pair-stream kernels decide which (user, item) pair each batch slot scores and where its result lands.  The
references here are written from the contracts in include/igmc_b200.h by plain enumeration, not taken from the host
twins in igmc_b200/recommend.py:
  igmc_candidate_plan / _lists   the candidate set of query slot j is sorted(set(cand or range(num_items)) - row(u))
                                 (per-user lists: the row's ids in [0, num_items), deduplicated); user_off is the
                                 prefix of the set sizes, rated_pos the positions in cand of the user's rated items
  igmc_candidate_pairs           positions in query-slot order, then item order; pair_id = u * num_items + v as a
                                 Python int; positions past P repeat the last pair with tag -1; cursor += B
  igmc_session_pairs             sess = the session index (0 when out of range), u = users[sess], pair_id = u *
                                 num_items + v
  igmc_explain_count / _offsets  num_edges[tag] = E / 2 for tag >= 0; offsets = the exclusive prefix in Python ints
  igmc_occlusion_pairs           position c belongs to the last q with offsets[q] <= c (a linear scan), j = c -
                                 offsets[q]; invalid pair ids give (0, 0)
  igmc_occlusion_mask            edge_keep all ones except edge_ptr[g] + j and edge_ptr[g] + E_g/2 + j of every graph
                                 with tag >= 0 and 0 <= j < E_g/2; the rating's (user, item, label) at position tag
  igmc_edge_grad_scatter         numpy float32, one operation at a time: k = 0 stores g_a + g_b, k > 0 adds it to the
                                 stored value, k = K - 1 divides by K
Every case claims the regimes it is built to reach; ``REGIMES[kernel](case)`` re-derives them from the case's data
alone (tests/test_pair_stream_cases.py on the host, and the GPU test before it compares), so a case that silently stops
reaching a chunk boundary fails.  The launch constants those regimes depend on are restated below and checked against
the sources."""
import functools

import numpy as np
import scipy.sparse as ssp

from tests.ranking_cases import palette

# launch constants the regimes depend on (checked against the constexprs by tests/test_pair_stream_cases.py)
PLAN_THREADS = 1024    # csrc/recommend.cu: `constexpr int PLAN_THREADS` - k_candidate_plan / k_lists_scan, one chunk
PAIR_THREADS = 512     # csrc/recommend.cu and csrc/explain.cu: `constexpr int PAIR_THREADS` - one stride of the pairs
LIST_THREADS = 256     # csrc/recommend.cu: `constexpr int LIST_THREADS` - one chunk of a k_lists_rows row
SCAN_THREADS = 512     # csrc/explain.cu: `constexpr int SCAN_THREADS` - one chunk of k_explain_offsets
MASK_THREADS = 256     # csrc/explain.cu: `constexpr int MASK_THREADS` - one stride of k_occlusion_mask / scatter
THREADS = 256          # csrc/session.cu: `constexpr int THREADS` - one block of k_session_pairs
CONSTANTS = {("recommend.cu", "PLAN_THREADS"): PLAN_THREADS, ("recommend.cu", "PAIR_THREADS"): PAIR_THREADS,
             ("recommend.cu", "LIST_THREADS"): LIST_THREADS, ("explain.cu", "SCAN_THREADS"): SCAN_THREADS,
             ("explain.cu", "PAIR_THREADS"): PAIR_THREADS, ("explain.cu", "MASK_THREADS"): MASK_THREADS,
             ("session.cu", "THREADS"): THREADS}

ERR_CANDIDATES = 7     # IGMC_ERR_CANDIDATES (csrc/common.cuh)
ID_MAX = 2 ** 31 - 1


# ---- rating graphs ------------------------------------------------------------------------------------------------------
def _csr(rows, ni, seed=0):
    """scipy CSR of the given item rows, labels 1..5 (stored value = label + 1)"""
    rng = np.random.default_rng(seed)
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    idx = np.concatenate([np.asarray(sorted(r), np.int64) for r in rows]) if rows else np.zeros(0, np.int64)
    data = rng.integers(1, 6, len(idx)).astype(np.float32)
    return ssp.csr_matrix((data, idx, indptr), shape=(len(rows), ni))


PLAN_NI, PLAN_NU = 300, 2600
# items of the shared candidate list: 120 of the 300, 0 and 299 among them
PLAN_LIST = np.unique(np.concatenate([[0, PLAN_NI - 1],
                                      np.random.default_rng(11).choice(PLAN_NI, 118, replace=False)]))[:120]
FULL_USERS = (0, 1, 2, 3, PLAN_NU - 1)     # rated every item
LISTED_USERS = (5, 6, 7, 8, 9)              # rated every listed item (and a few others)
DEG0_USERS = (4, 12, 13)


@functools.lru_cache(None)
def plan_graph():
    rng = np.random.default_rng(3)
    rows = []
    for u in range(PLAN_NU):
        if u in FULL_USERS:
            r = range(PLAN_NI)
        elif u in LISTED_USERS:
            r = set(PLAN_LIST.tolist()) | set(rng.choice(PLAN_NI, 5).tolist())
        elif u in DEG0_USERS:
            r = ()
        elif u == 10:
            r = (0, PLAN_NI - 1, 150)
        else:
            r = set(rng.choice(PLAN_NI, int(rng.integers(0, 31))).tolist())
        rows.append(list(r))
    return _csr(rows, PLAN_NI, 1)


def row(A, u):
    return A.indices[A.indptr[u]:A.indptr[u + 1]].astype(np.int64)


def plan_users(U):
    """U query slots: a full-row user first, a run of zero-candidate users in the middle (across the first chunk
    boundary when U > 1024), a full-row user last; zero-degree users, repeated users and users who rated every listed
    item between them"""
    rng = np.random.default_rng(U)
    others = [u for u in range(PLAN_NU) if u not in FULL_USERS + LISTED_USERS]
    body = list(rng.choice(others, U - 12))
    body[5:5] = [7, 8, 10, 10, 4]
    mid = min(U // 2, PLAN_THREADS - 2)
    body[mid:mid] = [1, 2, 3, 5, 6]               # zero candidates: full rows, then (shared list) every listed item
    return np.asarray([0] + body + [9, 9, 9, 9, PLAN_NU - 1], np.int64)


# ---- brute-force candidate enumeration ----------------------------------------------------------------------------------
def candidate_sets(A, users, cand, exclude):
    """per query slot the sorted candidate items: sorted(set(cand or range(num_items)) - row(u))"""
    ni = A.shape[1]
    base = set(range(ni)) if cand is None else set(int(x) for x in cand)
    out = []
    for u in users:
        s = base - set(row(A, int(u)).tolist()) if exclude else base
        out.append(sorted(s))
    return out


def list_sets(A, users, rows, exclude):
    """per query slot of igmc_candidate_lists: the row's ids in [0, num_items), without the user's rated ones"""
    ni = A.shape[1]
    out = []
    for u, r in zip(users, rows):
        s = set(int(x) for x in r if 0 <= x < ni)
        if exclude:
            s -= set(row(A, int(u)).tolist())
        out.append(sorted(s))
    return out


def corated_rows(A, users, m):
    """the candidate rows retrieve=m gives (igmc_corated_items with exclude_rated), by enumeration: paths[v] = the
    3-paths u - i - u' - v with u' != u, the user's rated items dropped, ordered by paths descending then item
    ascending, items without a path dropped, the rest of the row -1"""
    nu, ni = A.shape
    rated = [set(row(A, x).tolist()) for x in range(nu)]
    out = np.full((len(users), m), -1, np.int64)
    for j, u in enumerate(users):
        paths = {}
        for w in range(nu):
            if w == u:
                continue
            shared = len(rated[u] & rated[w])
            for v in rated[w]:
                paths[v] = paths.get(v, 0) + shared
        order = sorted((-n, v) for v, n in paths.items() if n > 0 and v not in rated[u])[:m]
        out[j, :len(order)] = [v for _, v in order]
    return out


def prefix(counts):
    """exclusive prefix in Python ints, [n + 1]"""
    off = [0]
    for c in counts:
        off.append(off[-1] + int(c))
    return np.asarray(off, np.int64)


def flat(lists):
    """the lists concatenated, int64"""
    return np.asarray([x for r in lists for x in r], np.int64)


def rated_positions(A, users, cand):
    """per slot the positions in cand of the user's rated items, ascending"""
    at = {int(x): p for p, x in enumerate(cand)}
    return [sorted(at[x] for x in row(A, int(u)).tolist() if x in at) for u in users]


def enumerate_positions(sets, users, ni):
    """(u, v, pair_id, tag) of every position in query-slot order, then item order"""
    u = np.concatenate([np.full(len(s), int(users[j]), np.int64) for j, s in enumerate(sets)] + [np.zeros(0, np.int64)])
    v = np.concatenate([np.asarray(s, np.int64) for s in sets] + [np.zeros(0, np.int64)])
    t = np.concatenate([np.full(len(s), j, np.int64) for j, s in enumerate(sets)] + [np.zeros(0, np.int64)])
    return u, v, u * ni + v, t


def batch_of(stream, pos, B, P):
    """the batch [pos, pos + B) of an enumerated stream: positions past P repeat the last one with tag -1"""
    c = pos + np.arange(B, dtype=np.int64)
    real = c < P
    c = np.where(real, c, P - 1)
    u, v, pid, t = (x[c] for x in stream)
    return u, v, pid, np.where(real, t, -1)


# ---- plan cases ---------------------------------------------------------------------------------------------------------
def plan_cases():
    cases = []
    for U in (700, 2700):
        for mode in ("no_list", "shared"):
            for exclude in (True, False):
                claims = {"mode:" + mode, "exclude" if exclude else "include", "deg0", "repeated_users",
                          "item0_rated", "itemlast_rated"}
                claims.add("U<=1024" if U <= PLAN_THREADS else "chunks>=3")
                if exclude:
                    claims |= {"zero_first", "zero_run_middle", "zero_last"}
                    claims.add("rated_every_item" if mode == "no_list" else "rated_every_listed")
                    if U > PLAN_THREADS:
                        claims.add("zero_across_chunk")
                cases.append(dict(kernel="plan", name="U=%d %s %s" % (U, mode, "excl" if exclude else "incl"),
                                  users=plan_users(U - 16), cand=PLAN_LIST if mode == "shared" else None,
                                  exclude=exclude, claims=claims))
    return cases


def plan_reference(case, A=None):
    """(user_off, rated_off or None, rated_pos or None, sets)"""
    A = plan_graph() if A is None else A
    sets = candidate_sets(A, case["users"], case["cand"], case["exclude"])
    user_off = prefix(len(s) for s in sets)
    if case["cand"] is None or not case["exclude"]:
        return user_off, None, None, sets
    rp = rated_positions(A, case["users"], case["cand"])
    return user_off, prefix(len(r) for r in rp), flat(rp), sets


def _zero_regimes(counts, chunk):
    got = set()
    counts = np.asarray(counts, np.int64)
    if len(counts) == 0:
        return got
    if counts[0] == 0:
        got.add("zero_first")
    if counts[-1] == 0:
        got.add("zero_last")
    z = counts == 0
    edges = np.flatnonzero(np.diff(np.concatenate([[0], z.astype(np.int8), [0]])))
    for a, b in zip(edges[::2], edges[1::2]):         # zero runs [a, b)
        if a > 0 and b < len(counts) and b - a >= 2:
            got.add("zero_run_middle")                # at least two, touching neither end
    if chunk and (z[chunk - 1:-1:chunk] & z[chunk::chunk]).any():      # a zero run over a chunk boundary
        got.add("zero_across_chunk")
    return got


def plan_regimes(case, A=None):
    A = plan_graph() if A is None else A
    users, cand, exclude = case["users"], case["cand"], case["exclude"]
    ni, U = A.shape[1], len(users)
    got = {"mode:" + ("no_list" if cand is None else "shared"), "exclude" if exclude else "include"}
    if U <= PLAN_THREADS:
        got.add("U<=1024")
    if U > 2 * PLAN_THREADS:
        got.add("chunks>=3")
    if len(set(users.tolist())) < U:
        got.add("repeated_users")
    rows = [set(row(A, int(u)).tolist()) for u in users]
    if any(len(r) == 0 for r in rows):
        got.add("deg0")
    if any(0 in r for r in rows):
        got.add("item0_rated")
    if any(ni - 1 in r for r in rows):
        got.add("itemlast_rated")
    if any(len(r) == ni for r in rows):
        got.add("rated_every_item")
    if cand is not None and any(set(cand.tolist()) <= r and len(r) < ni for r in rows):
        got.add("rated_every_listed")
    sets = candidate_sets(A, users, cand, exclude)
    return got | _zero_regimes([len(s) for s in sets], PLAN_THREADS)


# ---- per-user list cases (igmc_candidate_lists) ------------------------------------------------------------------------
def _list_rows(U, width, seed):
    """[U, width] int32 rows of random ids in [-1, num_items), a third of each row repeating its first id"""
    rng = np.random.default_rng(seed)
    rows = rng.integers(-1, PLAN_NI, (U, width))
    rows = np.where(rng.random((U, width)) < 0.3, rows[:, :1], rows)     # duplicates inside a row
    return rows.astype(np.int32)


def lists_case(name, U, width, exclude, seed, special=True, bad=False):
    users = plan_users(U - 16)
    rows = _list_rows(len(users), width, seed)
    A = plan_graph()
    if special and len(users) >= 4:
        rows[0] = -1                                              # all empty
        rows[len(users) - 1] = rows[len(users) - 1, 0] if rows[len(users) - 1, 0] >= 0 else 7   # all one id
        r = row(A, int(users[1]))                                 # only items the user rated
        if len(r):
            rows[1] = np.resize(r, width)
        rows[2] = np.resize(np.arange(PLAN_NI - 1, -1, -1), width)          # descending, item 0 and 299
    if bad:                                                       # ids >= num_items and < -1 next to valid ones
        U = len(users)
        rows[1, 0], rows[1, width - 1] = PLAN_NI, -2
        rows[U - 2, width // 2] = 2 ** 31 - 1
        rows[U // 2, 0] = -(2 ** 31)
    claims = {"exclude" if exclude else "include"}
    if width in (1, 255, 256, 257):
        claims.add("width=%d" % width)
    if width > 4 * LIST_THREADS:
        claims.add("width>1024")
    if len(users) > PLAN_THREADS:
        claims.add("U>1024")
    if special:
        claims |= {"row_all_empty", "row_all_dup", "zero_first"}
        if exclude:         # full-row users 1, 2, 3 in the middle and last: their rows are empty after exclusion
            claims |= {"row_all_rated", "zero_run_middle", "zero_last"}
    if bad:
        claims.add("invalid_ids")
    return dict(kernel="lists", name=name, users=np.asarray(users, np.int64), rows=rows, exclude=exclude,
                claims=claims)


def lists_cases():
    cases = []
    for width in (1, 255, 256, 257, 1100):
        for exclude in (True, False):
            c = lists_case("w=%d %s" % (width, "excl" if exclude else "incl"), 40, width, exclude, width,
                           special=width > 1)
            cases.append(c)
    cases.append(lists_case("U=1100 w=5 excl", 1100 + 16, 5, True, 5))
    cases.append(lists_case("U=1100 w=3 incl", 1100 + 16, 3, False, 3))
    cases.append(lists_case("invalid ids w=300", 40, 300, True, 8, bad=True))
    cases.append(lists_case("invalid ids U=1100", 1100 + 16, 4, False, 9, bad=True))
    return cases


def lists_reference(case, A=None):
    """(user_off, lists, err): the compact lists and the error the ids set"""
    A = plan_graph() if A is None else A
    sets = list_sets(A, case["users"], case["rows"], case["exclude"])
    ni = A.shape[1]
    bad = bool(((case["rows"] < -1) | (case["rows"] >= ni)).any())
    lists = flat(sets)
    return prefix(len(s) for s in sets), lists, ERR_CANDIDATES if bad else 0, sets


def lists_regimes(case, A=None):
    A = plan_graph() if A is None else A
    rows, users = case["rows"], case["users"]
    U, width = rows.shape
    ni = A.shape[1]
    got = {"exclude" if case["exclude"] else "include"}
    if width in (1, 255, 256, 257):
        got.add("width=%d" % width)
    if width > 4 * LIST_THREADS:
        got.add("width>1024")
    if U > PLAN_THREADS:
        got.add("U>1024")
    if (rows == -1).all(1).any():
        got.add("row_all_empty")
    if width > 1 and any((r == r[0]).all() and 0 <= r[0] < ni for r in rows):
        got.add("row_all_dup")
    if case["exclude"] and any(len(r) and set(r.tolist()) <= set(row(A, int(u)).tolist())
                               for r, u in zip(rows, users)):
        got.add("row_all_rated")
    if ((rows >= ni).any()) and (rows < -1).any():
        got.add("invalid_ids")
    sets = list_sets(A, users, rows, case["exclude"])
    return got | _zero_regimes([len(s) for s in sets], 0)


# ---- candidate pair cases -----------------------------------------------------------------------------------------------
SMALL_USERS = np.asarray([0, 4, 10, 11, 1, 2, 12, 14, 14, 9, 3], np.int64)    # zero candidates first, in a run, last
PAIR_BS = ((1, {"B=1"}), (511, {"B=511", "tail"}), (512, {"B=512", "tail"}), (513, {"B=513", "second_stride", "tail"}),
           (5000, {"B>P", "second_stride", "tail"}))                           # over SMALL_USERS (P < 5 000)
BIG_PAIR_BS = ((700, {"second_stride", "tail"}), (4096, {"second_stride", "tail"}))    # over 1 404 users
PAIR_PER_MODE = {"B=1", "B=511", "B=512", "B=513", "B>P", "second_stride", "tail"}     # each mode reaches all of them


def pairs_cases():
    """a run of igmc_candidate_pairs with the cursor walked from 0 in steps of B to one batch past the end"""
    cases = []
    rng = np.random.default_rng(21)
    big = plan_users(1400)
    for mode in ("no_list", "shared", "per_user", "explicit"):
        for exclude in ((True, False) if mode != "explicit" else (False,)):
            for users, Bs in ((SMALL_USERS, PAIR_BS), (big, BIG_PAIR_BS)):
                if mode == "explicit":
                    n = len(users) * 37
                    src = dict(pair_u=rng.integers(0, PLAN_NU, n), pair_v=rng.integers(0, PLAN_NI, n))
                elif mode == "per_user":
                    src = dict(users=users, rows=_list_rows(len(users), 70, len(users)))
                else:
                    src = dict(users=users, cand=PLAN_LIST if mode == "shared" else None)
                for B, b_claims in Bs:
                    claims = {"mode:" + mode, "exclude" if exclude else "include"} | b_claims
                    if exclude and mode != "explicit":      # full-row users first, in a run and last
                        claims |= {"zero_first", "zero_run_middle", "zero_last"}
                    cases.append(dict(kernel="pairs", name="%s %s U=%d B=%d" % (mode, "excl" if exclude else "incl",
                                                                                len(users), B),
                                      mode=mode, exclude=exclude, B=B, claims=claims, **src))
    return cases


def pairs_stream(case, A=None):
    """(P, enumerated stream, sets or None) of a pairs case"""
    A = plan_graph() if A is None else A
    ni = A.shape[1]
    if case["mode"] == "explicit":
        u, v = np.asarray(case["pair_u"], np.int64), np.asarray(case["pair_v"], np.int64)
        return len(u), (u, v, u * ni + v, np.arange(len(u), dtype=np.int64)), None
    if case["mode"] == "per_user":
        sets = list_sets(A, case["users"], case["rows"], case["exclude"])
    else:
        sets = candidate_sets(A, case["users"], case["cand"], case["exclude"])
    st = enumerate_positions(sets, case["users"], ni)
    return len(st[0]), st, sets


def pairs_regimes(case, A=None):
    P, _, sets = pairs_stream(case, A)
    B = case["B"]
    got = {"mode:" + case["mode"], "exclude" if case["exclude"] else "include"}
    if B in (1, 511, 512, 513):
        got.add("B=%d" % B)
    if B > P:
        got.add("B>P")
    if B > PAIR_THREADS:
        got.add("second_stride")
    if P % B:
        got.add("tail")
    if sets is not None:
        got |= _zero_regimes([len(s) for s in sets], 0)
    return got


# ---- session pair cases -------------------------------------------------------------------------------------------------
SESSION_NI = 5000


def session_cases():
    users = np.asarray([3, PLAN_NU + 5, 3, ID_MAX, 0, 1234567, PLAN_NU - 1, PLAN_NU, 17], np.int64)
    rng = np.random.default_rng(31)
    cases = []
    # ids below num_users, new ones, a shared one and 2^31 - 1: every pair id of a user >= 429 496 is past 2^31
    common = {"known_user", "new_user", "shared_id", "id=2^31-1", "pair_id>=2^31"}
    for name, B, bad, claims in (("B=700", 700, False, {"several_blocks"}), ("B=1", 1, False, {"B=1"}),
                                 ("B=513 out-of-range", 513, True, {"several_blocks", "session_out_of_range"})):
        s = rng.integers(0, len(users), B)
        if bad:
            s[[0, B // 2, B - 1]] = (len(users), -1, ID_MAX)
        v = rng.integers(0, SESSION_NI, B)
        c = dict(kernel="session", name=name, users=users, links_u=s.astype(np.int64), links_v=v.astype(np.int64),
                 num_items=SESSION_NI, num_users=PLAN_NU, claims=common | claims)
        cases.append(c)
    return cases


def session_reference(case):
    """(links_u, pair_id, sess, err)"""
    S = len(case["users"])
    s = np.asarray(case["links_u"], np.int64)
    ok = (s >= 0) & (s < S)
    sess = np.where(ok, s, 0)
    u = np.asarray(case["users"], np.int64)[sess]
    pid = np.asarray([int(a) * case["num_items"] + int(b) for a, b in zip(u, case["links_v"])], np.int64)
    return u, pid, sess, 0 if ok.all() else ERR_CANDIDATES


def session_regimes(case):
    users, B = np.asarray(case["users"], np.int64), len(case["links_u"])
    got = set()
    if (users < case["num_users"]).any():
        got.add("known_user")
    if (users >= case["num_users"]).any():
        got.add("new_user")
    if len(set(users.tolist())) < len(users):
        got.add("shared_id")
    if ID_MAX in users:
        got.add("id=2^31-1")
    if B > 2 * THREADS:
        got.add("several_blocks")
    if B == 1:
        got.add("B=1")
    s = np.asarray(case["links_u"])
    if ((s < 0) | (s >= len(users))).any():
        got.add("session_out_of_range")
    used = users[s[(s >= 0) & (s < len(users))]]
    if (used * case["num_items"] >= 2 ** 31).any():
        got.add("pair_id>=2^31")
    return got


# ---- explain count / offsets --------------------------------------------------------------------------------------------
def offsets_cases():
    rng = np.random.default_rng(41)
    cases = []
    for P in (1, 511, 512, 513):
        cases.append(dict(name="P=%d" % P, num_edges=rng.integers(0, 3000, P), claims={"P=%d" % P}))
    ne = rng.integers(1, 900, 5000)
    ne[:7] = 0
    ne[2000:2600] = 0            # a run of zero-count pairs across a 512-entry chunk boundary
    ne[4990:] = 0
    cases.append(dict(name="P=5000 zero runs", num_edges=ne,
                      claims={"P>4096", "zero_first", "zero_run_middle", "zero_across_chunk", "zero_last"}))
    cases.append(dict(name="total>=2^31", num_edges=np.asarray([0, ID_MAX, 5, 0], np.int64),
                      claims={"T>=2^31", "zero_first", "zero_last"}))
    ne = rng.integers(0, 10, 1300)
    ne[[3, 600, 1299]] = (ID_MAX, ID_MAX - 1, ID_MAX)
    cases.append(dict(name="total>=2^32 P=1300", num_edges=ne, claims={"T>=2^31", "T>=2^32"}))
    for c in cases:
        c["kernel"] = "offsets"
        c["num_edges"] = np.asarray(c["num_edges"], np.int64)
    return cases


def offsets_reference(case):
    return prefix(case["num_edges"])


def offsets_regimes(case):
    ne = case["num_edges"]
    P = len(ne)
    got = set()
    if P in (1, 511, 512, 513):
        got.add("P=%d" % P)
    if P > 8 * SCAN_THREADS:
        got.add("P>4096")
    total = sum(int(x) for x in ne)
    if total >= 2 ** 31:
        got.add("T>=2^31")
    if total >= 2 ** 32:
        got.add("T>=2^32")
    return got | _zero_regimes(ne, SCAN_THREADS)


def count_cases():
    """igmc_explain_count over a batch: graphs of even directed-edge counts, tags a permutation of some pairs and -1"""
    rng = np.random.default_rng(43)
    cases = []
    for B, P, claims in ((700, 900, {"several_blocks", "tag=-1", "zero_edges"}), (1, 3, set()),
                         (300, 300, {"several_blocks", "tag=-1", "zero_edges"})):
        E = 2 * rng.integers(0, 400, B)
        tag = rng.permutation(P)[:B].astype(np.int64)
        if B > 1:
            pair0 = tag[0]
            tag[rng.random(B) < 0.2] = -1
            tag[0], tag[1] = pair0, -1       # graph 0 has no edges and a pair; graph 1 is padding
            E[:3] = 0
        cases.append(dict(kernel="count", name="B=%d P=%d" % (B, P), edge_ptr=prefix(E), tag=tag, P=P,
                          claims=claims))
    return cases


def count_reference(case, sentinel):
    out = np.full(case["P"], sentinel, np.int64)
    E = np.diff(case["edge_ptr"])
    for i, t in enumerate(case["tag"]):
        if t >= 0:
            out[t] = E[i] // 2
    return out


def count_regimes(case):
    got = set()
    if (case["tag"] < 0).any():
        got.add("tag=-1")
    if len(case["tag"]) > THREADS:
        got.add("several_blocks")
    if (np.diff(case["edge_ptr"])[case["tag"] >= 0] == 0).any():
        got.add("zero_edges")
    return got


# ---- occlusion pairs ----------------------------------------------------------------------------------------------------
def occl_cases():
    rng = np.random.default_rng(51)
    cases = []
    ne = rng.integers(1, 60, 80)
    ne[:3] = 0
    ne[30:36] = 0
    ne[77:] = 0
    pu, pv = rng.integers(0, PLAN_NU, 80), rng.integers(0, PLAN_NI, 80)
    zeros = {"zero_first", "zero_run_middle", "zero_last", "tail"}
    for B, claims in ((1, {"B=1"}), (513, {"second_stride"}), (700, {"second_stride"}), (5000, {"second_stride"})):
        cases.append(dict(name="zero runs B=%d" % B, num_edges=ne, pair_u=pu, pair_v=pv, B=B, cursors=None,
                          claims=zeros | claims))
    bu, bv = pu.copy(), pv.copy()
    bu[10], bv[40], bu[76] = PLAN_NU, -3, -1
    cases.append(dict(name="invalid ids B=600", num_edges=ne, pair_u=bu, pair_v=bv, B=600, cursors=None,
                      claims=zeros | {"second_stride", "invalid_ids"}))
    # T just below 2^31 - 1: 2 100 pairs of about 10^6 ratings; only the last batches and one past the end run
    ne = rng.integers(1_000_000, 1_045_000, 2100)
    ne[-1] = 0
    ne[5:9] = 0
    ne[-2] = ne[-2] + (ID_MAX - 2 - int(ne.sum()))
    T = int(ne.sum())
    pu, pv = rng.integers(0, PLAN_NU, 2100), rng.integers(0, PLAN_NI, 2100)
    B = 700
    cases.append(dict(name="T=2^31-3 B=700", num_edges=ne, pair_u=pu, pair_v=pv, B=B,
                      cursors=(T - 2 * B, T - B, T, 2 ** 31 - 1000, int(prefix(ne)[1000]) - 350),
                      claims={"T~2^31", "second_stride", "tail", "zero_run_middle", "zero_last"}))
    for c in cases:
        c["kernel"] = "occl"
        c["num_edges"] = np.asarray(c["num_edges"], np.int64)
    return cases


def owner_linear(offsets, c):
    """the last q in [0, P) with offsets[q] <= c, by a linear scan (vectorised over c)"""
    P = len(offsets) - 1
    q = np.arange(P)
    return np.max(np.where(offsets[None, :P] <= np.asarray(c, np.int64)[:, None], q[None, :], -1), axis=1)


def occl_batch(case, pos, ni=PLAN_NI, nu=PLAN_NU):
    """(u, v, pair_id, tag, j, bad) of the positions [pos, pos + B)"""
    off = offsets_reference(case)
    T = int(off[-1])
    c = pos + np.arange(case["B"], dtype=np.int64)
    real = c < T
    c = np.where(real, c, T - 1)
    q = owner_linear(off, c)
    u, v = np.asarray(case["pair_u"], np.int64)[q], np.asarray(case["pair_v"], np.int64)[q]
    bad = (u < 0) | (u >= nu) | (v < 0) | (v >= ni)
    u, v = np.where(bad, 0, u), np.where(bad, 0, v)
    return u, v, u * ni + v, np.where(real, c, -1), c - off[q], bool(bad.any())


def occl_cursors(case):
    if case["cursors"] is not None:
        return list(case["cursors"])
    T = int(offsets_reference(case)[-1])
    return list(range(0, T + case["B"], case["B"]))


def occl_regimes(case):
    ne = case["num_edges"]
    off = offsets_reference(case)
    T, B = int(off[-1]), case["B"]
    got = _zero_regimes(ne, 0)
    if B > PAIR_THREADS:
        got.add("second_stride")
    if B == 1:
        got.add("B=1")
    curs = occl_cursors(case)
    if any(p < T < p + B for p in curs) or any(p >= T for p in curs):
        got.add("tail")
    if T >= 2 ** 31 - 8 and any(p + B > 2 ** 31 - 16 for p in curs):
        got.add("T~2^31")
    pu, pv = np.asarray(case["pair_u"]), np.asarray(case["pair_v"])
    if ((pu < 0) | (pu >= PLAN_NU) | (pv < 0) | (pv >= PLAN_NI)).any():
        got.add("invalid_ids")
    return got


# ---- occlusion mask and gradient scatter: a synthetic extracted batch --------------------------------------------------
def synthetic_batch(ms, seed, slack=37):
    """graphs with ms[g] ratings in the [u|v ; v|u] layout: edge_ptr [B+1], edge_index [2, edge_cap] (row stride
    edge_cap > edge_ptr[B]), edge_type [edge_cap], node_gid [N], node_ptr"""
    rng = np.random.default_rng(seed)
    B = len(ms)
    edge_ptr = prefix(2 * np.asarray(ms, np.int64))
    E = int(edge_ptr[-1])
    cap = E + slack
    ei = np.full((2, cap), -5, np.int64)
    et = np.full(cap, 99, np.int64)
    gids, n0 = [], 0
    for g, m in enumerate(ms):
        nu_, nv_ = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        a = n0 + rng.integers(0, nu_, m)
        b = n0 + nu_ + rng.integers(0, nv_, m)
        e0 = int(edge_ptr[g])
        ei[0, e0:e0 + m], ei[1, e0:e0 + m] = a, b
        ei[0, e0 + m:e0 + 2 * m], ei[1, e0 + m:e0 + 2 * m] = b, a
        lab = rng.integers(0, 5, m)
        et[e0:e0 + m] = et[e0 + m:e0 + 2 * m] = lab
        gids.append(rng.integers(0, 10 ** 6, nu_))
        gids.append(rng.integers(0, 10 ** 6, nv_) + 2 * 10 ** 6)
        n0 += nu_ + nv_
    return dict(edge_ptr=edge_ptr, edge_index=ei, edge_type=et, node_gid=np.concatenate(gids).astype(np.int64),
                edge_cap=cap)


MASK_MS = (0, 1, 255, 256, 257, 1100, 3, 0, 40, 2)


def mask_cases():
    cases = []
    ms = MASK_MS
    B = len(ms)
    # tag = the position c; T covers them; tag -1 on the zero-rating graphs and one more
    T = 5000
    tag = np.asarray([-1, 10, 4000, 300, 301, 2, -1, -1, 4999, 0], np.int64)
    j = np.asarray([0, 0, 254, 0, 256, 1099, 1, 0, 39, 1], np.int64)
    sizes = {"m=0", "m=1", "m=255", "m=256", "m=257", "m>1024", "edge_cap>E", "tag=-1", "drop_past_first_stride"}
    cases.append(dict(name="clean", ms=ms, tag=tag, j=j, T=T, claims=sizes))
    j2 = j.copy()
    j2[2], j2[8] = 255, -1                       # outside the graph: error, nothing dropped
    t2 = tag.copy()
    t2[7] = 77                                   # a zero-rating graph with a position: error too
    cases.append(dict(name="j outside", ms=ms, tag=t2, j=j2, T=T, claims=sizes | {"j_outside"}))
    for c in cases:
        c["kernel"] = "mask"
        c["batch"] = synthetic_batch(c["ms"], 61)
    return cases


def mask_reference(case, sentinel):
    """(edge_keep [E], user, item, rating [T] with `sentinel` where nothing is written, err)"""
    bt = case["batch"]
    ep, ei, et, gid = bt["edge_ptr"], bt["edge_index"], bt["edge_type"], bt["node_gid"]
    keep = np.ones(int(ep[-1]), np.uint8)
    rec = np.full((3, case["T"]), sentinel, np.int64)
    err = 0
    for g in range(len(ep) - 1):
        m = int(ep[g + 1] - ep[g]) // 2
        c, j = int(case["tag"][g]), int(case["j"][g])
        if c < 0:
            continue
        if not 0 <= j < m:
            err = ERR_CANDIDATES
            continue
        a = int(ep[g]) + j
        keep[a] = keep[a + m] = 0
        rec[:, c] = (gid[ei[0, a]], gid[ei[1, a]], et[a])
    return keep, rec, err


def mask_regimes(case):
    ms, tag, j = np.asarray(case["ms"]), case["tag"], case["j"]
    got = set()
    for m in (0, 1, 255, 256, 257):
        if m in ms:
            got.add("m=%d" % m)
    if (ms > 4 * MASK_THREADS).any():
        got.add("m>1024")
    if case["batch"]["edge_cap"] > case["batch"]["edge_ptr"][-1]:
        got.add("edge_cap>E")
    if (tag < 0).any():
        got.add("tag=-1")
    if ((tag >= 0) & ((j < 0) | (j >= ms))).any():
        got.add("j_outside")
    # a dropped edge in a later stride of the CTA: j or j + m at or past MASK_THREADS
    if ((tag >= 0) & (j < ms) & (j + ms >= MASK_THREADS)).any():
        got.add("drop_past_first_stride")
    return got


def scatter_cases():
    cases = []
    ms = MASK_MS
    # pair q of each graph; its count is the graph's (offsets of P = 14 pairs, 4 absent from the batch)
    q = np.asarray([-1, 3, 0, 12, 5, 7, 9, 1, -1, 13], np.int64)
    for K, pal in ((1, "signed_zero"), (2, "nan"), (3, "subnormal"), (3, "inf"), (2, "near_one"), (1, "random")):
        for bad in (False, True):
            if bad and K == 1 and pal == "random":
                continue
            counts = np.asarray([6, 0, 0, 4, 0, 0, 0, 0, 0, 0, 11, 0, 0, 0], np.int64)
            for g, p in enumerate(q):
                if p >= 0:
                    counts[p] = ms[g]
            if bad:
                counts[7] += 1                   # graph 5 (1100 ratings) disagrees with its base count
                counts[0] -= 1                   # graph 2 (255) too
            c = dict(kernel="scatter", name="K=%d %s%s" % (K, pal, " offsets disagree" if bad else ""), ms=ms,
                     tag=q, K=K, palette=pal, offsets=prefix(counts), seed=K * 7 + len(pal),
                     claims={"K=%d" % K, "palette:" + pal, "tag=-1", "m>1024"} | ({"offsets_disagree"} if bad else set()))
            c["batch"] = synthetic_batch(ms, 71)
            cases.append(c)
    return cases


def scatter_grads(case):
    """edge_grad [K, edge_cap] from the case's palette (ragged past edge_ptr[B])"""
    rng = np.random.default_rng(case["seed"])
    cap = case["batch"]["edge_cap"]
    return np.stack([palette(case["palette"], cap, rng) for _ in range(case["K"])]).astype(np.float32)


def scatter_reference(case, grads, sentinel_f, sentinel_i):
    """(out [T] after every checkpoint k = 0..K-1 (a list), user/item/rating [3, T], err)"""
    bt = case["batch"]
    ep, ei, et, gid = bt["edge_ptr"], bt["edge_index"], bt["edge_type"], bt["node_gid"]
    off = case["offsets"]
    T, K = int(off[-1]), case["K"]
    out = np.full(T, sentinel_f, np.float32)
    rec = np.full((3, T), sentinel_i, np.int64)
    err, outs = 0, []
    with np.errstate(all="ignore"):
        for k in range(K):
            for g in range(len(ep) - 1):
                q = int(case["tag"][g])
                if q < 0:
                    continue
                e0, m = int(ep[g]), int(ep[g + 1] - ep[g]) // 2
                o = int(off[q])
                if int(off[q + 1]) - o != m:
                    err = ERR_CANDIDATES
                    continue
                for j in range(m):
                    v = np.float32(grads[k][e0 + j]) + np.float32(grads[k][e0 + m + j])
                    if k > 0:
                        v = np.float32(out[o + j]) + v
                    if k == K - 1:
                        v = np.float32(v) / np.float32(K)
                    out[o + j] = v
                    if k == 0:
                        a = e0 + j
                        rec[:, o + j] = (gid[ei[0, a]], gid[ei[1, a]], et[a])
            outs.append(out.copy())
    return outs, rec, err


def scatter_regimes(case):
    got = {"K=%d" % case["K"], "palette:" + case["palette"]}
    ms, q, off = np.asarray(case["ms"]), case["tag"], case["offsets"]
    if (q < 0).any():
        got.add("tag=-1")
    if (ms > 4 * MASK_THREADS).any():
        got.add("m>1024")
    if any(p >= 0 and off[p + 1] - off[p] != m for p, m in zip(q, ms)):
        got.add("offsets_disagree")
    return got


# ---- the int64 regime ---------------------------------------------------------------------------------------------------
BIG_NI, BIG_NU = 2 ** 22 + 3, 1100


@functools.lru_cache(None)
def big_graph():
    """2^22 + 3 items, 1 100 users of 0..5 ratings: the full-catalogue plan passes 2^32"""
    rng = np.random.default_rng(81)
    rows = []
    for u in range(BIG_NU):
        r = set(rng.integers(0, BIG_NI, int(rng.integers(0, 6))).tolist())
        if u % 97 == 0:
            r |= {0, BIG_NI - 1}
        rows.append(list(r))
    return _csr(rows, BIG_NI, 2)


BIG_LIST = np.arange(0, BIG_NI, 2, dtype=np.int64)      # half the catalogue, 0 and 2^22 + 2 among them


def big_cases():
    rng = np.random.default_rng(83)
    users = rng.permutation(BIG_NU).astype(np.int64)
    users = np.concatenate([users, users[:20]])          # repeated users
    cases = []
    for cand in (None, BIG_LIST):
        claims = {"P>2^31", "straddle_2^31-1", "straddle_2^31", "tail", "last_full_batch"}
        claims |= {"mode:no_list", "P>2^32", "straddle_2^32"} if cand is None else {"mode:shared"}
        c = dict(kernel="int64", name="full catalogue" if cand is None else "half-catalogue list", users=users,
                 cand=cand, exclude=True, B=600, claims=claims)
        off = big_user_off(c)
        P = int(off[-1])
        curs = [2 ** 31 - 300, 2 ** 31 - 601, P - c["B"], P - 250, P]
        if P > 2 ** 32:
            curs += [2 ** 32 - 300, 2 ** 32 + 3 * BIG_NI - 7]
        c["cursors"] = curs
        cases.append(c)
    return cases


def big_counts(case):
    """per slot |set(cand or range(num_items)) - row(u)|, and the rated positions in cand"""
    A = big_graph()
    counts, rp = [], []
    for u in case["users"]:
        r = row(A, int(u))
        if case["cand"] is None:
            counts.append(BIG_NI - len(r))
        else:
            p = np.searchsorted(case["cand"], r)
            hit = (p < len(case["cand"])) & (case["cand"][np.minimum(p, len(case["cand"]) - 1)] == r)
            rp.append(sorted(p[hit].tolist()))
            counts.append(len(case["cand"]) - int(hit.sum()))
    return counts, rp


def big_user_off(case):
    return prefix(big_counts(case)[0])


def big_batch(case, pos, user_off):
    """the batch at pos: the owners by a linear scan over user_off, their candidate sets by np.setdiff1d"""
    A = big_graph()
    B, U = case["B"], len(case["users"])
    P = int(user_off[-1])
    c = pos + np.arange(B, dtype=np.int64)
    real = c < P
    c = np.where(real, c, P - 1)
    j = np.max(np.where(user_off[None, :U] <= c[:, None], np.arange(U)[None, :], -1), axis=1)
    v = np.zeros(B, np.int64)
    for jj in np.unique(j):
        u = int(case["users"][jj])
        s = np.setdiff1d(np.arange(BIG_NI) if case["cand"] is None else case["cand"], row(A, u))
        sel = j == jj
        v[sel] = s[c[sel] - user_off[jj]]
    u = case["users"][j]
    return u, v, u * BIG_NI + v, np.where(real, j, -1)


def big_regimes(case):
    off = big_user_off(case)
    P, B = int(off[-1]), case["B"]
    got = {"mode:" + ("no_list" if case["cand"] is None else "shared")}
    if P > 2 ** 32:
        got.add("P>2^32")
    if P > 2 ** 31:
        got.add("P>2^31")
    for name, x in (("straddle_2^31-1", 2 ** 31 - 1), ("straddle_2^31", 2 ** 31), ("straddle_2^32", 2 ** 32)):
        if any(p <= x < p + B for p in case["cursors"]) and x < P:
            got.add(name)
    if any(p < P < p + B for p in case["cursors"]):
        got.add("tail")
    if P - B in case["cursors"]:
        got.add("last_full_batch")
    return got


# ---- all cases ----------------------------------------------------------------------------------------------------------
REQUIRED = {
    "plan": {"mode:no_list", "mode:shared", "exclude", "include", "U<=1024", "chunks>=3", "repeated_users", "deg0",
             "rated_every_item", "rated_every_listed", "zero_first", "zero_run_middle", "zero_last",
             "zero_across_chunk", "item0_rated", "itemlast_rated"},
    "lists": {"width=1", "width=255", "width=256", "width=257", "width>1024", "U>1024", "row_all_empty",
              "row_all_dup", "row_all_rated", "invalid_ids", "exclude", "include", "zero_first", "zero_run_middle",
              "zero_last"},
    "pairs": {"mode:no_list", "mode:shared", "mode:per_user", "mode:explicit", "exclude", "include", "B=1", "B=511",
              "B=512", "B=513", "B>P", "second_stride", "tail", "zero_first", "zero_run_middle", "zero_last"},
    "session": {"known_user", "new_user", "shared_id", "id=2^31-1", "several_blocks", "B=1", "session_out_of_range",
                "pair_id>=2^31"},
    "offsets": {"P=1", "P=511", "P=512", "P=513", "P>4096", "T>=2^31", "T>=2^32", "zero_first", "zero_run_middle",
                "zero_last", "zero_across_chunk"},
    "count": {"tag=-1", "several_blocks", "zero_edges"},
    "occl": {"zero_first", "zero_run_middle", "zero_last", "second_stride", "B=1", "tail", "T~2^31", "invalid_ids"},
    "mask": {"m=0", "m=1", "m=255", "m=256", "m=257", "m>1024", "edge_cap>E", "tag=-1", "j_outside",
             "drop_past_first_stride"},
    "scatter": {"K=1", "K=2", "K=3", "tag=-1", "m>1024", "offsets_disagree", "palette:signed_zero", "palette:nan",
                "palette:subnormal", "palette:inf", "palette:near_one"},
    "int64": {"mode:no_list", "mode:shared", "P>2^32", "P>2^31", "straddle_2^31-1", "straddle_2^31",
              "straddle_2^32", "tail", "last_full_batch"},
}

REGIMES = {"plan": plan_regimes, "lists": lists_regimes, "pairs": pairs_regimes, "session": session_regimes,
           "offsets": offsets_regimes, "count": count_regimes, "occl": occl_regimes, "mask": mask_regimes,
           "scatter": scatter_regimes, "int64": big_regimes}


@functools.lru_cache(None)
def all_cases():
    return (plan_cases() + lists_cases() + pairs_cases() + session_cases() + offsets_cases() + count_cases() +
            occl_cases() + mask_cases() + scatter_cases() + big_cases())
