"""Rating sessions without a GPU: the numpy twin of the session row build (csrc/session.cu) against a dict-of-keys
rebuild, input validation, the candidate and retrieval twins on session rows against brute force, and the argument
of the session contract on the extraction oracle: extracting a pair on the graph with the session's edits applied
equals extracting it on the unchanged graph with only the target user's row swapped for the session row."""
import numpy as np
import pytest
import scipy.sparse as ssp

from igmc_b200 import recommend as rc
from igmc_b200.data import build_adj, synth_ratings
from oracle import extract_np


def _graph(nu=60, ni=40, n=700, R=5, seed=0):
    u, v, lab = synth_ratings(nu, ni, n, R, seed=seed)
    A = build_adj(u, v, lab, nu, ni)
    A = ssp.csr_matrix(A)
    A.sort_indices()
    host = dict(row_ptr=A.indptr.astype(np.int32), col_idx=A.indices.astype(np.int32),
                rating=(np.rint(A.data).astype(np.int64) - 1).astype(np.uint8))
    return A, host


def _dok_rows(A, users, session, items, values):
    """per session the dict item -> label of its user's row after its edits, in input order (last wins)"""
    nu = A.shape[0]
    rows = []
    for s, u in enumerate(users):
        d = {}
        if u < nu:
            for c, x in zip(A.indices[A.indptr[u]:A.indptr[u + 1]], A.data[A.indptr[u]:A.indptr[u + 1]]):
                d[int(c)] = int(round(x)) - 1
        for ss, it, x in zip(session, items, values):
            if ss != s:
                continue
            if x > 0:
                d[int(it)] = int(x) - 1
            else:
                d.pop(int(it), None)
        rows.append(d)
    return rows


def _random_edits(rng, A, users, D, R=5):
    """inserts, overwrites and deletes of present and absent ratings, repeats of a (session, item)"""
    S, ni = len(users), A.shape[1]
    session = rng.integers(0, S, D)
    items = rng.integers(0, ni, D)
    for k in range(0, D, 3):                       # a third of the edits touch a rated item of the user
        u = users[session[k]]
        if u < A.shape[0] and A.indptr[u + 1] > A.indptr[u]:
            items[k] = A.indices[rng.integers(A.indptr[u], A.indptr[u + 1])]
    values = np.where(rng.random(D) < 0.3, 0, rng.integers(1, R + 1, D))
    if D >= 4:
        rep = rng.integers(0, D, D // 4)
        session, items = np.r_[session, session[rep]], np.r_[items, items[rep]]
        values = np.r_[values, rng.integers(0, R + 1, len(rep))]
    return session, items, values


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_row_twin_matches_dict_rebuild(seed):
    A, host = _graph(seed=seed)
    rng = np.random.default_rng(seed)
    nu = A.shape[0]
    # existing users, new ids, a shared id, and sessions without edits
    users = np.r_[rng.integers(0, nu, 6), [nu, nu + 5, 3, 3], rng.integers(0, nu, 2)]
    session, items, values = _random_edits(rng, A, users[:10], 80)
    # session 4: every rating of its user deleted (an emptied row)
    u4 = users[4]
    row4 = A.indices[A.indptr[u4]:A.indptr[u4 + 1]]
    other = session != 4
    session, items, values = session[other], items[other], values[other]
    session = np.r_[session, np.full(len(row4), 4)]
    items = np.r_[items, row4]
    values = np.r_[values, np.zeros(len(row4), np.int64)]
    rp, ci, rt = rc.session_rows_host(host, A.shape, users, session, items, values)
    want = _dok_rows(A, users, session, items, values)
    assert len(rp) == len(users) + 1 and rp[0] == 0
    for s, d in enumerate(want):
        cols, labs = ci[rp[s]:rp[s + 1]], rt[rp[s]:rp[s + 1]]
        assert np.all(np.diff(cols) > 0)
        assert dict(zip(cols.tolist(), labs.tolist())) == d, s
    assert rp[5] == rp[4]                                    # emptied
    for s in (10, 11):                                       # no edits: the graph row
        u = users[s]
        assert np.array_equal(ci[rp[s]:rp[s + 1]], A.indices[A.indptr[u]:A.indptr[u + 1]])


def test_row_twin_without_edits_is_the_graph_rows():
    A, host = _graph()
    users = np.array([0, 5, 5, A.shape[0] + 2])
    rp, ci, rt = rc.session_rows_host(host, A.shape, users, [], [], [])
    for s, u in enumerate(users[:3]):
        assert np.array_equal(ci[rp[s]:rp[s + 1]], A.indices[A.indptr[u]:A.indptr[u + 1]])
    assert rp[4] == rp[3]


def test_edit_validation_through_update_inputs():
    S, ni = 3, 10
    names = ("session", "items", "values")
    for bad in (([3], [0], [1]), ([-1], [0], [1]), ([0], [10], [1]), ([0], [-1], [1])):
        with pytest.raises(IndexError):
            rc._update_inputs(*bad, S, ni, names)
    for bad in (([0], [0], [257]), ([0], [0], [-1]), ([0, 1], [0], [1])):
        with pytest.raises(ValueError):
            rc._update_inputs(*bad, S, ni, names)
    with pytest.raises(TypeError):
        rc._update_inputs([0.5], [0], [1], S, ni, names)
    s, i, v, D = rc._update_inputs([0, 2], [9, 0], [256, 0], S, ni, names)
    assert D == 2 and list(s) == [0, 2]


def test_candidate_twins_on_session_rows():
    """the candidate plan / pairs twins applied to the session rows as a CSR over query slots 0..S-1 give, per
    session, the items of a brute-force rebuild (every item or a list, minus the session's rated items)"""
    A, host = _graph(seed=4)
    rng = np.random.default_rng(4)
    nu, ni = A.shape
    users = np.array([1, 7, nu, nu + 1, 7])
    session, items, values = _random_edits(rng, A, users, 40)
    rp, ci, _ = rc.session_rows_host(host, A.shape, users, session, items, values)
    want_rows = _dok_rows(A, users, session, items, values)
    slots = np.arange(len(users))
    for cand in (None, np.sort(rng.choice(ni, 15, replace=False))):
        for excl in (True, False):
            plan = rc.candidate_plan_host(rp, ci, ni, slots, cand, excl)
            P = int(plan[0][-1])
            got = rc.candidate_pairs_host(rp, ci, ni, slots, cand, excl, plan, 0, P)
            for s in slots:
                pool = np.arange(ni) if cand is None else cand
                if excl:
                    pool = pool[~np.isin(pool, list(want_rows[s].keys()))]
                mine = got[1][got[3] == s]
                assert np.array_equal(mine, pool), (s, excl, cand is None)
    # per-session candidate lists
    rows = rng.integers(-1, ni, (len(users), 12))
    uo, lists = rc.candidate_lists_host(rp, ci, ni, slots, rows, True)
    for s in slots:
        want = np.unique(rows[s][rows[s] >= 0])
        want = want[~np.isin(want, list(want_rows[s].keys()))]
        assert np.array_equal(lists[uo[s]:uo[s + 1]], want)


def test_corated_twin_on_session_rows():
    """paths[v] = sum over u' != u of |N_s(u) & N(u')| [u' rated v], N_s the session row, equals corated_host on the
    graph with the session's edits applied"""
    A, host = _graph(seed=6)
    rng = np.random.default_rng(6)
    nu, ni = A.shape
    users = np.array([2, nu, 9])
    session, items, values = _random_edits(rng, A, users, 30)
    want_rows = _dok_rows(A, users, session, items, values)
    m = 12
    for s, u in enumerate(users):
        As = _apply(A, u, want_rows[s])
        hs = ssp.csr_matrix(As)
        wi, wp = rc.corated_host(hs.indptr, hs.indices, As.shape[0], ni, [u], m)
        # brute force on the unchanged graph with N(u) swapped for the session row
        Nu = np.array(sorted(want_rows[s].keys()), np.int64)
        B = (ssp.csr_matrix(A) > 0).astype(np.int64)
        w = np.asarray(B[:, Nu].sum(1)).ravel()
        if u < nu:
            w[u] = 0
        paths = np.asarray(B.T @ w).ravel()
        paths[Nu] = 0
        o = np.argsort(-paths, kind="stable")[:m]
        o = o[paths[o] > 0]
        assert np.array_equal(wi[0][:len(o)], o) and np.array_equal(wp[0][:len(o)], paths[o]), s


def _apply(A, u, row):
    """A with user u's row replaced by ``row`` (item -> label), the shape grown to hold u"""
    coo = ssp.coo_matrix(A)
    keep = coo.row != u
    r = np.r_[coo.row[keep], np.full(len(row), u)]
    c = np.r_[coo.col[keep], np.array(list(row.keys()), np.int64)]
    d = np.r_[coo.data[keep], np.array(list(row.values()), np.float64) + 1]
    return ssp.csr_matrix((d, (r, c)), shape=(max(A.shape[0], u + 1), A.shape[1]))


class _SwapRow(object):
    """the oracle's graph interface over the unchanged graph, with user i's row swapped for a session row"""

    def __init__(self, g, i, cols, labs):
        self.g, self.i, self.cols, self.labs = g, i, np.asarray(cols, np.int64), np.asarray(labs, np.int64)
        self.shape = g.shape

    def row(self, u):
        return (self.cols, self.labs) if u == self.i else self.g.row(u)

    def col(self, v):
        return self.g.col(v)


@pytest.mark.parametrize("h,mnph,ratio", [(1, None, 1.0), (1, 5, 1.0), (1, None, 0.6), (2, None, 1.0), (2, 4, 1.0),
                                          (3, 3, 0.8)])
def test_extraction_oracle_swaps_only_the_target_row(h, mnph, ratio):
    A, host = _graph(seed=8)
    rng = np.random.default_rng(8 + h)
    nu, ni = A.shape
    users = np.array([0, 11, nu, 11])
    session, items, values = _random_edits(rng, A, users, 30)
    # session 1 holds the target item of its pair below
    session, items, values = np.r_[session, [1]], np.r_[items, [5]], np.r_[values, [4]]
    want_rows = _dok_rows(A, users, session, items, values)
    g = extract_np.RatingCSR(A)
    for s, u in enumerate(users):
        row = want_rows[s]
        As = _apply(A, u, row)
        gs = extract_np.RatingCSR(As)
        cols = np.array(sorted(row.keys()), np.int64)
        swap = _SwapRow(g, u, cols, [row[c] for c in cols])
        for v in (5, int(rng.integers(ni)), int(cols[0]) if len(cols) else 0):
            pid = int(u) * ni + v
            a = extract_np.extract_subgraph(gs, u, v, h, ratio, mnph, seed=3, pair_id=pid)
            b = extract_np.extract_subgraph(swap, u, v, h, ratio, mnph, seed=3, pair_id=pid)
            for k in a:
                assert np.array_equal(a[k], b[k]), (s, v, k)
