"""In-place graph updates on the host (no GPU): the numpy twin of igmc_graph_update_plan / _apply
(util_functions.graph_update_host) against a dict-of-keys rebuild through scipy, and RatingGraph.update's input
validation."""
import numpy as np
import pytest
import scipy.sparse as ssp

from igmc_b200.data import build_adj, synth_ratings
from igmc_b200.util_functions import RatingGraph, graph_update_host


def _host_graph(A):
    """the host arrays RatingGraph builds, without touching a device"""
    A = ssp.csr_matrix(A)
    A.sum_duplicates()
    A.sort_indices()
    Cc = A.tocsc()
    Cc.sort_indices()
    return dict(row_ptr=A.indptr.astype(np.int32), col_idx=A.indices.astype(np.int32),
                rating=(np.rint(A.data).astype(np.int64) - 1).astype(np.uint8), col_ptr=Cc.indptr.astype(np.int32),
                row_idx=Cc.indices.astype(np.int32))


def _dok_apply(A, users, items, values, shape):
    """the reference semantics: a dict of keys, each entry applied in order, rebuilt at ``shape``"""
    A = A.tocoo()
    d = {(int(a), int(b)): float(x) for a, b, x in zip(A.row, A.col, A.data)}
    for a, b, x in zip(users, items, values):
        if x == 0:
            d.pop((int(a), int(b)), None)
        else:
            d[(int(a), int(b))] = float(x)
    if d:
        k = np.array(list(d.keys()), np.int64)
        v = np.array(list(d.values()), np.float32)
        return ssp.csr_matrix((v, (k[:, 0], k[:, 1])), shape=shape, dtype=np.float32)
    return ssp.csr_matrix(shape, dtype=np.float32)


def _check(A, users, items, values, shape_req=None):
    nu, ni = A.shape
    host = _host_graph(A)
    got, hdr = graph_update_host(host, A.shape, users, items, values, shape_req)
    req = (0, 0) if shape_req is None else shape_req
    shape = (max(nu, req[0], int(np.max(users)) + 1), max(ni, req[1], int(np.max(items)) + 1))
    want_A = _dok_apply(A, users, items, values, shape)
    want = _host_graph(want_A)
    for k in want:
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k
    assert (hdr["num_users"], hdr["num_items"]) == shape
    assert hdr["nnz"] == want_A.nnz
    deg_r, deg_c = np.diff(want["row_ptr"]), np.diff(want["col_ptr"])
    assert hdr["max_row_deg"] == (int(deg_r.max()) if want_A.nnz else 0)
    assert hdr["max_col_deg"] == (int(deg_c.max()) if want_A.nnz else 0)
    # counts: what changed between the two matrices
    old = {(int(a), int(b)): float(x) for a, b, x in zip(*ssp.find(A))}
    new = {(int(a), int(b)): float(x) for a, b, x in zip(*ssp.find(want_A))}
    assert hdr["inserted"] == len(new.keys() - old.keys())
    assert hdr["removed"] == len(old.keys() - new.keys())
    assert hdr["changed"] == sum(1 for k in new.keys() & old.keys() if new[k] != old[k])
    return want_A


def _random_delta(rng, A, n, grow=(0, 0), R=5):
    nu, ni = A.shape
    coo = A.tocoo()
    kinds = rng.integers(0, 4, n)
    u = np.empty(n, np.int64)
    v = np.empty(n, np.int64)
    x = np.empty(n, np.int64)
    for i, k in enumerate(kinds):
        if k in (0, 1) and A.nnz:          # overwrite / delete an existing rating
            e = rng.integers(A.nnz)
            u[i], v[i] = coo.row[e], coo.col[e]
            x[i] = rng.integers(1, R + 1) if k == 0 else 0
        else:                               # insert anywhere (new users / items included) or delete an absent pair
            u[i] = rng.integers(nu + grow[0])
            v[i] = rng.integers(ni + grow[1])
            x[i] = rng.integers(1, R + 1) if k == 2 else 0
    dup = rng.integers(0, n, n // 5)        # repeated pairs: the last occurrence wins
    if len(dup):
        u = np.concatenate([u, u[dup]])
        v = np.concatenate([v, v[dup]])
        x = np.concatenate([x, rng.integers(0, R + 1, len(dup))])
    return u, v, x


def _small(seed, nu=40, ni=30, nnz=300, R=5):
    u, v, lab = synth_ratings(nu, ni, nnz, R, seed=seed)
    return build_adj(u, v, lab, nu, ni)


@pytest.mark.parametrize("seed", range(8))
def test_twin_matches_scipy_rebuild_random(seed):
    rng = np.random.default_rng(seed)
    A = _small(seed)
    for n in (1, 7, 200):
        u, v, x = _random_delta(rng, A, n, grow=(5, 4))
        A = _check(A, u, v, x)


def test_twin_chain_with_growth_and_shape():
    rng = np.random.default_rng(11)
    A = _small(3)
    for step in range(20):
        u, v, x = _random_delta(rng, A, int(rng.integers(1, 60)), grow=(2, 2))
        req = (A.shape[0] + 3, A.shape[1] + 1) if step % 5 == 0 else None
        A = _check(A, u, v, x, req)


def test_twin_duplicates_last_wins():
    A = _small(1)
    coo = A.tocoo()
    a, b = int(coo.row[0]), int(coo.col[0])
    # insert-then-delete of a new pair, delete-then-insert of an existing one, three overwrites
    u = np.array([0, 0, a, a, a, a, a])
    v = np.array([29, 29, b, b, b, b, b])
    if (0, 29) in set(zip(coo.row.tolist(), coo.col.tolist())):
        u[:2] = 39
    x = np.array([3, 0, 0, 2, 5, 1, 4])
    _check(A, u, v, x)


def test_twin_delete_everything_and_empty_rows():
    A = _small(2)
    coo = A.tocoo()
    B = _check(A, coo.row, coo.col, np.zeros(A.nnz, np.int64))
    assert B.nnz == 0
    # refill one rating into an empty graph, plus a new user and a new item
    _check(B, np.array([3, 40]), np.array([2, 30]), np.array([5, 1]))


def test_twin_all_noop():
    A = _small(4)
    coo = A.tocoo()
    dense = A.toarray()
    free = np.argwhere(dense == 0)[:10]
    u = np.concatenate([coo.row[:10], free[:, 0]])
    v = np.concatenate([coo.col[:10], free[:, 1]])
    x = np.concatenate([coo.data[:10].astype(np.int64), np.zeros(len(free), np.int64)])   # same labels, absent deletes
    got, hdr = graph_update_host(_host_graph(A), A.shape, u, v, x)
    assert hdr["inserted"] == hdr["changed"] == hdr["removed"] == 0
    want = _host_graph(A)
    for k in want:
        assert np.array_equal(got[k], want[k]), k


def test_twin_new_user_with_ratings():
    A = _small(5)
    u = np.full(4, 44)
    v = np.array([3, 1, 29, 31])
    _check(A, u, v, np.array([1, 2, 3, 4]))


# ---- input validation: refused before anything runs (a host graph: no device needed) ----------------------------------
def _cpu_graph(monkeypatch, **reserve):
    """a graph that stays on the host even where a GPU exists"""
    import torch
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    return RatingGraph(_small(6), **reserve)


def test_update_validation(monkeypatch):
    g = _cpu_graph(monkeypatch, reserve_users=2, reserve_items=1, reserve_nnz=10)
    assert tuple(g.capacity) == (42, 31, g.nnz + 10)
    with pytest.raises(IndexError):
        g.update([-1], [0], [1])
    with pytest.raises(IndexError):
        g.update([0], [-3], [1])
    with pytest.raises(IndexError):
        g.update([42], [0], [1])           # id at the capacity
    with pytest.raises(IndexError):
        g.update([0], [31], [1])
    with pytest.raises(ValueError):
        g.update([0], [0], [257])
    with pytest.raises(ValueError):
        g.update([0], [0], [-1])
    with pytest.raises(ValueError):
        g.update([0, 1], [0], [1])          # length mismatch
    with pytest.raises(ValueError):
        g.update([0], [0], [1], shape=(39, 30))   # shrinking
    with pytest.raises(ValueError):
        g.update([0], [0], [1], shape=(43, 30))   # beyond the capacity
    with pytest.raises(TypeError):
        g.update([0.5], [0], [1])
    # an empty delta changes nothing and needs no device
    assert g.update([], [], []) == dict(inserted=0, changed=0, removed=0)
    assert g.version == 0
    # a valid delta needs the device
    with pytest.raises(RuntimeError):
        g.update([0], [0], [1])
    assert g.version == 0 and g.shape == (40, 30)


def test_defaults_keep_the_graph_as_before(monkeypatch):
    g = _cpu_graph(monkeypatch)
    assert tuple(g.capacity) == (40, 30, g.nnz)
    with pytest.raises(ValueError):
        RatingGraph(_small(6), reserve_nnz=-1)
