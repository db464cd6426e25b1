"""The group-recommendation twins (group_rows_host, group_pairs_host, group_stats_host, predict_groups_host,
recommend_groups_host) against brute forces written from the header contract, and the input checks of
recommend_groups / predict_groups, all without a GPU."""
import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from igmc_b200 import recommend as rc
from tests import support


ROWS = [[1, 4, 7], [], [0, 4, 9, 11], [2, 7], [4], [1, 3, 5, 7, 9, 11]]


def test_group_rows_twin_is_the_union():
    rp, ci = support.rows_csr(ROWS)
    members = np.array([[0, 2, -1], [1, -1, -1], [3, 0, 5], [4, 1, 0]], np.int32)   # overlaps, an empty row, dups
    urp, uci = rc.group_rows_host(rp, ci, members)
    assert urp.dtype == np.int32 and uci.dtype == np.int32
    for g, row in enumerate(members):
        want = sorted(set(x for u in row if u >= 0 for x in ROWS[u]))
        assert uci[urp[g]:urp[g + 1]].tolist() == want
    assert urp[-1] <= sum(len(ROWS[u]) for u in members[members >= 0])               # the capacity the engine gives


def _pairs_brute(members, ni, ug, uv, ut, B):
    M = members.shape[1]
    out = []
    for i in range(B):
        u0, j = divmod(i, M)
        if u0 >= B // M:
            u0, j, real = 0, 0, False
        else:
            real = True
        grp = members[ug[u0]]
        m = int(grp[j])
        u = m if m >= 0 else int(grp[0])
        v = int(uv[u0])
        out.append((u, v, u * ni + v, int(ut[u0]) if real and m >= 0 else -1))
    return np.array(out, np.int64).T


@pytest.mark.parametrize("B", [12, 13, 15, 3])
def test_group_pairs_twin(B):
    members = np.array([[5, 2, -1], [0, -1, -1], [3, 1, 4]], np.int32)               # mixed sizes, M = 3
    ni = 3_000_000_000 // 4                                                            # pair ids past 2^31
    Gu = B // 3
    ug = np.array([0, 0, 1, 2, 2][:max(Gu, 1)], np.int32)
    uv = np.array([7, 9, 7, 123456789, 0][:max(Gu, 1)], np.int32)
    ut = np.array([0, 0, 1, 2, -1][:max(Gu, 1)], np.int64)                           # the last unit: a tail unit
    got = rc.group_pairs_host(members, ni, ug, uv, ut, B)
    assert np.array_equal(got, _pairs_brute(members, ni, ug, uv, ut, B))
    assert got[2].max() > 2 ** 31
    if B % 3 == 0:
        assert (got[3][Gu * 3:] == -1).all()                                           # B filled exactly: no tail
    assert (got[3][B - B % 3:] == -1).all()


def _seq_mean(x):
    s = 0.0
    for a in x:                                                                         # sequential, not pairwise
        s = s + float(a)
    return np.float32(s / len(x))


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def test_aggregates_on_ties_signed_zero_inf_nan():
    f = np.float32
    assert _bits(rc._aggregate_of([f(0.0), f(-0.0)], "min")) == _bits(f(0.0))           # the first in member order
    assert _bits(rc._aggregate_of([f(-0.0), f(0.0)], "min")) == _bits(f(-0.0))
    assert _bits(rc._aggregate_of([f(-0.0), f(0.0)], "max")) == _bits(f(-0.0))
    assert _bits(rc._aggregate_of([f(0.0), f(-0.0)], "max")) == _bits(f(0.0))
    assert rc._aggregate_of([f(1), f(np.inf), f(2)], "max") == np.inf
    assert rc._aggregate_of([f(1), f(-np.inf)], "min") == -np.inf
    assert np.isnan(rc._aggregate_of([f(np.inf), f(-np.inf)], "mean"))
    for agg in ("mean", "min", "max"):
        assert np.isnan(rc._aggregate_of([f(1), f(np.nan), f(2)], agg))
        assert np.isnan(rc._aggregate_of([f(np.nan)], agg))
    # a sum past fp32's range on the way, exact in fp64 and rounded once at the end
    x = np.array([3.4028235e38, 3.4028235e38, -3.4028235e38, 1.0], np.float32)          # no fp32 overflow in fp64
    assert _bits(rc._aggregate_of(x, "mean")) == _bits(_seq_mean(x))
    rng = np.random.default_rng(0)
    for _ in range(200):
        x = (rng.standard_normal(rng.integers(1, 9)) * 10.0 ** rng.integers(-3, 4)).astype(np.float32)
        assert _bits(rc._aggregate_of(x, "mean")) == _bits(_seq_mean(x))
        assert rc._aggregate_of(x, "min") == x.min() and rc._aggregate_of(x, "max") == x.max()


@pytest.mark.parametrize("agg", ["mean", "min", "max"])
def test_group_stats_twin(agg):
    rng = np.random.default_rng(3)
    K, M, B = 2, 3, 11                                                                   # Gu = 3, positions 9, 10 pad
    preds = rng.standard_normal((K, B)).astype(np.float32)
    preds[:, 1] = [np.nan, 0.0]
    preds[:, 4] = [0.0, -0.0]
    preds[:, 5] = [-0.0, 0.0]
    tag = np.array([0, 0, 0, 5, 5, -1, -1, -1, -1, 0, 0], np.int64)                  # unit 2 without real slots
    key, xs, utag = rc.group_stats_host(preds, K, B, M, agg, tag)
    x = rc._ckpt_mean_host(preds, K, B)
    assert utag.tolist() == [0, 5, -1] and key[2] == 0 and np.isnan(xs[2]).all()
    assert np.isnan(key[0])                                                             # a NaN member
    want = rc._aggregate_of(x[3:5], agg)
    assert _bits(key[1]) == _bits(want)
    assert _bits(xs[1, :2]).tolist() == _bits(x[3:5]).tolist() and np.isnan(xs[1, 2])


def test_predict_and_recommend_host_compose_pair_scores():
    rp, ci = support.rows_csr(ROWS)
    ni = 12
    members = np.array([[0, 2], [4, -1], [3, 1]], np.int32)

    def scorer(u, v):                                                                   # any deterministic pair score
        return (np.sin(np.asarray(u) * 7.0 + np.asarray(v) * 0.37) * 2.5).astype(np.float32)
    for agg in ("mean", "min", "max"):
        s, m = rc.predict_groups_host(members, [0, 1, 2, 0], [3, 3, 11, 4], agg, scorer)
        assert np.isnan(m[1, 1]) and m[0].tolist() == scorer([0, 2], [3, 3]).tolist()
        assert _bits(s[0]) == _bits(rc._aggregate_of(scorer([0, 2], [3, 3]), agg))
        ti, ts = rc.recommend_groups_host(rp, ci, ni, members, 20, agg, scorer)
        for g in range(3):
            rated = set(x for u in members[g] if u >= 0 for x in ROWS[u])
            cand = np.array([v for v in range(ni) if v not in rated])
            keys = np.array([rc._aggregate_of(scorer([u for u in members[g] if u >= 0], [v] * (members[g] >= 0).sum()),
                                              agg) for v in cand], np.float32)
            want_s, want_i = rc.rank_host(keys, cand, 20)
            assert np.array_equal(ti[g], want_i) and np.array_equal(_bits(ts[g]), _bits(want_s))
        ti, _ = rc.recommend_groups_host(rp, ci, ni, members, 3, agg, scorer, items=[[4, 5, -1], [4, 4, 0], [9, 8, 7]],
                                         exclude_rated=False)
        assert sorted(ti[1].tolist()) == [-1, 0, 4]


# ---- input checks (no engine is built: they fail first) ----------------------------------------------------------------
class _Graph(object):
    shape = (10, 20)


def test_group_members_layout():
    got = rc._group_members([[3, 1], [7], [0, 2, 4]], 10, 256)
    assert got.dtype == np.int32 and got.tolist() == [[3, 1, -1], [7, -1, -1], [0, 2, 4]]
    arr = rc._group_members(np.array([[-1, 3, 1], [7, -1, -1]]), 10, 256)               # -1 entries skipped
    assert arr.tolist() == [[3, 1], [7, -1]]
    assert rc._group_members(torch.tensor([[5, 6]]), 10, 256).tolist() == [[5, 6]]
    assert rc._group_members([list(range(64))], 100, 256).shape == (1, 64)


@pytest.mark.parametrize("groups,batch,exc", [
    ([[1, 2], []], 256, ValueError),                                                     # an empty group
    (np.array([[1, -1], [-1, -1]]), 256, ValueError),
    ([[1, 2, 1]], 256, ValueError),                                                      # a duplicate member
    ([[1, 10]], 256, IndexError),                                                        # out of range
    ([[-2, 1]], 256, IndexError),
    ([[0, 1, 2, 3]], 3, NotImplementedError),                                            # M > batch_size
    ([list(range(65))], 256, NotImplementedError),                                       # M > IGMC_GROUP_MAX
    ([[1.5, 2]], 256, TypeError),
    (np.zeros(3, np.int64), 256, ValueError),                                            # not 2-D
])
def test_group_members_refused(groups, batch, exc):
    with pytest.raises(exc):
        rc._group_members(groups, 10 if exc is not NotImplementedError else 100, batch)


def test_public_entry_points_check_before_any_engine():
    g = _Graph()
    m = None                                                                            # never reached
    with pytest.raises(ValueError, match="aggregate"):
        rc.recommend_groups(m, g, [[1]], 3, aggregate="median")
    with pytest.raises(ValueError, match="aggregate"):
        rc.predict_groups(m, g, [[1]], [0], [1], aggregate="sum")
    with pytest.raises(NotImplementedError, match="retrieve"):
        rc.recommend_groups(m, g, [[1]], 3, retrieve=10)
    with pytest.raises(NotImplementedError, match="draws"):
        rc.recommend_groups(m, g, [[1]], 3, draws=4)
    with pytest.raises(ValueError):
        rc.recommend_groups(m, g, [[1], []], 3)
    with pytest.raises(ValueError):
        rc.recommend_groups(m, g, [[1, 1]], 3)
    with pytest.raises(IndexError):
        rc.recommend_groups(m, g, [[1, 10]], 3)
    with pytest.raises(NotImplementedError):
        rc.recommend_groups(m, g, [[1, 2, 3]], 3, batch_size=2)
    with pytest.raises(ValueError):
        rc.recommend_groups(m, g, [[1]], 0)
    with pytest.raises(NotImplementedError):
        rc.recommend_groups(m, g, [[1]], _lib.TOPK_MAX + 1)
    with pytest.raises(IndexError):
        rc.predict_groups(m, g, [[1]], [1], [1])                                         # group 1 of one
    with pytest.raises(ValueError, match="same length"):
        rc.predict_groups(m, g, [[1]], [0, 0], [1])


def test_aggregate_codes_match_header():
    src = open(_lib.os.path.join(_lib.HERE, "..", "include", "igmc_b200.h")).read()
    for code, name in enumerate(_lib.GROUP_AGGREGATES):
        assert "#define IGMC_GROUP_AGG_%s %d" % (name.upper(), code) in src
    assert "#define IGMC_GROUP_MAX %d" % _lib.GROUP_MAX in src
