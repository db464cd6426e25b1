"""Question impact on the host: the numpy twins of igmc_elicit_pairs / igmc_elicit_stats against brute forces written
from include/igmc_b200.h, elicit_host over a deterministic fake scorer against a hand-worked example, and the
argument checks.  No GPU."""
import types

import numpy as np
import pytest

from igmc_b200 import recommend as rc
from tests import elicit_cases as ec
from tests import support


def test_launch_constants_match_the_source():
    support.launch_constants_match(ec.CONSTANTS)


@pytest.mark.parametrize("case", ec.pair_cases(), ids=lambda c: c["name"])
def test_pairs_twin_is_the_brute_force(case):
    c = case
    rp, ci, rt = ec.csr(c["rows"])
    out, sess, (ru, wptr, wcol, wrat) = rc.elicit_pairs_host(rp, ci, rt, c["users"], c["num_items"], c["A"],
                                                             c["targets"], c["unit_s"], c["unit_q"], c["unit_tag"],
                                                             c["B"])
    pos, trial = ec.brute_pairs(c["rows"], c["users"], c["num_items"], c["A"], c["targets"], c["unit_s"],
                                c["unit_q"], c["unit_tag"], c["B"])
    assert [tuple(int(x) for x in out[:, i]) + (int(sess[i]),) for i in range(c["B"])] == pos
    assert list(ru) == [u for u, _ in trial]
    assert np.array_equal(np.diff(wptr), [len(r) for _, r in trial])
    assert [(int(i), int(lab)) for i, lab in zip(wcol, wrat)] == [e for _, r in trial for e in r]


def test_pairs_map_by_hand():
    """the first case spelled out: U = 15, G = 5, positions 75..79 are padding; the trial rows insert the question"""
    c = ec.pair_cases()[0]
    rp, ci, rt = ec.csr(c["rows"])
    out, sess, (ru, wptr, wcol, wrat) = rc.elicit_pairs_host(rp, ci, rt, c["users"], 12, 5, c["targets"],
                                                             c["unit_s"], c["unit_q"], c["unit_tag"], 80)
    assert list(out[1, 15:18]) == [1, 5, 11] and list(out[3, 15:30]) == [11] * 15    # unit 1, answer 0
    assert list(sess[15:30]) == [5, 5, 5, 6, 6, 6, 7, 7, 7, 8, 8, 8, 9, 9, 9]
    assert list(out[3, 75:]) == [-1] * 5 and list(sess[75:]) == [0] * 5 and list(out[1, 75:]) == [0] * 5
    assert list(out[0, 45:60]) == [500] * 15 and out[2, 45] == 500 * 12 + 1
    rows = [list(zip(wcol[wptr[r]:wptr[r + 1]], wrat[wptr[r]:wptr[r + 1]])) for r in range(25)]
    assert rows[0] == [(0, 0), (2, 0), (5, 3), (9, 1)]                  # at the start
    assert rows[7] == [(2, 0), (5, 3), (7, 2), (9, 1)]                  # in the middle, answer 2
    assert rows[14] == [(2, 0), (5, 3), (9, 1), (10, 4)]                # at the end
    assert rows[16] == [(4, 1)]                                         # an empty row
    assert rows[24] == [(0, 4), (1, 4)]


@pytest.mark.parametrize("case", ec.stats_cases(), ids=lambda c: c["name"])
def test_stats_twin_is_the_brute_force(case):
    c = case
    impact, mean, utag = rc.elicit_stats_host(np.asarray(c["preds"], np.float32), c["K"], c["B"], c["A"], c["W"],
                                              c["tag"])
    want = ec.brute_stats(c["preds"], c["K"], c["B"], c["A"], c["W"], c["tag"])
    assert len(want) == len(impact)
    for g, w in enumerate(want):
        if w is None:
            assert utag[g] == -1
            continue
        assert support.same(impact[g], w[0]) and support.same(mean[g], w[1]) and utag[g] == w[2], g


def test_stats_by_hand():
    imp, mean, _ = rc.elicit_stats_host(np.asarray(ec.stats_cases()[0]["preds"], np.float32), 1, 13, 2, 3,
                                        ec.stats_cases()[0]["tag"])
    assert imp[0] == np.float32((1 + 2.0 ** -23) / 3) != np.float32(np.float32(1) / 3)
    c = ec.stats_cases()[1]
    imp, mean, utag = rc.elicit_stats_host(np.asarray(c["preds"], np.float32), 1, 30, 3, 2, c["tag"])
    assert imp[0] == np.float32(0.75) and list(mean[0]) == [0.5, 1.0, 0.25]         # slot 1 ignored
    assert np.isnan(imp[1]) and np.isnan(mean[1, 1]) and list(mean[1, [0, 2]]) == [1.5, 4.5]
    assert imp[2] == np.inf and mean[2, 0] == np.inf
    assert np.isnan(imp[3])                                                            # inf - inf
    assert imp[4] == np.inf and np.isnan(mean[4, 0]) and list(utag) == [0, 1, 2, 3, 4]


# ---- elicit_host over a fake scorer -------------------------------------------------------------------------------------
def _fake_scorer(rows):
    """score of (session s, target t) with (q, a) added: 1 + the sum of the labels in s's row plus a, times t + 1,
    when q < t; otherwise (q >= t) the score without the new rating"""
    def score(session, question, answer, target):
        base = np.array([sum(lab for _, lab in rows[s]) for s in session], np.float64)
        add = np.where(np.asarray(question) < np.asarray(target), np.asarray(answer), 0)
        return ((1 + base + add) * (np.asarray(target) + 1)).astype(np.float32)
    return score


def test_elicit_host_by_hand():
    rows = [[(1, 2)], []]
    rp, ci, _ = ec.csr(rows)
    scorer = _fake_scorer(rows)
    # A = 3, targets {2, 4}: question q moves target t by (A - 1) * (t + 1) when q < t, else not at all
    imp, mean = rc.question_impact_host(3, [2, 4], [0, 0, 1], [0, 3, 3], scorer)
    assert list(imp) == [(2 * 3 + 2 * 5) / 2, (0 + 2 * 5) / 2, 5.0]
    assert list(mean[0]) == [(3 * 3 + 3 * 5) / 2, (4 * 3 + 4 * 5) / 2, (5 * 3 + 5 * 5) / 2]
    assert list(mean[2]) == [(1 * 3 + 1 * 5) / 2, (1 * 3 + 2 * 5) / 2, (1 * 3 + 3 * 5) / 2]
    items, top = rc.elicit_host(rp, ci, 5, 3, 3, [2, 4], scorer)
    # session 0 (item 1 rated): 0 -> 8, 2 -> 5, 3 -> 5, 4 -> 0; session 1: 0 and 1 -> 8, 2 and 3 -> 5
    assert items.tolist() == [[0, 2, 3], [0, 1, 2]] and top.tolist() == [[8, 5, 5], [8, 8, 5]]
    # per-session targets with -1 and per-session questions with -1, a session with fewer questions than n
    items, top = rc.elicit_host(rp, ci, 5, 3, 4, [[4, -1], [-1, 2]], scorer, questions=[[1, 3, -1], [-1, 4, 0]])
    assert items.tolist() == [[3, -1, -1, -1], [0, 4, -1, -1]]
    assert top[0, 0] == 10 and top[1].tolist()[:2] == [6, 0]


# ---- argument checks ----------------------------------------------------------------------------------------------------
def test_target_checks():
    t, per = rc._elicit_targets([3, 3, 0], 4, 10, 5, 15, np.arange(4))
    assert t.shape == (1, 3) and per == 0 and t.dtype == np.int32
    t, per = rc._elicit_targets(np.array([[1, -1], [-1, 2]]), 2, 10, 5, 10, [0, 1])
    assert t.shape == (2, 2) and per == 1
    with pytest.raises(ValueError, match="raise batch_size"):
        rc._elicit_targets([1, 2, 3], 1, 10, 5, 14, [0])
    with pytest.raises(ValueError, match="empty"):
        rc._elicit_targets([], 1, 10, 5, 14, [0])
    with pytest.raises(ValueError, match="empty"):
        rc._elicit_targets(np.zeros((2, 0), np.int64), 2, 10, 5, 14, [0])
    with pytest.raises(ValueError, match="session 1 has no target"):
        rc._elicit_targets([[1, -1], [-1, -1]], 2, 10, 5, 14, [0, 1])
    rc._elicit_targets([[1, -1], [-1, -1]], 2, 10, 5, 14, [0])             # session 1 not queried
    with pytest.raises(ValueError, match="rows"):
        rc._elicit_targets([[1], [2], [3]], 2, 10, 5, 14, [0])
    with pytest.raises(IndexError):
        rc._elicit_targets([10], 1, 10, 5, 14, [0])
    with pytest.raises(IndexError):
        rc._elicit_targets([-1], 1, 10, 5, 14, [0])                        # -1 pads rows only
    with pytest.raises(IndexError):
        rc._elicit_targets([[-2]], 1, 10, 5, 14, [0])
    with pytest.raises(TypeError):
        rc._elicit_targets([1.5], 1, 10, 5, 14, [0])


def test_unit_checks():
    s = types.SimpleNamespace(num_sessions=3, graph=types.SimpleNamespace(num_items=10))
    sess, q = rc._question_units(s, [0, 2], [9, 0])
    assert sess.tolist() == [0, 2] and q.tolist() == [9, 0]
    with pytest.raises(IndexError):
        rc._question_units(s, [3], [0])
    with pytest.raises(IndexError):
        rc._question_units(s, [0], [10])
    with pytest.raises(ValueError, match="same length"):
        rc._question_units(s, [0, 1], [0])
    assert [len(a) for a in rc._question_units(s, [], [])] == [0, 0]


def test_public_checks_before_any_device():
    with pytest.raises(TypeError):
        rc.elicit(None, object(), 3, [1])
    with pytest.raises(TypeError):
        rc.question_impact(None, [0], [0], [0], [1])
