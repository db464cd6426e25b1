"""The draw, counterfactual and online-draw cases of tests/draw_cases.py, tests/counterfactual_cases.py and
tests/online_cases.py, checked without a GPU.

* every case reaches the regimes it claims, re-derived from its data alone, and between them the cases of each kernel
  reach every regime that kernel branches on;
* the launch constants the regimes depend on equal the constexprs of csrc/draws.cu, csrc/counterfactual.cu and
  csrc/online.cu, so a changed block size flags the cases before they silently stop reaching a stride or chunk boundary;
* the host twins of igmc_b200/recommend.py and igmc_b200/train_eval.py agree with the brute-force enumerations on the
  cases they run, so the twins other tests rely on are held to the contract at these regimes too: adj_dropout = 1
  keeps no edge, not even one whose hash has all 32 high bits set."""
import numpy as np
import pytest

from igmc_b200 import recommend as rc
from igmc_b200 import train_eval as te
from igmc_b200.models import _keep_threshold, edge_keep_reference, hidden_keep_reference
from tests import counterfactual_cases as cc
from tests import draw_cases as dc
from tests import online_cases as oc
from tests import support
from tests.ranking_cases import same_f32

MODULES = (dc, cc, oc)
CASES = [c for m in MODULES for c in m.all_cases()]


def _module(kernel):
    return next(m for m in MODULES if kernel in m.REQUIRED)


def _of(kernel):
    return [c for c in CASES if c["kernel"] == kernel]


@pytest.mark.parametrize("case", CASES, ids=support.pid)
def test_case_reaches_its_regimes(case):
    got = _module(case["kernel"]).REGIMES[case["kernel"]](case)
    assert case["claims"] <= got, (case["claims"] - got)


@pytest.mark.parametrize("mod", MODULES, ids=lambda m: m.__name__)
def test_every_regime_is_reached(mod):
    reached = {k: set() for k in mod.REQUIRED}
    for c in mod.all_cases():
        reached[c["kernel"]] |= c["claims"]
    for kernel, need in mod.REQUIRED.items():
        assert need <= reached[kernel], (kernel, need - reached[kernel])


@pytest.mark.parametrize("mod", MODULES, ids=lambda m: m.__name__)
def test_claims_are_declared_not_derived(mod):
    support.claims_are_declared(mod)


@pytest.mark.parametrize("mod", MODULES, ids=lambda m: m.__name__)
def test_launch_constants_match_the_sources(mod):
    support.launch_constants_match(mod.CONSTANTS)


# ---- the brute force's own footing --------------------------------------------------------------------------------------
def test_the_constructed_hashes():
    """the seeds built by inverting splitmix64 give the hashes they were built for"""
    state = dc.draw_state(dc.P1_SEED, dc.P1_PID, 0, 0)
    assert dc.hash_hi(state, dc.P1_EDGE) == 0xFFFFFFFF and not dc.keeps(state, dc.P1_EDGE, 1.0)
    th = dc.keep_thresh(dc.P_DECIMAL)
    assert th == 429496736 != int(dc.P_DECIMAL * 2 ** 32)
    for high in (th, th - 1, 0, 0xFFFFFFFF):
        seed = dc.seed_for(dc.AT_PID, dc.AT_DRAW, dc.AT_EDGE, high)
        assert dc.hash_hi(dc.draw_state(seed, dc.AT_PID, dc.AT_DRAW, 0), dc.AT_EDGE) == high
    for x in (0, 1, dc.M64, 0x3f0d2d8aa7a78368):
        assert dc.unsplitmix64(dc.splitmix64(x)) == x


def test_dropout_at_one_keeps_nothing():
    """p >= 1 keeps no unit in the model twins either (the hidden dropout's kept scale 1 / (1 - p) would be inf)"""
    assert _keep_threshold(1.0) == 2 ** 32 and _keep_threshold(np.float32(1.0)) == 2 ** 32
    assert _keep_threshold(np.nextafter(np.float32(1), np.float32(0))) == 2 ** 32 - 256
    assert [_keep_threshold(p) for p in (0.0, 0.5)] == [0, 2 ** 31]
    seed = (dc.draw_state(dc.P1_SEED, dc.P1_PID, 0, 0) + dc.P1_EDGE) & dc.M64   # its one edge hashes to 0xFFFFFFFF
    assert not edge_keep_reference(seed, 1, 1.0).any() and edge_keep_reference(seed, 1, 0.999).all()
    hseed = seed ^ 0x5bd1e995a5a5a5a5
    assert not hidden_keep_reference(hseed, 1, 1.0).any() and hidden_keep_reference(hseed, 1, 0.999)[0, 0]


# ---- the host twins against the brute force -----------------------------------------------------------------------------
@pytest.mark.parametrize("case", _of("expand"), ids=support.pid)
def test_draws_expand_twin(case):
    got = rc.draws_expand_host(case["S"], case["B"], case["pair_u"], case["pair_v"], case["pair_pid"],
                               case["pair_tag"])
    for g, w in zip(got, dc.expand_reference(case)):
        assert np.array_equal(g, w)


@pytest.mark.parametrize("case", _of("mask"), ids=support.pid)
def test_draws_mask_twin(case):
    ek, hk = dc.mask_reference(case)
    gek, ghk = rc.draws_mask_host(case["edge_ptr"], case["pair_id"], case["tag"], case["draw"], case["p"],
                                  case["seed"])
    assert np.array_equal(gek, ek), np.flatnonzero(gek != ek)[:5]
    assert np.array_equal(ghk, hk)


@pytest.mark.parametrize("case", _of("stats"), ids=support.pid)
def test_draws_stats_twin(case):
    x, mean, sd, key = dc.stats_reference(case)
    with np.errstate(all="ignore"):
        hx, hm, hs, hk = rc.draws_stats_host(case["preds"], case["K"], case["B"], case["S"], case["beta"])
    assert same_f32(hx, x) and same_f32(hm, mean) and same_f32(hs, sd) and same_f32(hk, key)


@pytest.mark.parametrize("case", [c for c in _of("cf_pairs")
                                  if c["name"] not in ("invalid ids", "candidate past the row")], ids=support.pid)
def test_counterfactual_pairs_twin(case):
    rp, col, rat = cc.graph()
    for pos in case["cursors"]:
        want = cc.pairs_reference(case, pos)
        out, rows = rc.counterfactual_pairs_host(rp, col, rat, cc.NI, case["users"], case["items"], case["rivals"],
                                                 case["removed"], case["size"], case["offsets"], case["step"], pos,
                                                 case["B"])
        for g, w in zip(list(out) + list(rows), want[:4] + want[4:8]):
            assert np.array_equal(g, w), pos


@pytest.mark.parametrize("case", [c for c in _of("cf_select") if c["name"] != "not the plan's trials"], ids=support.pid)
def test_counterfactual_select_twin(case):
    rp, col, rat = cc.graph()
    want, err, _ = cc.select_reference(case)
    assert err == 0
    Q, M = len(case["users"]), case["M"]
    st = dict(removed=case["removed"].copy(), size=case["size"].copy(), count=np.full(Q, cc.S32, np.int32),
              found=np.full(Q, 0xAB, np.uint8), items=np.full((Q, M), cc.S32, np.int32),
              ratings=np.full((Q, M), cc.S32, np.int32), score=np.full((Q, M + 1), cc.SF, np.float32),
              rival_score=np.full((Q, M + 1), cc.SF, np.float32))
    with np.errstate(invalid="ignore"):
        rc.counterfactual_select_host(rp, col, rat, case["users"], case["items"], case["rivals"], case["offsets"],
                                      case["scores"], case["step"], st)
    for k, w in want.items():
        if k in ("score", "rival_score"):
            assert same_f32(st[k], w), k
        else:
            assert np.array_equal(st[k], w), k


@pytest.mark.parametrize("case", [c for c in _of("online_draw") if not c["empty"]], ids=support.pid)
def test_online_draw_twin(case):
    rp, col, rat, nu, ni = oc.graph()
    u, v, lab, pid, seeds, err, _ = oc.draw_reference(case)
    got = te.online_draw_host(rp, col, rat, ni, case["ring"][0], case["ring"][1], case["total"], case["thresh"],
                              case["step_count"] + case["step_ahead"], case["sample_seed"], case["drop_seed"],
                              case["B"])
    for g, w in zip(got[:5], (u, v, lab, pid, seeds)):
        assert np.array_equal(g, w)


@pytest.mark.parametrize("case", _of("append"), ids=support.pid)
def test_recent_append_twin(case):
    ring = (np.full(case["capacity"], oc.RING_SENT, np.int32), np.full(case["capacity"], oc.RING_SENT, np.int32),
            case["total"])
    for (u, v, x), (wu, wv, wt, _) in zip(case["calls"], oc.append_reference(case)):
        ring = te.recent_append_host(*ring, u, v, x)
        assert np.array_equal(ring[0], wu) and np.array_equal(ring[1], wv) and ring[2] == wt
