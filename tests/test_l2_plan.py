"""The L2 plan (csrc/rgcn_l2.cu) through the C-ABI and the host's plan rule, without a GPU: which shapes it accepts,
that its shared memory does not grow with the subgraph, which entry points refuse it, and that ``select_plan`` picks
it exactly where no shared-memory plan fits."""
import ctypes
import functools

import pytest

from igmc_b200 import _lib
from igmc_b200.models import l2_cluster, select_plan
from tests import support

_cpu_model = functools.partial(support.model, seed=None, cuda=False)   # plan queries: unseeded, on the host

SMS = 132   # H100 SXM


def _plan_bytes(m, n_cap, plan):
    lib, c = _lib.load(), ctypes.byref(m._cmodel)
    return lib.igmc_model_plan(c, n_cap, plan, 0), lib.igmc_model_plan(c, n_cap, plan, 1)


@pytest.mark.parametrize("R", [5, 10, 71])
@pytest.mark.parametrize("n_cap", [802, 1476, 8000])
def test_l2_plan_accepts_large_subgraphs(R, n_cap):
    for NB in (2, 4):
        m = _cpu_model(R, nb=NB)
        for c in (1, 2, 4, 8):
            f, b = _plan_bytes(m, n_cap, _lib.plan_l2(c))
            assert f > 0 and b > 0, (R, NB, n_cap, c, f, b)
            assert (f, b) == _plan_bytes(m, 2, _lib.plan_l2(c)) == _plan_bytes(m, _lib.L2_MAX_NODES, _lib.plan_l2(c))
        # no shared-memory plan takes these subgraphs
        for plan in (0, 1, 2, 3, 4):
            f, b = _plan_bytes(m, n_cap, plan)
            assert f <= 0 or b <= 0, (R, NB, n_cap, plan)


def test_l2_plan_limits():
    m = _cpu_model(5)
    assert min(_plan_bytes(m, _lib.L2_MAX_NODES + 1, _lib.plan_l2(2))) < 0       # 16-bit neighbour field
    for bad in (_lib.PLAN_L2_BASE, _lib.plan_l2(3), _lib.plan_l2(16)):            # cluster sizes other than 1/2/4/8
        assert min(_plan_bytes(m, 802, bad)) < 0, bad
    assert min(_plan_bytes(_cpu_model(256, in0=8, layers=8), 802, _lib.plan_l2(8))) > 0   # any R <= 256, up to 8 layers
    assert min(_plan_bytes(_cpu_model(257), 802, _lib.plan_l2(2))) < 0


def test_l2_plan_rejected_by_cluster_only_entry_points():
    """the one-launch train kernel and the list images exist for the relation-space plans only; the forward and
    backward refuse the plan's shape errors before they touch a device pointer"""
    lib = _lib.load()
    m = _cpu_model(5)
    c = ctypes.byref(m._cmodel)
    img = _lib.Stage()
    S = _lib.Saved()
    S.zsave = 16                              # (only tested for NULL)
    D = _lib.Dropout()
    A = _lib.Adj()
    for cs in (1, 2, 4, 8):
        p = _lib.plan_l2(cs)
        assert lib.igmc_stage_plan(c, 802, p, 0, ctypes.byref(img)) < 0
        assert lib.igmc_stage_plan(c, 802, p, 1, ctypes.byref(img)) < 0
        assert lib.igmc_forward_backward(c, None, None, None, None, ctypes.byref(A), 1, 802, ctypes.byref(D),
                                         ctypes.byref(S), None, 1.0, None, None, None, None, p, None, None, None,
                                         None) == -16
        # backward without its scratch buffers
        assert lib.igmc_backward(c, None, None, None, None, ctypes.byref(A), 1, 802, ctypes.byref(D), ctypes.byref(S),
                                 None, None, None, p, None, None, None) == -17
        assert lib.igmc_forward(c, None, None, None, None, ctypes.byref(A), 1, _lib.L2_MAX_NODES + 1, ctypes.byref(D),
                                0, ctypes.byref(S), None, 0.0, None, None, p, None, None, None) == -3
    assert _lib.ERR_NAMES[6].startswith("subgraph of more than 65535 nodes")


def _old_rule(m, n_cap, B, sms):
    """the plan rule before the L2 plan existed (None where it raised)"""
    lib, c = _lib.load(), ctypes.byref(m._cmodel)
    if n_cap > 256 and m.num_relations <= 12:
        cands = [4, 3, 2, 1, 0]
    else:
        cands = [cl for cl in (4, 2, 1) if B * cl <= sms or cl == 1] + [0]
    for cl in cands:
        if lib.igmc_model_plan(c, n_cap, cl, 0) > 0 and lib.igmc_model_plan(c, n_cap, cl, 1) > 0:
            return cl
    return None


N_CAPS = sorted(set(list(range(2, 1201, 40)) + [256, 257, 382, 383, 422, 423, 434, 435, 446, 447, 568, 569, 1200]))


@pytest.mark.parametrize("R", [1, 5, 10, 12, 13, 71, 256])
def test_select_plan_keeps_existing_plans(R):
    """wherever an existing plan fits, the rule picks it as before; everywhere else it picks the L2 plan"""
    l2_seen = 0
    for NB in (2, 4):
        for in0 in (4, 6, 8):
            m = _cpu_model(R, in0=in0, nb=NB)
            for B in (16, 50):
                for n_cap in N_CAPS:
                    old = _old_rule(m, n_cap, B, SMS)
                    new = select_plan(m._cmodel, n_cap, B, SMS)
                    if old is not None:
                        assert new == old, (R, NB, in0, B, n_cap, old, new)
                    else:
                        assert new == _lib.plan_l2(l2_cluster(n_cap, B, SMS)), (R, NB, in0, B, n_cap, new)
                        l2_seen += 1
    assert l2_seen > 0


def test_select_plan_forced_and_refused():
    m = _cpu_model(5)
    assert select_plan(m._cmodel, 402, 50, SMS, want=_lib.plan_l2(4)) == _lib.plan_l2(4)
    assert select_plan(m._cmodel, 402, 50, SMS, want=0) == 0
    with pytest.raises(RuntimeError, match="no kernel plan fits"):
        select_plan(m._cmodel, _lib.L2_MAX_NODES + 1, 50, SMS)


def test_l2_cluster_rule():
    assert l2_cluster(1476, 50, SMS) == 8          # 400 CTAs: four per SM at most
    assert l2_cluster(1476, 100, SMS) == 4
    assert l2_cluster(8000, 3, SMS) == 8
    assert l2_cluster(802, 50, SMS) == 8
    assert l2_cluster(300, 16, SMS) == 4           # every CTA keeps one 64-node tile
    assert l2_cluster(100, 16, SMS) == 1
    assert l2_cluster(1476, 600, SMS) == 1
    for B in (1, 16, 50, 64, 128, 512):
        for n_cap in (2, 100, 600, 1476, 9000):
            c = l2_cluster(n_cap, B, SMS)
            assert c in (1, 2, 4, 8) and (c == 1 or B * c <= 4 * SMS)
