"""Element-by-element fp32 error bounds of the model kernels, one layer at a time (tests/error_bounds.py).

Each case runs an eval forward and a train step (``fused_step``: the kernels' own hash edge and hidden dropout, ARR
0.001, the gradient assembled by ``_launch_grad_reduce``; one case runs the one-launch train kernel of the train
engine instead) and checks every layer's states, the predictions, ``d hid`` and ``flat_grad`` against fp64
recomputations from the kernel's own inputs:

    |got - ref| <= KAPPA[quantity] * 2^-24 * M   per element,   got == 0 exactly where M == 0,

a NaN anywhere fails, and every ReLU, dropout, MaxPool and sort-pool branch the kernel took away from its kink must be
the one the fp64 value takes.

The suite's other bars (RMSE over a batch, error relative to a tensor's largest gradient) let one wrong graph, node
or small gradient entry through; these do not.  Each check prints its largest err / (u M)."""
import numpy as np
import pytest
import torch

from igmc_b200 import _lib
from tests import error_bounds as eb
from tests.helpers import REGIMES
from tests.test_gpu_model import _gpu_batch, _oracle_batch
from tests.test_gpu_regimes import _dense, _extracted, _images, _matrix, _ml_100k

pytestmark = pytest.mark.gpu


def _igmc(in0, R, NB=4, plan="auto", adj_dropout=0.2, rgcn="pyg-1.4"):
    from tests.test_gpu_relation_mean import _models
    return _models(in0, R, NB=NB, adj_dropout=adj_dropout, plan=plan, rgcn=rgcn)[1]


def _dgcnn(k, last, plan, NB=4):
    from tests.test_gpu_dgcnn import _models
    return _models(5, NB, k, adj_dropout=0.2, plan=plan, last=last)[1]


def _small(R=5, h=1):
    ob = _oracle_batch(R=R, h=h)[3]
    return _gpu_batch(ob), ob


def _ml_1m_full():
    from tests.test_gpu_large_subgraphs import _ml_1m
    ds = _ml_1m()
    tu, tv, tl = ds["train"]
    idx = np.arange(50)
    return _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, 1, 100)


def _ml_100k_batch(h, mnph, B):
    ds = _ml_100k()
    tu, tv, tl = ds["train"]
    idx = np.arange(B)
    return _extracted(ds["adj_train"], (tu[idx], tv[idx], tl[idx]), 5, h, mnph)


def _bwd_chunks_past_xch():
    r = REGIMES["bwd_chunks_past_xch"]
    A, (u, v, lab) = _matrix([_dense(150, 150, 0.75, r["R"], 1)], 150, 150)
    pick = np.random.default_rng(0).choice(len(u), 4, replace=False)
    b, ob = _extracted(A, (u[pick], v[pick], lab[pick]), r["R"], 1, 100)
    assert b._priv["n_cap"] == r["n_cap"]
    return b, ob


def _many_relations():
    from tests.test_gpu_large_subgraphs import _many_relations_batch
    return _many_relations_batch()[1:]


def _scaled(m, s=4.0):
    """every conv parameter times s: saturated tanh, large pre-activations, sums that cancel"""
    with torch.no_grad():
        for c in m.convs:
            for p in c.parameters():
                p.mul_(s)
    m._prepped = False
    return m


def _chunked_staging(m, b):
    """ml_100k* mnph 200: 402-node subgraphs, and a CTA of plan 4 that owns more nodes than one backward staging chunk"""
    assert b._priv["n_cap"] == 402
    tabs, imgs = _images(m, b)
    b._stage = None
    assert int(tabs["bwd"][:, 3].max()) > imgs["bwd"].chunk


# case id -> (model builder, batch builder, expected plan)
CASES = {
    **{"oracle_batch_plan%d" % p: (lambda p=p: _igmc(4, 5, plan=p), _small, p) for p in (0, 1, 2, 3, 4)},
    "ml_1m_full_plan2": (lambda: _igmc(4, 5, plan=2), _ml_1m_full, 2),
    "ml_1m_full_plan2_one_launch": (lambda: _igmc(4, 5, plan=2), _ml_1m_full, 2),
    "ml_100k_mnph200_plan4": (lambda: _igmc(4, 5, plan=4), lambda: _ml_100k_batch(1, 200, 16), 4),
    "R12_plan1_ncap202": (lambda: _igmc(4, 12, plan=1), _bwd_chunks_past_xch, 1),
    "h2_plan2": (lambda: _igmc(6, 5, plan=2), lambda: _ml_100k_batch(2, 40, 4), 2),
    "h3_plan2": (lambda: _igmc(8, 5, plan=2), lambda: _ml_100k_batch(3, 25, 4), 2),
    "R13_plan0": (lambda: _igmc(4, 13, plan=0), lambda: _small(R=13), 0),
    "R71_l2_c1": (lambda: _igmc(4, 71, plan=_lib.plan_l2(1)), _many_relations, _lib.plan_l2(1)),
    "R71_l2_c8": (lambda: _igmc(4, 71, plan=_lib.plan_l2(8)), _many_relations, _lib.plan_l2(8)),
    **{"pyg2_plan%d" % p: (lambda p=p: _igmc(4, 5, plan=p, rgcn="pyg-2"), _small, p)
       for p in (2, 0, _lib.plan_l2(2))},
    **{"dgcnn_k%d_last%d" % (k, last): (lambda k=k, last=last: _dgcnn(k, last, 2), _small, 2)
       for k in (30, 80) for last in (1, 8)},
    **{"scaled4_plan%d" % p: (lambda p=p: _scaled(_igmc(4, 5, plan=p)), _small, p) for p in (2, 0)},
    # num_bases = 2, the default of the reference's IGMC and DGCNN_RS: the NB = 2 instantiation of every model kernel
    **{"nb2_oracle_batch_plan%d" % p: (lambda p=p: _igmc(4, 5, NB=2, plan=p), _small, p) for p in (0, 1, 2, 4)},
    "nb2_ml_1m_full_plan2_one_launch": (lambda: _igmc(4, 5, NB=2, plan=2), _ml_1m_full, 2),
    **{"nb2_R71_l2_c%d" % c: (lambda c=c: _igmc(4, 71, NB=2, plan=_lib.plan_l2(c)), _many_relations, _lib.plan_l2(c))
       for c in (1, 8)},
    **{"nb2_pyg2_plan%d" % p: (lambda p=p: _igmc(4, 5, NB=2, plan=p, rgcn="pyg-2"), _small, p)
       for p in (0, 2, _lib.plan_l2(2))},
    **{"nb2_dgcnn_k30_last1_plan%d" % p: (lambda p=p: _dgcnn(30, 1, p, NB=2), _small, p) for p in (2, _lib.plan_l2(2))},
}
# the regime a case is there for, asserted on its model and batch before the checks
REGIME = {"ml_100k_mnph200_plan4": _chunked_staging}
# cases whose train step runs the way the train engine runs it on cluster plans: forward, loss and backward in one
# launch (igmc_forward_backward), then the gradient assembly (igmc_grad_reduce)
ONE_LAUNCH = {"ml_1m_full_plan2_one_launch", "nb2_ml_1m_full_plan2_one_launch"}


def _ws(m, train):
    return next(v for k, v in m._ws.items() if k[2] == train)


def _report(case, mode, res):
    if "branches" in res:
        print("error bounds %-28s %-5s branches mismatched %d" % (case, mode, res["branches"]))
    for key, val in res.items():
        if key != "branches":
            r, pad, worst = val
            print("error bounds %-28s %-5s %-8s err/(uM) %9.3f  kappa %4g  nonzero-at-M=0 %d  worst %d"
                  % (case, mode, key, r, eb.kappa_of(key), pad, worst))
    return eb.violations(res)


@pytest.mark.parametrize("case", list(CASES))
def test_error_bounds(case, monkeypatch):
    from igmc_b200.models import edge_keep_reference, hidden_keep_reference, splitmix64
    build_model, build_batch, plan = CASES[case]
    b, ob = build_batch()
    m = build_model()
    REGIME.get(case, lambda m, b: None)(m, b)
    m.eval()
    with torch.no_grad():
        m(b)
    b.check()
    assert m._plan(b) == plan
    bad = _report(case, "eval", eb.check_device(m, ob, _ws(m, False), False))
    m.train()
    step = 30
    m._step = step
    seed = splitmix64(m.drop_seed + step + 1)      # the step's own draws (the step increments _step first)
    ek = edge_keep_reference(seed, ob["edge_index"].shape[1], m.adj_dropout)
    hk = hidden_keep_reference(seed, b.num_graphs, m.hidden_dropout_p)
    if case in ONE_LAUNCH:
        monkeypatch.setenv("IGMC_FUSED_FB", "1")
        assert m.fused_update_ok(b)
        saved = m.forward_backward(b)
        m._launch_grad_reduce(b, saved, loss_scale=1.0 / b.num_graphs, arr=0.001)
    else:
        m.fused_step(b, ARR=0.001)
    b.check()
    bad += _report(case, "train", eb.check_device(m, ob, _ws(m, True), True, ek, 0.001, hk))
    assert not bad, bad
