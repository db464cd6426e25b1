"""Train-step parity at the FULL batch of every BASELINE config (VERDICT r1 task 4): predictions, loss and every
parameter gradient of the fused kernels against fp64 autograd of the restated oracle, on the batches the CUDA
extractor produces, with the kernels' own hash dropout draws.

The oracle runs in its memory-light "transform" message formulation (pinned against the reference-era gather + bmm
formulation by tests/test_oracle_model.py); tolerances as everywhere: ratings 1e-4 RMSE, gradients 2e-4 relative."""
import numpy as np
import pytest
import torch

from oracle import extract_np, pyg_restated
from tests.helpers import check_step

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name,mnph,B,plan", [("ml_100k", 200, 50, "auto"), ("ml_1m", 100, 50, "auto"),
                                              ("ml_1m", 100, 50, 3), ("ml_1m_r02", 100, 256, 1)])
def test_full_batch_train_step_parity_dynamic(name, mnph, B, plan):
    """configs 1/2 (ml_100k* batch 50, edge dropout 0.2), 4 (ml_1m* batch 50) and 5 (ml_1m* ratio 0.2, batch 256,
    one CTA per subgraph): extraction bit-exact vs the oracle, then the whole train step"""
    from igmc_b200.data import make_synthetic_dataset
    from igmc_b200.models import IGMC
    from igmc_b200.util_functions import MyDynamicDataset
    ds = make_synthetic_dataset(name, seed=0)
    tu, tv, tl = ds["train"]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, mnph, None, None, ds["class_values"], seed=11)
    idx = np.random.default_rng(5).choice(len(tu), B, replace=False)
    b = d.extract_batch(idx)
    g = extract_np.RatingCSR(ds["adj_train"])
    ob = extract_np.extract_batch(g, tu[idx], tv[idx], tl[idx], ds["class_values"], 1, 1.0, mnph, seed=11, pair_ids=idx)
    assert np.array_equal(b.edge_index.cpu().numpy(), ob["edge_index"])
    assert np.array_equal(b.edge_type.cpu().numpy(), ob["edge_type"])
    torch.manual_seed(0)
    ref = pyg_restated.set_formulation(
        pyg_restated.IGMCRef(4, (32, 32, 32, 32), 5, 4, ds["adj_dropout"]).double().train(), "transform")
    m = IGMC(d, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True,
             adj_dropout=ds["adj_dropout"]).cuda().train()
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    m.kernel_plan = plan
    hk = torch.rand(B, 128, generator=torch.Generator().manual_seed(2)) > 0.5
    check_step(m, ref, b, ob, 0.001, ds["adj_dropout"], hk)
    if plan == "auto":
        # batch 50: two CTAs per subgraph; four for the 402-node subgraphs of ml_100k* (edge lists must fit in shared
        # memory next to the node features)
        assert m._plan(b) == (4 if b._priv["n_cap"] > 256 else 2)
    # the same step with the list images of the pipelined engine: bit-identical gradient
    g0 = m.flat_grad.clone()
    m._step = 31
    m.stage_batch(b, True, m.make_dropout(True))
    m._step = 30
    m.fused_step(b, ARR=0.001, hidden_keep=hk)
    assert torch.equal(m.flat_grad, g0)


def test_full_batch_train_step_parity_flixster_static():
    """config 3: REAL flixster split, R = 10 (the 1024-thread kernel instantiation), static MyDataset store, batch 50,
    edge dropout 0.2"""
    from igmc_b200.data import make_synthetic_dataset
    from igmc_b200.models import IGMC
    from igmc_b200.util_functions import MyDataset
    ds = make_synthetic_dataset("flixster", seed=0)
    tu, tv, tl = ds["train"]
    n = 400
    d = MyDataset(None, ds["adj_train"], (tu[:n], tv[:n]), tl[:n], 1, 1.0, ds["max_nodes_per_hop"], None, None,
                  ds["class_values"])
    idx = np.random.default_rng(1).choice(n, 50, replace=False)
    b = d.extract_batch(idx)
    g = extract_np.RatingCSR(ds["adj_train"])
    ob = extract_np.extract_batch(g, tu[idx], tv[idx], tl[idx], ds["class_values"], 1, 1.0, ds["max_nodes_per_hop"],
                                  pair_ids=idx)
    assert np.array_equal(b.edge_index.cpu().numpy(), ob["edge_index"])
    R = ds["num_relations"]
    torch.manual_seed(0)
    ref = pyg_restated.set_formulation(
        pyg_restated.IGMCRef(4, (32, 32, 32, 32), R, 4, 0.2).double().train(), "transform")
    m = IGMC(d, latent_dim=[32] * 4, num_relations=R, num_bases=4, regression=True, adj_dropout=0.2).cuda().train()
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    hk = torch.rand(50, 128, generator=torch.Generator().manual_seed(3)) > 0.5
    check_step(m, ref, b, ob, 0.001, 0.2, hk)
    assert m._plan(b) > 0


def test_full_batch_dgcnn_rs_ml_1m():
    """DGCNN_RS (models.py:123-167) on a full ml_1m* batch: k from the reference's 0.6-percentile rule over ALL
    subgraphs of a 3000-pair dataset (the ``for g in dataset`` count, models.py:70-72), train step vs fp64 oracle"""
    from igmc_b200.data import make_synthetic_dataset
    from igmc_b200.models import DGCNN_RS, edge_keep_reference, splitmix64   # noqa: F401
    from igmc_b200.util_functions import MyDynamicDataset
    ds = make_synthetic_dataset("ml_1m", seed=0)
    tu, tv, tl = ds["train"]
    n = 3000
    d = MyDynamicDataset(None, ds["adj_train"], (tu[:n], tv[:n]), tl[:n], 1, 1.0, 100, None, None, ds["class_values"],
                         seed=4)
    m = DGCNN_RS(d, latent_dim=[32, 32, 32, 1], k=0.6, num_relations=5, num_bases=4, regression=True,
                 adj_dropout=0.0).cuda().train()
    counts = np.sort(d.node_counts())
    assert m.k == max(10, int(counts[int(np.ceil(0.6 * n)) - 1]))
    idx = np.arange(50)
    b = d.extract_batch(idx)
    g = extract_np.RatingCSR(ds["adj_train"])
    ob = extract_np.extract_batch(g, tu[idx], tv[idx], tl[idx], ds["class_values"], 1, 1.0, 100, seed=4, pair_ids=idx)
    torch.manual_seed(0)
    ref = pyg_restated.set_formulation(
        pyg_restated.DGCNN_RSRef(4, (32, 32, 32, 1), m.k, 5, 4, 0.0).double().train(), "transform")
    m.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    hk = torch.rand(50, 128, generator=torch.Generator().manual_seed(2)) > 0.5
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    out_ref = ref(tb["x"], tb["edge_index"], tb["edge_type"], tb["batch"], None, hk, tb["num_graphs"])
    loss_ref = torch.nn.functional.mse_loss(out_ref, tb["y"].view(-1)) + 0.001 * pyg_restated.arr_regulariser(ref)
    loss_ref.backward()
    loss = m.fused_step(b, ARR=0.001, hidden_keep=hk)
    b.check()
    ws = next(iter(v for k, v in m._ws.items() if k[2]))
    rmse = float(torch.sqrt(torch.mean((ws["sp"]["pred"].double().cpu() - out_ref.detach()) ** 2)))
    assert rmse <= 1e-4, rmse
    assert abs(float(loss) - float(loss_ref)) <= 1e-4 * max(1.0, abs(float(loss_ref)))
    names = {id(p): nme for nme, p in m.named_parameters()}
    sd_ref = dict(ref.named_parameters())
    table = []
    for e, (_, _, p) in zip(m._layout, m._named_order()):
        gref = sd_ref[names[id(p)]].grad
        ggpu = m._pview(m.flat_grad, e).double().cpu()
        table.append((names[id(p)], float((ggpu - gref).abs().max()), float(gref.abs().max())))
    gmax = max(t[2] for t in table)
    for name, err, scale in table:
        # relative to the tensor's own largest entry, plus an fp32 noise floor: the first-layer att gradient is a sum of
        # O(1) products that cancel to 1e-3 of the model's largest gradient (measured: |att grad| 7e-3 next to 7.1),
        # so its attainable accuracy is a few ulp of the SUMMANDS, i.e. ~1e-6 of the largest gradient
        assert err <= 3e-4 * scale + 2e-6 * gmax, (name, err, scale, gmax, table)


def test_dataset_iteration_idiom_and_bounds():
    """``for g in dataset`` / ``dataset[i]`` (reference models.py:71, train_eval.py:266-267): iteration stops after
    len(dataset) graphs, negative indices count from the end, out-of-range indices raise IndexError (both datasets)"""
    from igmc_b200.data import make_synthetic_dataset
    from igmc_b200.util_functions import MyDataset, MyDynamicDataset
    ds = make_synthetic_dataset("tiny", seed=0)
    tu, tv, tl = ds["train"]
    n = 23
    for cls in (MyDynamicDataset, MyDataset):
        d = cls(None, ds["adj_train"], (tu[:n], tv[:n]), tl[:n], 1, 1.0, 10, None, None, ds["class_values"])
        nodes = [g.num_nodes for g in d]
        assert len(nodes) == n and nodes == [int(v) for v in d.node_counts()]
        assert torch.equal(d[-1].edge_index, d[n - 1].edge_index) and d[0].num_nodes == nodes[0]
        for bad in (n, n + 5, -n - 1):
            with pytest.raises(IndexError):
                d[bad]
