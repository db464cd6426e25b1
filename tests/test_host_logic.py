"""CPU tests of the host-side mirror of the reference API (no kernels run here)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import pyg_restated
from igmc_b200.models import IGMC, FusedAdam, edge_keep_reference, hidden_keep_reference, splitmix64
from igmc_b200.train_eval import shard_batches


def test_state_dict_keys_match_reference_names():
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True)
    ref = pyg_restated.IGMCRef(4, (32, 32, 32, 32), 5, 4)
    assert sorted(m.state_dict().keys()) == sorted(ref.state_dict().keys())
    for k, v in ref.state_dict().items():
        assert tuple(m.state_dict()[k].shape) == tuple(v.shape), k
    # PyG-1.4.2 init bound 1/sqrt(num_bases*in) and parameter count 49,233 (SURVEY.md A.6)
    assert sum(p.numel() for p in m.parameters()) == 49233
    assert float(m.convs[0].basis.abs().max()) <= 0.25 and float(m.convs[1].basis.abs().max()) <= 1 / np.sqrt(128)
    m.load_state_dict(ref.state_dict())
    assert torch.equal(m.convs[2].att, ref.convs[2].att)


def test_flat_bucket_aliases_parameters():
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True)
    for (o, n, s), (_, _, p) in zip(m._layout, m._named_order()):
        assert o % 4 == 0                                   # 16-byte aligned slices for float4 access
        assert p.data_ptr() == m.flat_params[o:o + n].data_ptr()
    with torch.no_grad():
        m.lin2.bias.fill_(3.0)
    assert float(m.flat_params[m._cmodel.off_lin2_b]) == 3.0
    m2 = m.double().float()                                  # _apply re-flattens and keeps values
    assert float(m2.flat_params[m2._cmodel.off_lin2_b]) == 3.0
    opt = FusedAdam(m, lr=1e-3)
    sd = opt.state_dict()
    assert len(sd["state"]) == len(list(m.parameters())) and sd["param_groups"][0]["lr"] == 1e-3
    assert set(sd["state"][0]) >= {"step", "exp_avg", "exp_avg_sq"}


def test_unsupported_options_fail_loudly():
    with pytest.raises(NotImplementedError):
        IGMC(4, regression=False)
    with pytest.raises(NotImplementedError):
        IGMC(4, regression=True, side_features=True)
    with pytest.raises(NotImplementedError):
        IGMC(4, regression=True, latent_dim=[32, 32, 32, 1])


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_no_cpu_fallback():
    from igmc_b200.data import make_synthetic_dataset
    from igmc_b200.util_functions import MyDynamicDataset
    ds = make_synthetic_dataset("tiny")
    with pytest.raises(RuntimeError, match="CUDA"):
        MyDynamicDataset(None, ds["adj_train"], ds["train"][:2], ds["train"][2], 1, 1.0, 10, None, None,
                         ds["class_values"])


def test_shard_batches_partition():
    perm = np.random.default_rng(0).permutation(1037)
    for world in (1, 2, 4, 8):
        per_rank = [shard_batches(perm, 50, r, world) for r in range(world)]
        steps = len(per_rank[0])
        assert all(len(p) == steps for p in per_rank)
        seen = []
        for s in range(steps):
            G = per_rank[0][s][1]
            assert all(p[s][1] == G for p in per_rank)
            assert sum(len(p[s][0]) for p in per_rank) == G
            if s < steps - 1:
                assert all(len(p[s][0]) == 50 for p in per_rank)
            seen += [x for p in per_rank for x in p[s][0]]
        assert sorted(seen) == sorted(perm.tolist())


def test_edge_keep_reference_rate():
    k = edge_keep_reference(splitmix64(7), 4000, 0.2)
    assert 0.76 < float(k.float().mean()) < 0.84


def test_hidden_keep_reference_rate():
    k = hidden_keep_reference(splitmix64(7), 50, 0.5)
    assert k.dtype == torch.bool and k.shape == (50, 128)
    assert 0.45 < float(k.float().mean()) < 0.55
    # its own stream: not the edge draw of the same seed
    assert not torch.equal(k.view(-1), edge_keep_reference(splitmix64(7), 50 * 128, 0.5))
    assert bool(hidden_keep_reference(3, 2, 0.0).all()) and not bool(hidden_keep_reference(3, 2, 1.0).any())


def _dp_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import extract_np
    from igmc_b200.data import synth_ratings, build_adj
    u, v, lab = synth_ratings(60, 50, 700, 5, 1)
    g = extract_np.RatingCSR(build_adj(u, v, lab, 60, 50))
    cv = np.arange(1, 6, dtype=np.float32)
    B, G = 6, 6 * world
    perm = np.arange(G)
    mine, Gs = shard_batches(perm, B, rank, world)[0]
    torch.manual_seed(0)
    model = pyg_restated.IGMCRef(4, (32, 32, 32, 32), 5, 4, 0.0).double().eval()
    # this rank's contribution: sum over its graphs of (out-y)^2 / G, + ARR * reg on rank 0 only (TrainEngine.arr_local:
    # the regulariser enters once per global batch, also when a short tail batch leaves other ranks empty)
    ob = extract_np.extract_batch(g, u[mine], v[mine], lab[mine], cv, 1, 1.0, 20, pair_ids=mine)
    tb = pyg_restated.to_torch_batch(ob, torch.float64)
    pred = model(tb["x"], tb["edge_index"], tb["edge_type"])
    loss = ((pred - tb["y"]) ** 2).sum() / Gs + (0.001 if rank == 0 else 0.0) * pyg_restated.arr_regulariser(model)
    loss.backward()
    flat = torch.cat([p.grad.reshape(-1) for p in model.parameters()])
    dist.all_reduce(flat)                                    # the one collective of a step
    if rank == 0:
        model.zero_grad()
        ob = extract_np.extract_batch(g, u[perm], v[perm], lab[perm], cv, 1, 1.0, 20, pair_ids=perm)
        tb = pyg_restated.to_torch_batch(ob, torch.float64)
        full, _ = pyg_restated.train_loss(model, tb, 0.001)
        full.backward()
        want = torch.cat([p.grad.reshape(-1) for p in model.parameters()])
        out.put(float((flat - want).abs().max() / want.abs().max()))
    dist.destroy_process_group()


def test_data_parallel_gradient_identity_gloo():
    """world_size 2 on CPU (gloo): all-reduce(SUM) of per-rank gradients with the loss scaled by the GLOBAL
    batch and ARR on rank 0 equals the single-process gradient of the concatenated batch (SURVEY.md §8e)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert out.get(timeout=5) < 1e-9


def test_dgcnn_rs_bucket_layout_and_state_dict():
    """DGCNN_RS (reference models.py:123-167): reference state_dict keys / shapes, the narrow last R-GCN layer lives
    padded in the flat bucket (unused columns zero, also after reset_parameters), optimizer state round-trips."""
    from oracle.pyg_restated import DGCNN_RSRef
    from igmc_b200.models import DGCNN_RS, FusedAdam
    torch.manual_seed(0)
    ref = DGCNN_RSRef(4, (32, 32, 32, 1), 30, 5, 4, 0.2)
    m = DGCNN_RS(4, latent_dim=[32, 32, 32, 1], k=30, num_relations=5, num_bases=4, regression=True)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == \
        {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    assert m.dense_dim == ref.dense_dim == (30 // 2 - 5 + 1) * 32
    m.load_state_dict(ref.state_dict())
    for name, p in m.named_parameters():
        assert torch.equal(p.detach(), dict(ref.named_parameters())[name].detach()), name
    padded = [e for e in m._layout if len(e) == 4]
    assert len(padded) == 3                                   # basis, root, bias of the 32 -> 1 layer
    m.reset_parameters()
    for e in padded:
        slot = m.flat_params[e[0]:e[0] + e[1]].view(e[3])
        assert float(slot[..., e[2][-1]:].abs().max()) == 0.0
        assert float(slot[..., :e[2][-1]].abs().max()) > 0.0
    assert m._cmodel.readout == 1 and m._csort.param_begin == m._cmodel.conv_param_count
    assert m._csort.param_end == m.flat_params.numel()
    opt = FusedAdam(m, lr=1e-3)
    opt.load_state_dict(opt.state_dict())
    # percentile k (models.py:69-73) on a stand-in dataset
    class DS(list):
        num_features = 4
    class G(object):
        def __init__(self, n):
            self.num_nodes = n
    ds = DS([G(n) for n in (5, 50, 20, 30, 40, 12, 60, 33, 47, 25)])
    m2 = DGCNN_RS(ds, latent_dim=[32, 32, 32, 1], k=0.6, num_relations=5, num_bases=4, regression=True)
    assert m2.k == sorted(g.num_nodes for g in ds)[int(np.ceil(0.6 * len(ds))) - 1]


def test_fused_adam_state_dict_loads_into_torch_adam():
    """an optimizer checkpoint written by FusedAdam must load into the reference's torch.optim.Adam (Main.py:45,
    train_eval.py:60-62): independent per-parameter `step`s (shared storage would be incremented once per
    parameter by torch's step()), contiguous moments of the parameters' shapes"""
    import io
    from igmc_b200.models import IGMC, FusedAdam
    torch.manual_seed(0)
    m = IGMC(4, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True)
    opt = FusedAdam(m, lr=1e-3)
    opt.step_count[0] = 7
    opt.exp_avg.uniform_(-1e-3, 1e-3)
    opt.exp_avg_sq.uniform_(1e-8, 1e-6)
    buf = io.BytesIO()
    torch.save(opt.state_dict(), buf)
    sd = torch.load(io.BytesIO(buf.getvalue()))
    steps = [st["step"] for st in sd["state"].values()]
    assert len(steps) == 20 and len({t.untyped_storage().data_ptr() for t in steps}) == 20
    params = [torch.nn.Parameter(p.detach().clone()) for p in m.parameters()]
    ref = torch.optim.Adam(params, lr=1e-3)
    ref.load_state_dict(sd)
    for p in params:
        p.grad = torch.full_like(p, 1e-3)
    ref.step()
    assert all(float(ref.state[p]["step"]) == 8.0 for p in params)          # 7 -> 8, not 7 -> 7 + 20
    for p, q in zip(params, m.parameters()):
        assert ref.state[p]["exp_avg"].shape == q.shape and ref.state[p]["exp_avg"].is_contiguous()
    # and back into FusedAdam
    opt2 = FusedAdam(m, lr=1e-3)
    opt2.load_state_dict(torch.load(io.BytesIO(buf.getvalue())))   # (torch's Adam stepped the tensors of `sd` in place)
    assert int(opt2.step_count[0]) == 7
    for p in m.parameters():   # (the flat buffers also hold alignment padding that is not part of any state entry)
        assert torch.equal(opt2.state[p]["exp_avg"], opt.state[p]["exp_avg"])
        assert torch.equal(opt2.state[p]["exp_avg_sq"], opt.state[p]["exp_avg_sq"])


def test_balanced_dealing_partitions_and_balances():
    """deal_balanced / shard_batches(cost=...): every pair of every global batch goes to exactly one rank, rank sizes
    differ by at most one, the same global batches as the contiguous split, and the ranks' largest costs are close"""
    from igmc_b200.train_eval import deal_balanced
    rng = np.random.default_rng(0)
    n, B = 1003, 50
    perm = rng.permutation(n)
    cost = rng.lognormal(0, 1, n)
    for world in (2, 4, 8):
        per_rank = [shard_batches(perm, B, r, world, cost) for r in range(world)]
        plain = [shard_batches(perm, B, r, world) for r in range(world)]
        for step in range(len(per_rank[0])):
            got = np.concatenate([per_rank[r][step][0] for r in range(world)])
            want = np.concatenate([plain[r][step][0] for r in range(world)])
            assert sorted(got.tolist()) == sorted(want.tolist())
            sizes = [len(per_rank[r][step][0]) for r in range(world)]
            assert max(sizes) - min(sizes) <= 1 and per_rank[0][step][1] == plain[0][step][1]
            if sizes[0] == B:
                tops = [cost[per_rank[r][step][0]].max() for r in range(world)]
                srt = np.sort(cost[got])[::-1]
                assert min(tops) >= srt[world - 1] - 1e-12          # each rank holds one of the `world` largest
    parts = deal_balanced(np.arange(7), np.array([5, 1, 4, 2, 3, 0, 6.0]), 3)
    assert sorted(np.concatenate(parts).tolist()) == list(range(7)) and [len(p) for p in parts] == [3, 2, 2]
