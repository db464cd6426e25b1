"""Small end-to-end exercise of every kernel (smoke())."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(verbose=True):
    from igmc_b200.data import make_synthetic_dataset
    from igmc_b200.models import IGMC, FusedAdam
    from igmc_b200.train_eval import TrainEngine, eval_rmse
    from igmc_b200.util_functions import MyDynamicDataset
    from oracle import extract_np, pyg_restated

    ds = make_synthetic_dataset("tiny", seed=0)
    tu, tv, tl = ds["train"]
    d = MyDynamicDataset(None, ds["adj_train"], (tu, tv), tl, 1, 1.0, 10, None, None, ds["class_values"], seed=3)
    idx = np.arange(8)
    b = d.extract_batch(idx)
    g = extract_np.RatingCSR(ds["adj_train"])
    ob = extract_np.extract_batch(g, tu[idx], tv[idx], tl[idx], ds["class_values"], 1, 1.0, 10, seed=3, pair_ids=idx)
    ok_extract = (np.array_equal(b.edge_index.cpu().numpy(), ob["edge_index"])
                  and np.array_equal(b.edge_type.cpu().numpy(), ob["edge_type"])
                  and np.array_equal(b.x.cpu().numpy(), ob["x"]))
    torch.manual_seed(0)
    ref = pyg_restated.IGMCRef(4, (32, 32, 32, 32), 5, 4, 0.0).eval()
    m = IGMC(d, latent_dim=[32] * 4, num_relations=5, num_bases=4, regression=True, adj_dropout=0.0).cuda()
    m.load_state_dict(ref.state_dict())
    m.eval()
    tb = pyg_restated.to_torch_batch(ob)
    with torch.no_grad():
        want = ref(tb["x"], tb["edge_index"], tb["edge_type"])
        got = m(b).cpu()
    rmse = float(torch.sqrt(torch.mean((got - want) ** 2)))
    m.train()
    opt = FusedAdam(m, lr=1e-3)
    eng = TrainEngine(d, m, opt, 8, ARR=0.001, use_graph=True)
    for s in range(4):
        eng.step(np.arange(s * 8, s * 8 + 8), epoch=1)
    eng.check()
    loss = float(eng.last_loss.item())
    # the production path: pipelined engine (extraction of the next batch + list images on the side branch behind the
    # launch-order gate, TMA-staged model kernels, one fused reduce -> exchange -> Adam kernel, zero-copy step I/O),
    # first eager, then as replayed CUDA graphs
    eng.prime(np.arange(32, 40), epoch=1)
    for s in range(6):
        eng.step_pipe(np.arange(40 + s * 8, 48 + s * 8) if s < 5 else None, epoch=1)
    eng.check()
    torch.cuda.synchronize()
    loss_pipe = eng.loss_of_update(eng._updates - 1) if eng.zero_copy and eng.exchange is not None else float(eng.last_loss)
    assert np.isfinite(loss_pipe) and bool(torch.isfinite(m.flat_params).all())
    if verbose:
        print("smoke: extract_exact=%s forward_rmse=%.3e train_loss=%.4f pipelined_loss=%.4f" % (
            ok_extract, rmse, loss, loss_pipe))
    assert ok_extract, "extraction differs from the oracle"
    assert rmse <= 1e-4, "forward differs from the oracle: %g" % rmse
    assert np.isfinite(loss)
    return dict(extract_exact=ok_extract, forward_rmse=rmse, train_loss=loss)


if __name__ == "__main__":
    main()
