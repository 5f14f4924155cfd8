"""torchrun worker of tests/test_gpu_lstm_widths.py::test_row_sharded_model_at_wide_hidden (one rank per GPU, NCCL): the row-shard
model (shard.sharded_forward, whose LSTM is the engine's on the rank's origin rows) at hidden 96 / 128 against the whole model.

    torchrun --nproc-per-node=W tests/_shard_nccl_worker_wide.py HIDDEN OUT.json
"""
import json
import os
import sys

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import MPGCN as shim  # noqa: E402
from mpgcn_b200 import dist as mdist, shard  # noqa: E402
from oracle import mpgcn_oracle as orc  # noqa: E402


def _set(model, lstm_prec, layer_prec):
    model.lstm_precision = lstm_prec
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = layer_prec


def main(hid, out_path):
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    rank, world = mdist.init_from_env("nccl", device=dev)
    if not torch.distributed.is_initialized():      # world 1: init_from_env leaves it to us; the shard's collectives need a group
        torch.distributed.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    N, K, T, B = 66, 3, 5, 2
    torch.manual_seed(0)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU).to(dev)
    with torch.no_grad():          # keep both heads alive whatever the init draws (an all-zero prediction would make the comparison vacuous)
        for m in range(2):
            model.branch_models[m]['fc'][0].bias.add_(0.5)
    rng = np.random.default_rng(1)
    x = torch.from_numpy((rng.random((B, T, N, N, 1)) * 6).astype(np.float32))
    y = torch.from_numpy((rng.random((B, 1, N, N, 1)) * 2).astype(np.float32))
    G = torch.from_numpy(orc.adj_process(rng.random((1, N, N)).astype(np.float32), "random_walk_diffusion", K - 1)[0].astype(np.float32)).to(dev)
    go = torch.from_numpy(orc.adj_process(rng.random((B, N, N)).astype(np.float32), "random_walk_diffusion", K - 1).astype(np.float32))
    gd = torch.from_numpy(orc.adj_process(rng.random((B, N, N)).astype(np.float32), "random_walk_diffusion", K - 1).astype(np.float32))
    plan = shard.ShardPlan("row", rank, world, N, K)
    xs, ys, gos, gds = (t.to(dev) for t in shard.shard_host_inputs(plan, x, y, go, gd))
    rows = []
    # the LSTM always on the tensor-core kernel (the sharded model has no nn.LSTM); the whole model at the same precisions is the
    # yardstick: fp32 layers -> summation order only; fp16 layers -> the fp16 row partials against the fp16 whole layer
    for layer_prec, tol_f, tol_g in (("fp32", 1e-5, 2e-3), ("fp16", 1e-3, 8e-2)):
        _set(model, "fp16", layer_prec)
        model.zero_grad(set_to_none=True)
        pred_w = model(x_seq=x.to(dev), G_list=[G, (go.to(dev), gd.to(dev))])
        assert float((pred_w > 0).float().mean()) > 0.5, "degenerate test case: the whole model's prediction is (almost) all zero"
        nn.functional.mse_loss(pred_w, y.to(dev)).backward()
        want = {k: p.grad.clone() for k, p in model.named_parameters()}
        model.zero_grad(set_to_none=True)
        pred = shard.sharded_forward(model, plan, xs, G, (gos, gds))
        loss = shard.sharded_mse_loss(plan, pred, ys)
        loss.backward()
        shard.allreduce_sum_gradients(list(model.parameters()), plan, model)
        torch.cuda.synchronize()
        ref_pred = pred_w[:, :, plan.row_lo:plan.row_hi]
        linf, l2 = orc.rel_errors(pred.detach().cpu().numpy(), ref_pred.detach().cpu().numpy())
        rows.append(dict(what=f"nccl world-{world} row shard hidden {hid}, lstm fp16, layers {layer_prec}: y (rank {rank})", linf=linf, l2=l2,
                         tol=tol_f))
        for k, p in model.named_parameters():
            linf, l2 = orc.rel_errors(p.grad.cpu().numpy(), want[k].cpu().numpy())
            rows.append(dict(what=f"nccl world-{world} row shard hidden {hid}, layers {layer_prec}: grad {k} (rank {rank})", linf=l2, l2=l2,
                             tol=tol_g))
    gathered = [None] * world
    torch.distributed.all_gather_object(gathered, rows)
    if rank == 0:
        json.dump({"rows": [r for part in gathered for r in part]}, open(out_path, "w"))
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main(int(sys.argv[1]), sys.argv[2])
