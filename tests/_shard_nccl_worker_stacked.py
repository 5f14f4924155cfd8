"""torchrun worker of tests/test_gpu_lstm_stacked.py::test_sharded_model_with_stacked_lstm_matches_the_whole_model (row shard,
one rank per GPU, NCCL): the sharded model with lstm_num_layers = 2 against the whole model on this GPU at the same precision."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import MPGCN as shim  # noqa: E402
from mpgcn_b200 import dist as mdist, shard  # noqa: E402
from oracle import mpgcn_oracle as orc  # noqa: E402


def main(out_path):
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    rank, world = mdist.init_from_env("nccl", device=dev)
    if not dist.is_initialized():      # world 1: init_from_env leaves the group to the caller; the row shard's collectives need one
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
    N, K, B = 40, 3, 2
    rng = np.random.default_rng(1)
    G = torch.from_numpy(orc.adj_process(rng.random((1, N, N)).astype(np.float32), "random_walk_diffusion", K - 1)[0].astype(np.float32)).to(dev)
    go = torch.from_numpy((rng.standard_normal((B, K, N, N)) / N ** 0.5).astype(np.float32))
    gd = torch.from_numpy((rng.standard_normal((B, K, N, N)) / N ** 0.5).astype(np.float32))
    plan = shard.ShardPlan("row", rank, world, N, K)
    rows = []
    # (hidden, T, precision, forward / gradient bars of test_gpu_shard.py): the tensor-core stacks at 32 and 96, and hidden 64 at
    # T = 16, which the model runs on nn.LSTM (the fp32 kernels' backward does not hold 16 steps at 64)
    for hid, T, prec, tol_f, tol_g in ((32, 5, "fp16", 1e-3, 8e-2), (96, 4, "fp16", 1e-3, 8e-2), (64, 16, "auto", 1e-5, 2e-3)):
        torch.manual_seed(hid)
        model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=2, gcn_hidden_dim=32, gcn_num_layers=3,
                           num_nodes=N, user_bias=True, activation=nn.ReLU).to(dev)
        with torch.no_grad():      # keep both heads alive whatever the init draws
            for m in range(2):
                model.branch_models[m]['fc'][0].bias.add_(0.5)
        model.lstm_precision = prec
        for mod in model.modules():
            if isinstance(mod, shim.BDGCN):
                mod.precision = "fp32"
        x = torch.from_numpy((rng.random((B, T, N, N, 1)) * 6).astype(np.float32))
        y = torch.from_numpy((rng.random((B, 1, N, N, 1)) * 2).astype(np.float32))
        model.zero_grad(set_to_none=True)
        pred_w = model(x_seq=x.to(dev), G_list=[G, (go.to(dev), gd.to(dev))])
        nn.functional.mse_loss(pred_w, y.to(dev)).backward()
        want = {k: p.grad.clone() for k, p in model.named_parameters()}
        model.zero_grad(set_to_none=True)
        xs, ys, gos, gds = (t.to(dev) for t in shard.shard_host_inputs(plan, x, y, go, gd))
        pred = shard.sharded_forward(model, plan, xs, G, (gos, gds))
        shard.sharded_mse_loss(plan, pred, ys).backward()
        shard.allreduce_sum_gradients(list(model.parameters()), plan, model)
        torch.cuda.synchronize()
        ref_pred = pred_w[:, :, plan.row_lo:plan.row_hi]
        linf, l2 = orc.rel_errors(pred.detach().cpu().numpy(), ref_pred.detach().cpu().numpy())
        rows.append(dict(hid=hid, what=f"nccl world-{world} row shard, L=2 hidden {hid}: y (rank {rank})", linf=linf, l2=l2, tol=tol_f))
        for k, p in model.named_parameters():
            linf, l2 = orc.rel_errors(p.grad.cpu().numpy(), want[k].cpu().numpy())
            rows.append(dict(hid=hid, what=f"nccl world-{world} row shard, L=2 hidden {hid}: grad {k} (rank {rank})", linf=l2, l2=l2, tol=tol_g))
    gathered = [None] * world
    dist.all_gather_object(gathered, rows)
    if rank == 0:
        json.dump({"rows": [r for part in gathered for r in part]}, open(out_path, "w"))
    dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
