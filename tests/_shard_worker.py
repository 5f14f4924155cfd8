"""Worker of tests/test_shard_gloo.py: one rank of a world-2 gloo run of the sharded model (CPU stand-in engine).
Arguments: kind, output path[, lstm_hidden_dim, gcn_hidden_dim] (both 8 by default); kind "k-layer": one K-shard layer on a
static support stack instead of the model."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import MPGCN as shim  # noqa: E402
from mpgcn_b200 import dist as mdist, shard  # noqa: E402
from shard_standin import TorchEngine  # noqa: E402


def main(kind, out_path, lstm_hid=8, gcn_hid=8):
    rank, world = mdist.init_from_env("gloo")
    shard._ENGINE = TorchEngine()
    N, K, T, B = 8, 3, 3, 2
    torch.manual_seed(0)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=lstm_hid, lstm_num_layers=1, gcn_hidden_dim=gcn_hid, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU)
    with torch.no_grad():                       # non-zero biases so that the bias gradient path is exercised
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.05)
    rng = np.random.default_rng(1)
    x = torch.from_numpy((rng.random((B, T, N, N, 1)) * 4).astype(np.float32))
    y = torch.from_numpy(rng.random((B, 1, N, N, 1)).astype(np.float32))
    G = torch.from_numpy((rng.random((K, N, N)) / N).astype(np.float32))
    go = torch.from_numpy((rng.random((B, K, N, N)) / N).astype(np.float32))
    gd = torch.from_numpy((rng.random((B, K, N, N)) / N).astype(np.float32))
    n_groups, sample0 = 1, 0
    if kind == "rowhyb":          # hybrid: world = 4 = 2 batch groups x 2 row ranks (bench.py --shard row --row-ranks 2)
        R = 2
        n_groups = world // R
        groups = [dist.new_group(list(range(gi * R, (gi + 1) * R))) for gi in range(n_groups)]
        Bg = B // n_groups
        sample0 = (rank // R) * Bg
        x, y, go, gd = (t[sample0:sample0 + Bg] for t in (x, y, go, gd))
        plan = shard.ShardPlan("row", rank % R, R, N, K, group=groups[rank // R])
    else:
        plan = shard.ShardPlan(kind, rank, world, N, K)
    xs, ys, gos, gds = shard.shard_host_inputs(plan, x, y, go, gd)
    pred = shard.sharded_forward(model, plan, xs, G, (gos, gds))
    loss = shard.sharded_mse_loss(plan, pred, ys)
    loss.backward()
    params = list(model.parameters())
    shard.allreduce_sum_gradients(params, plan, model, over_world=n_groups > 1, scale=1.0 / n_groups)
    loss_all = loss.detach().clone()
    if kind in ("row", "rowhyb"):
        dist.all_reduce(loss_all)
        loss_all /= n_groups
    torch.save({"rank": rank, "pred": pred.detach(), "rows": (plan.row_lo, plan.row_hi), "sample0": sample0, "loss": float(loss_all),
                "grads": {k: p.grad.clone() for k, p in model.named_parameters()}}, out_path)
    dist.destroy_process_group()


def k_layer(out_path):
    """shard.sharded_bdgcn on a K shard with a static [K,N,N] stack (C != H), its parameter gradients summed over the ranks"""
    rank, world = mdist.init_from_env("gloo")
    shard._ENGINE = TorchEngine()
    B, N, K, C, H = 2, 8, 3, 4, 6
    torch.manual_seed(0)
    layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=H, use_bias=True, activation=nn.ReLU)
    with torch.no_grad():
        layer.b.add_(0.05)
    rng = np.random.default_rng(2)
    X = torch.from_numpy(rng.random((B, N, N, C)).astype(np.float32)).requires_grad_(True)
    G = torch.from_numpy((rng.random((K, N, N)) / N).astype(np.float32))
    d_out = torch.from_numpy(rng.standard_normal((B, N, N, H)).astype(np.float32))
    plan = shard.ShardPlan("k", rank, world, N, K)
    out = shard.sharded_bdgcn(layer, X, G, plan)
    (out * d_out).sum().backward()
    shard.allreduce_sum_gradients([layer.W, layer.b], plan)
    torch.save({"X": X.detach(), "G": G, "W": layer.W.detach(), "b": layer.b.detach(), "d_out": d_out, "out": out.detach(),
                "dX": X.grad, "dW": layer.W.grad, "db": layer.b.grad}, out_path)
    dist.destroy_process_group()


if __name__ == "__main__":
    if sys.argv[1] == "k-layer":
        k_layer(sys.argv[2])
    else:
        main(sys.argv[1], sys.argv[2], *(int(a) for a in sys.argv[3:5]))
