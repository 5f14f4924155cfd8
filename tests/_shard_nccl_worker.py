"""torchrun worker of the NCCL tests of the sharded model (test_gpu_shard.py, test_gpu_lstm_widths.py, test_gpu_lstm_stacked.py),
one rank per GPU: for each model of the spec, shard.sharded_forward, the loss and the gradient reduction against the whole model on
this GPU.  A test calls `run`; every row of the result holds `err` to `tol`: max(rel_Linf, rel_L2) for the prediction, rel_L2 for a
gradient (summation order and the handful of ReLU-mask flips it causes move single gradient elements by O(1))."""
import json
import os
import socket
import subprocess
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

# One model of a run.  cases: (LSTM precision, layer precision, forward bar, gradient bar); "follow" runs the LSTM at the layer
# precision.  yardstick: "fp32" -> the whole model on the fp32 engine for every case; "same" -> at the case's precisions.
# dynamic: the dynamic supports, dense N(0,1)/sqrt(N) stacks (no structure: the harshest case for the fp16 engine, DESIGN.md
# section 3) or random-walk diffusion like the static branch's (the trainer's kind of supports).
MODEL = dict(N=260, T=5, hidden=32, gcn_hidden=None, lstm_layers=1, seed=0, dynamic="dense", yardstick="fp32",
             cases=[("follow", "fp32", 1e-5, 2e-3), ("follow", "fp16", 1e-3, 8e-2)])


def run(world, tmp_path, models=({},), kind="row", peer=False):
    """This worker on `world` GPUs; `models`: overrides of MODEL, one per model.  kind "rowhyb": 2 batch groups x world/2 row
    ranks (bench.py --shard row --row-ranks).  peer: the row shard exchanges over peer memory.  -> rank 0's result"""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = tmp_path / "res.json"
    spec = json.dumps(dict(kind=kind, peer=peer, models=list(models)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
                        "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__), spec, str(out)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return json.load(open(out))


def _set(model, lstm_prec, layer_prec):
    model.lstm_precision = layer_prec if lstm_prec == "follow" else lstm_prec
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = layer_prec


def main(spec, out_path):
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    rank, world = mdist.init_from_env("nccl", device=dev)
    if not dist.is_initialized():      # world 1: init_from_env leaves the group to the caller; the shard's collectives need one
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
    kind, B = spec["kind"], 2
    R = 2 if kind == "rowhyb" else world            # ranks per row group
    n_groups, gi = world // R, rank // R
    groups = [dist.new_group(list(range(g * R, (g + 1) * R))) for g in range(n_groups)] if n_groups > 1 else [None]
    s0, s1 = gi * B // n_groups, (gi + 1) * B // n_groups      # the group's samples
    rows, peer = [], False
    for m in spec["models"]:
        m = dict(MODEL, **m)
        N, T, hid, L = m["N"], m["T"], m["hidden"], m["lstm_layers"]
        K = 4 if kind == "k" else 3
        torch.manual_seed(m["seed"])
        model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=L, gcn_hidden_dim=m["gcn_hidden"] or hid,
                           gcn_num_layers=3, num_nodes=N, user_bias=True, activation=nn.ReLU).to(dev)
        with torch.no_grad():      # keep both heads alive whatever the init draws (an all-zero prediction would make the comparison vacuous)
            for b in range(2):
                model.branch_models[b]['fc'][0].bias.add_(0.5)
        rng = np.random.default_rng(1)
        x = torch.from_numpy((rng.random((B, T, N, N, 1)) * 6).astype(np.float32))
        y = torch.from_numpy((rng.random((B, 1, N, N, 1)) * 2).astype(np.float32))

        def diffusion(n):
            flow = rng.random((n, N, N)).astype(np.float32)
            return torch.from_numpy(orc.adj_process(flow, "random_walk_diffusion", K - 1).astype(np.float32))

        G = diffusion(1)[0].to(dev)
        if m["dynamic"] == "dense":
            scale = 0.5 if kind == "k" else 1.0          # K = 4 dense stacks at full scale leave no margin under 1e-3 (measured 9.7e-4)
            go, gd = (torch.from_numpy((scale * rng.standard_normal((B, K, N, N)) / N ** 0.5).astype(np.float32)) for _ in range(2))
        else:
            go, gd = diffusion(B), diffusion(B)
        plan = shard.ShardPlan("row" if kind == "rowhyb" else kind, rank % R, R, N, K, group=groups[gi])
        peer = shard.enable_peer_exchange(plan, dev) if spec["peer"] else False
        xs, ys, gos, gds = (t.to(dev) for t in shard.shard_host_inputs(plan, x[s0:s1], y[s0:s1], go[s0:s1], gd[s0:s1]))
        for lstm_prec, layer_prec, tol_f, tol_g in m["cases"]:
            _set(model, *(("fp32", "fp32") if m["yardstick"] == "fp32" else (lstm_prec, layer_prec)))
            model.zero_grad(set_to_none=True)
            pred_w = model(x_seq=x.to(dev), G_list=[G, (go.to(dev), gd.to(dev))])
            assert float((pred_w > 0).float().mean()) > 0.5, "degenerate test case: the whole model's prediction is (almost) all zero"
            nn.functional.mse_loss(pred_w, y.to(dev)).backward()
            want = {k: p.grad.clone() for k, p in model.named_parameters()}
            _set(model, lstm_prec, layer_prec)
            model.zero_grad(set_to_none=True)
            pred = shard.sharded_forward(model, plan, xs, G, (gos, gds))
            shard.sharded_mse_loss(plan, pred, ys).backward()
            shard.allreduce_sum_gradients(list(model.parameters()), plan, model, over_world=n_groups > 1, scale=1.0 / n_groups)
            torch.cuda.synchronize()
            tag = f"nccl world-{world} {kind} shard hidden {hid} L={L}, lstm {lstm_prec}, layers {layer_prec}"
            ref_pred = pred_w[s0:s1, :, plan.row_lo:plan.row_hi] if kind != "k" else pred_w
            linf, l2 = orc.rel_errors(pred.detach().cpu().numpy(), ref_pred.detach().cpu().numpy())
            rows.append(dict(hid=hid, what=f"{tag}: y (rank {rank})", linf=linf, l2=l2, err=max(linf, l2), tol=tol_f))
            for k, p in model.named_parameters():
                linf, l2 = orc.rel_errors(p.grad.cpu().numpy(), want[k].cpu().numpy())
                rows.append(dict(hid=hid, what=f"{tag}: grad {k} (rank {rank})", linf=linf, l2=l2, err=l2, tol=tol_g))
    gathered = [None] * world
    dist.all_gather_object(gathered, rows)
    if rank == 0:
        json.dump({"rows": [r for part in gathered for r in part], "peer_exchange": bool(peer)}, open(out_path, "w"))
    dist.destroy_process_group()


if __name__ == "__main__":
    main(json.loads(sys.argv[1]), sys.argv[2])
