"""CUDA-event times of the stacked LSTM (lstm_num_layers = L) against nn.LSTM (cuDNN), and of a whole model step.

    python tools/lstm_stack_timing.py [--nodes 250] [--batch 4] [--steps 12] [--layers 2] [--hidden 32 96] [--reps 10]

Per hidden width: forward + backward of the LSTM alone (the engine's stack vs nn.LSTM on the [B N N, T, 1] sequences it would
otherwise get), and one training step of MPGCN(M=2, K=3, gcn 3 layers, fp16 engine) with the stacked LSTM on the engine.
LSTM TFLOP/s count the gate GEMMs as DESIGN.md section 7 does, times L, with an upper layer's gate GEMM 2H + 1 deep:
forward 8 H (KH + 1), backward 12 H (KH + 1) per cell and step, KH = H for the first layer and 2 H above it.
Prints the card's name and power limit; needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import MPGCN as shim  # noqa: E402
from mpgcn_b200 import ops  # noqa: E402


def _time(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def lstm_flops(cells, T, H, L):
    per = sum(20.0 * H * ((H if l == 0 else 2 * H) + 1) for l in range(L))      # 8 H (KH + 1) forward + 12 H (KH + 1) backward
    return per * cells * T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=250)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--hidden", type=int, nargs="+", default=[32, 96])
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    dev = torch.device("cuda")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    B, T, N, L = a.batch, a.steps, a.nodes, a.layers
    cells = B * N * N
    out = dict(card=card, nodes=N, batch=B, T=T, layers=L, widths={})
    for H in a.hidden:
        torch.manual_seed(0)
        lstm = nn.LSTM(1, H, L, batch_first=True).to(dev)
        x = torch.rand(B, T, N, N, 1, device=dev) * 8
        d_h = torch.randn(cells, H, device=dev)
        params = [getattr(lstm, f"{k}_l{l}") for l in range(L) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]

        def engine():
            ops.lstm_stack(x, params).backward(d_h)

        seq = x.permute(0, 2, 3, 1, 4).reshape(cells, T, 1).contiguous()

        def cudnn():
            lstm(seq)[0][:, -1, :].backward(d_h)

        r = dict(engine_ms=_time(engine, a.reps))
        try:
            r["cudnn_ms"] = _time(cudnn, a.reps)
        except torch.OutOfMemoryError:
            r["cudnn_ms"] = None
        torch.cuda.empty_cache()
        r["engine_tflops"] = lstm_flops(cells, T, H, L) / (r["engine_ms"] * 1e-3) / 1e12
        model = shim.MPGCN(M=2, K=3, input_dim=1, lstm_hidden_dim=H, lstm_num_layers=L, gcn_hidden_dim=H, gcn_num_layers=3, num_nodes=N,
                           user_bias=True, activation=nn.ReLU).to(dev)
        G = torch.rand(3, N, N, device=dev) / N
        dyn = (torch.rand(B, 3, N, N, device=dev) / N, torch.rand(B, 3, N, N, device=dev) / N)
        y = torch.rand(B, 1, N, N, 1, device=dev)

        def step():
            model.zero_grad(set_to_none=True)
            nn.functional.mse_loss(model(x_seq=x, G_list=[G, dyn]), y).backward()

        r["model_step_ms"] = _time(step, a.reps)
        out["widths"][H] = r
        del model, lstm
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
