#!/usr/bin/env python
"""Peak memory and step time of a training step with the recomputing LSTM backward (MPGCN.lstm_recompute = True) against
the stored-state LSTM (off).

    python tools/lstm_recompute_timing.py [--reps 5]

Workloads (M = 2, K = 3, T = 12, three BDGCN layers, tensor cores): the headline (N = 1000, B = 8, hidden 32); N = 500, B = 4 at
hidden 96 and 128, where both modes fit; N = 1000, B = 4 at hidden 96 and 128, where the stored-state mode is reported as out of
memory if it is.  One training step is forward, MSE loss and backward.  Peak memory is torch.cuda.max_memory_allocated after a
reset, around one warmed step; step time is the median over `reps` steps timed with CUDA events, the two modes alternated step by
step.  The card's name and power limit are read in the same run.  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import MPGCN as shim  # noqa: E402

WORKLOADS = [(1000, 8, 32), (500, 4, 96), (500, 4, 128), (1000, 4, 96), (1000, 4, 128)]
T, K = 12, 3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or [","])[0].split(",")[:2]
    return name.strip(), power.strip()


def workload(N, B, hid, reps, dev):
    torch.manual_seed(0)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3, num_nodes=N,
                       user_bias=True, activation=nn.ReLU).to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.rand(B, T, N, N, 1, device=dev, generator=g) * 6
    y = torch.rand(B, 1, N, N, 1, device=dev, generator=g) * 2
    G = torch.rand(K, N, N, device=dev, generator=g) / N
    go, gd = (torch.rand(B, K, N, N, device=dev, generator=g) / N for _ in range(2))

    def step():
        model.zero_grad(set_to_none=True)
        loss = nn.functional.mse_loss(model(x_seq=x, G_list=[G, (go, gd)]), y)
        loss.backward()
        return loss

    res = {}
    modes = {"stored": None, "recompute": True}
    for name, rc in modes.items():          # warm-up and peak memory
        model.lstm_recompute = rc
        try:
            step()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            loss = float(step().detach())
            torch.cuda.synchronize()
            res[name] = dict(peak_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), model_gib=round(base / 2 ** 30, 2),
                             loss=loss, ms=[])
        except torch.OutOfMemoryError as e:
            res[name] = dict(oom=str(e).split(".")[0])
        model.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()
    live = [n for n in modes if "oom" not in res[n]]
    for _ in range(reps):                   # alternated
        for name in live:
            model.lstm_recompute = modes[name]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            torch.cuda.synchronize()
            res[name]["ms"].append(e0.elapsed_time(e1))
    for name in live:
        res[name]["step_ms"] = round(statistics.median(res[name].pop("ms")), 2)
    del model
    torch.cuda.empty_cache()
    return dict(N=N, B=B, hidden=hid, T=T, **res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lstm_recompute_timing: needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    rows = [workload(N, B, hid, a.reps, dev) for N, B, hid in WORKLOADS]
    print(json.dumps(dict(gpu=name, power_limit=power, workloads=rows)))


if __name__ == "__main__":
    main()
