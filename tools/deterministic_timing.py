"""Cost of torch.use_deterministic_algorithms(True) on a training step: flag off and on, alternated, same model and inputs.

    python tools/deterministic_timing.py [--steps 10] [--rounds 3] [--dump-outputs DIR]

Two workloads, each the bench.py step (MPGCN M=2, K=3, 3 GCN layers, fp16 engine, MSE, backward):
  headline   N = 1000, T = 12, batch 8, hidden 32;
  hidden96   N = 250,  T = 12, batch 4, hidden 96 (the DESIGN.md section 7 setting: N = 1000 does not fit at hidden 96).
Per workload and flag: step ms (CUDA events around `steps` steps after a warm-up, best and all rounds) and gpu_launches of one
step.  Prints the card's name and power limit, read in the same run, as one JSON line per workload.  --dump-outputs DIR writes
prediction, loss and every parameter gradient of one step under the flag (DIR/<workload>.npz), so that two builds can be
compared bit for bit.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import MPGCN as shim  # noqa: E402
from mpgcn_b200 import _lib  # noqa: E402

WORKLOADS = {"headline": (1000, 3, 12, 8, 32), "hidden96": (250, 3, 12, 4, 96)}      # N, K, T, B, hidden


def build(N, K, T, B, hid, dev):
    torch.manual_seed(1234)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU).to(dev)
    model.lstm_precision = "fp16"
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = "fp16"
    g = torch.Generator().manual_seed(4321)
    x = (torch.rand(B, T, N, N, 1, generator=g) * 8).to(dev)
    y = (torch.rand(B, 1, N, N, 1, generator=g) * 8).to(dev)
    G = (torch.randn(K, N, N, generator=torch.Generator().manual_seed(7)) / N ** 0.5).to(dev)
    go = (torch.randn(B, K, N, N, generator=g) / N ** 0.5).to(dev)
    gd = (torch.randn(B, K, N, N, generator=g) / N ** 0.5).to(dev)
    crit = nn.MSELoss()
    params = list(model.parameters())

    def step():
        for p in params:
            p.grad = None
        out = model(x_seq=x, G_list=[G, (go, gd)])
        loss = crit(out, y)
        loss.backward()
        return out, loss

    return step, model


def time_steps(step, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def launches(step):
    lib = _lib.load()
    torch.cuda.synchronize()
    lib.mpgcn_profile_reset()
    lib.mpgcn_profile_enable(1)
    step()
    torch.cuda.synchronize()
    lib.mpgcn_profile_enable(0)
    prof = _lib.profile_read()
    return sum(v["launches"] for t, v in prof.items() if t not in _lib.REGION_TAGS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    dev = torch.device("cuda")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    for name in a.workloads:
        step, model = build(*WORKLOADS[name], dev)
        ms = {False: [], True: []}
        n_launch = {}
        for flag in (False, True):           # warm-up of both modes (module loads, allocator, slot buffers)
            torch.use_deterministic_algorithms(flag)
            for _ in range(2):
                step()
            torch.cuda.synchronize()
            n_launch[flag] = launches(step)
        for _ in range(a.rounds):            # alternated
            for flag in (False, True):
                torch.use_deterministic_algorithms(flag)
                ms[flag].append(time_steps(step, a.steps))
        torch.use_deterministic_algorithms(False)
        off, on = min(ms[False]), min(ms[True])
        print(json.dumps({"workload": name, "shape": dict(zip("NKTBH", WORKLOADS[name])), "card": card,
                          "step_ms_off": round(off, 3), "step_ms_on": round(on, 3), "cost_pct": round(100 * (on - off) / off, 2),
                          "rounds_ms_off": [round(v, 3) for v in ms[False]], "rounds_ms_on": [round(v, 3) for v in ms[True]],
                          "gpu_launches_off": n_launch[False], "gpu_launches_on": n_launch[True]}), flush=True)
        if a.dump_outputs:
            os.makedirs(a.dump_outputs, exist_ok=True)
            torch.use_deterministic_algorithms(True)
            out, loss = step()
            torch.cuda.synchronize()
            torch.use_deterministic_algorithms(False)
            arrays = {"prediction": out.detach().cpu().numpy(), "loss": loss.detach().cpu().numpy()}
            for pname, p in model.named_parameters():
                if p.grad is not None:
                    arrays["grad." + pname] = p.grad.detach().cpu().numpy()
            np.savez(os.path.join(a.dump_outputs, name + ".npz"), **arrays)
        del step, model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
