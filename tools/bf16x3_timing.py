"""Time the BDGCN layer in its three precisions -- fp16 (1), bf16x3 (2) and fp32 (0) -- alternated in one process, and the model
training step at hidden 128 in fp16 and bf16x3.  CUDA events, medians over --reps; the card's name and power limit are printed
beside every number.  Per-stage algorithmic TFLOP/s come from the engine's profile tags (a separate, profiled pass).

    python tools/bf16x3_timing.py [--reps 10] [--out timing.json]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from mpgcn_b200 import _lib, ops  # noqa: E402

PRECS = ("fp16", "bf16x3", "fp32")
LAYERS = [dict(N=1000, K=3, C=32, B=8), dict(N=500, K=3, C=32, B=32), dict(N=500, K=3, C=128, B=8)]


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return f"{name}, power limit {power}"


def layer_inputs(N, K, C, B, dev):
    g = torch.Generator(device=dev).manual_seed(N + K + C + B)
    X = torch.tanh(torch.randn(B, N, N, C, device=dev, generator=g)).requires_grad_(True)
    G = torch.randn(K, N, N, device=dev, generator=g) / N ** 0.5
    W = (torch.randn(K * K * C, C, device=dev, generator=g) * (2.0 / (K * K * C + C)) ** 0.5).requires_grad_(True)
    b = (torch.randn(C, device=dev, generator=g) * 0.1).requires_grad_(True)
    d_out = torch.randn(B, N, N, C, device=dev, generator=g) * 1e-5
    return X, G, W, b, d_out


def layer_step(inp, prec):
    X, G, W, b, d_out = inp
    X.grad = W.grad = b.grad = None
    out = ops.bdgcn(X, G, W, b, True, precision=prec)
    out.backward(d_out)


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(a.elapsed_time(e))
    return ts


def stage_rates(fn):
    lib = _lib.load()
    torch.cuda.synchronize()
    lib.mpgcn_profile_reset()
    lib.mpgcn_profile_enable(1)
    fn()
    torch.cuda.synchronize()
    lib.mpgcn_profile_enable(0)
    prof = _lib.profile_read()
    return {k: dict(ms=round(v["ms"], 3), tflops=round(v["flops"] / v["ms"] / 1e9, 1) if v["ms"] > 0 else None)
            for k, v in prof.items() if k in _lib.PROFILE_TAGS[:7] and v["launches"]}


def model_step_fn(prec, dev):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    import MPGCN as shim
    from torch import nn
    N, K, B, T, hid = 500, 3, 4, 7, 128
    torch.manual_seed(0)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3, num_nodes=N,
                       user_bias=True, activation=nn.ReLU).to(dev)
    model.lstm_precision = prec
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = prec
    x = torch.rand(B, T, N, N, 1, device=dev) * 8
    G = torch.rand(K, N, N, device=dev) / N
    dyn = (torch.rand(B, K, N, N, device=dev) / N, torch.rand(B, K, N, N, device=dev) / N)
    y_t = torch.rand(B, 1, N, N, 1, device=dev)

    def step():
        model.zero_grad(set_to_none=True)
        loss = torch.nn.functional.mse_loss(model(x_seq=x, G_list=[G, dyn]), y_t)
        loss.backward()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bf16x3_timing needs a CUDA device"
    dev = torch.device("cuda")
    where = card()
    results = {"card": where, "layers": [], "model": {}}
    for shape in LAYERS:
        inp = layer_inputs(**shape, dev=dev)
        precs = PRECS if shape["C"] == 32 or shape["N"] <= 500 else PRECS[:2]
        for p in precs:                                  # warm-up: modules, prepared supports, allocator
            layer_step(inp, p)
        times = {p: [] for p in precs}
        for _ in range(args.reps):                       # alternated
            for p in precs:
                times[p] += timed(lambda: layer_step(inp, p), 1)
        med = {p: float(np.median(v)) for p, v in times.items()}
        rates = {p: stage_rates(lambda: layer_step(inp, p)) for p in ("fp16", "bf16x3")}
        row = dict(shape=shape, median_ms=med, stages=rates)
        if "fp32" in med:
            row["bf16x3_speedup_over_fp32"] = med["fp32"] / med["bf16x3"]
        row["bf16x3_over_fp16"] = med["bf16x3"] / med["fp16"]
        results["layers"].append(row)
        print(f"[{where}] layer fwd+bwd {shape}: " + ", ".join(f"{p} {m:.2f} ms" for p, m in med.items()), flush=True)
        for p, st in rates.items():
            print(f"[{where}]   {p} stages (ms / algorithmic TFLOP/s): " + ", ".join(f"{k} {v['ms']}/{v['tflops']}" for k, v in st.items()),
                  flush=True)
        del inp
        torch.cuda.empty_cache()
    steps = {p: model_step_fn(p, dev) for p in ("fp16", "bf16x3")}
    for p, f in steps.items():
        f()
    times = {p: [] for p in steps}
    for _ in range(max(3, args.reps // 2)):
        for p, f in steps.items():
            times[p] += timed(f, 1)
    results["model"] = {p: float(np.median(v)) for p, v in times.items()}
    print(f"[{where}] model training step, hidden 128, N=500, B=4, T=7: " +
          ", ".join(f"{p} {m:.1f} ms" for p, m in results["model"].items()), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
