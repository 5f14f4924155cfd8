"""Per-launch timing of the four N^3 tensor-core contractions (FWD_A, FWD_B, BWD_V, BWD_DX) of one BDGCN layer.

    python tools/contract_timing.py [--reps 20] [--warmup 3] [--json out.json]

One fp16 layer forward + backward runs through the C ABI, and the library's profile tags time every contraction launch with
its own pair of CUDA events (DESIGN.md section 7).  Printed per kind, after warm-up:

* algorithmic TFLOP/s (2 B K R N^2 32 per launch over the summed event time) and k-blocks per tile, at the headline layer
  (N = 1000, K = 3, batch 8) and at N = 500 and 2000;
* a fit of  t_launch / waves = kb * t + E  over runs that change the k-blocks per tile (kb) at a fixed tile count: FWD_B and
  BWD_DX take K * N / 64 resp. K * ceil(N / 64) k-blocks per tile over ceil(N / 128) * ceil(N / 8) * B tiles, so K = 1 .. 8 at
  N = 1000 moves kb alone.  t is the time of one k-block of MMAs, E the fixed cost of a tile (epilogue, pipeline drain and
  refill), both in microseconds; waves = ceil(tiles / SMs) (one persistent CTA per SM).

The card's name, power limit and SM clocks are read in the same run, since every number here depends on them.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KINDS = ("FWD_A", "FWD_B", "BWD_V", "BWD_DX")


def cdiv(a, b):
    return -(-a // b)


def kb_per_tile(kind, N, K):
    return {"FWD_A": cdiv(N, 64), "BWD_V": cdiv(N, 64), "FWD_B": cdiv(K * N, 64), "BWD_DX": K * cdiv(N, 64)}[kind]


def tiles(kind, N, K, B):
    per = cdiv(N, 128) * cdiv(N, 8)
    return per * B * (K if kind in ("FWD_A", "BWD_V") else 1)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def time_layer(N, K, B, reps, warmup):
    """-> {kind: {launches, ms, tflops}} summed over `reps` forward + backward calls after `warmup` untimed ones."""
    import torch
    from mpgcn_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    C = H = 32
    X = torch.rand((B, N, N, C), device=dev, generator=g)
    Go = torch.rand((K, N, N), device=dev, generator=g) / N
    Gd = torch.rand((K, N, N), device=dev, generator=g) / N
    W = torch.randn((K * K * C, H), device=dev, generator=g) * 0.05
    bias = torch.zeros(H, device=dev)
    d_out = torch.randn((B, N, N, H), device=dev, generator=g)
    out = torch.empty((B, N, N, H), device=dev)
    saved = torch.empty(lib.mpgcn_bdgcn_saved_bytes(B, N, K, C, H, 1), dtype=torch.uint8, device=dev)
    ws = torch.empty(lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, C, H, 0, 1), dtype=torch.uint8, device=dev)
    wsb = torch.empty(lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, 0, 1), dtype=torch.uint8, device=dev)
    dX, dW, db = torch.empty_like(X), torch.empty_like(W), torch.empty_like(bias)
    st = torch.cuda.current_stream().cuda_stream

    def step():
        _lib.check(lib.mpgcn_bdgcn_forward(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), 0, W.data_ptr(), bias.data_ptr(), 1, out.data_ptr(),
                                           saved.data_ptr(), ws.data_ptr(), ws.numel(), B, N, K, C, H, 1, st), "forward")
        _lib.check(lib.mpgcn_bdgcn_backward(d_out.data_ptr(), out.data_ptr(), Go.data_ptr(), Gd.data_ptr(), 0, W.data_ptr(), 1,
                                            saved.data_ptr(), dX.data_ptr(), dW.data_ptr(), db.data_ptr(), wsb.data_ptr(), wsb.numel(),
                                            B, N, K, C, H, 1, st), "backward")

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    lib.mpgcn_profile_reset()
    lib.mpgcn_profile_enable(1)
    for _ in range(reps):
        step()
    torch.cuda.synchronize()
    lib.mpgcn_profile_enable(0)
    prof = _lib.profile_read()
    res = {}
    for k in KINDS:
        v = prof[k]
        res[k] = dict(launches=v["launches"], ms=v["ms"], tflops=v["flops"] / (v["ms"] * 1e-3) / 1e12 if v["ms"] > 0 else None)
    del X, Go, Gd, W, d_out, out, saved, ws, wsb, dX
    torch.cuda.empty_cache()
    return res


def fit(points):
    """least squares y = t * x + E over [(x, y)] -> (t, E)"""
    n = len(points)
    sx = sum(x for x, _ in points); sy = sum(y for _, y in points)
    sxx = sum(x * x for x, _ in points); sxy = sum(x * y for x, y in points)
    t = (n * sxy - sx * sy) / (n * sxx - sx * sx)
    return t, (sy - t * sx) / n


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--fit-ks", default="1,2,3,4,6,8", help="supports K of the (t, E) fit at N = 1000, batch 8")
    ap.add_argument("--json", default=None, help="also write every number to this file")
    a = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "contract_timing needs a CUDA device"
    info = card()
    sms = info["sms"]
    print(f"card: {info['name']}, {sms} SMs; power.limit, clocks.sm, clocks.max.sm, throttle: {info['nvidia_smi']}")
    report = {"card": info, "shapes": [], "fit": {}}

    print(f"{'N':>5} {'K':>2} {'B':>2} {'kind':>7} {'kb/tile':>7} {'tiles':>7} {'launches':>8} {'ms/launch':>9} {'TFLOP/s':>8}")
    for N, K, B in ((1000, 3, 8), (500, 3, 8), (2000, 3, 2)):
        r = time_layer(N, K, B, a.reps, a.warmup)
        for k in KINDS:
            v = r[k]
            row = dict(N=N, K=K, B=B, kind=k, kb=kb_per_tile(k, N, K), tiles=tiles(k, N, K, B), launches=v["launches"],
                       ms_per_launch=v["ms"] / max(1, v["launches"]), tflops=v["tflops"])
            report["shapes"].append(row)
            print(f"{N:>5} {K:>2} {B:>2} {k:>7} {row['kb']:>7} {row['tiles']:>7} {row['launches']:>8} {row['ms_per_launch']:>9.3f} "
                  f"{row['tflops']:>8.1f}")

    N, B = 1000, 8
    pts = {"FWD_B": [], "BWD_DX": []}
    for K in (int(s) for s in a.fit_ks.split(",")):
        r = time_layer(N, K, B, a.reps, a.warmup)
        for k in pts:
            waves = math.ceil(tiles(k, N, K, B) / sms)
            us = r[k]["ms"] / max(1, r[k]["launches"]) * 1e3
            pts[k].append((kb_per_tile(k, N, K), us / waves))
    for k, p in pts.items():
        t, E = fit(p)
        report["fit"][k] = dict(points=p, t_us=t, E_us=E, E_kblocks=E / t, main_loop_tflops=2 * 128 * 256 * 64 * sms / (t * 1e-6) / 1e12)
        print(f"fit {k:>6} (N = {N}, B = {B}, kb = {[x for x, _ in p]}): t = {t:.3f} us per k-block, E = {E:.3f} us per tile "
              f"= {E / t:.2f} k-blocks; main loop alone {report['fit'][k]['main_loop_tflops']:.0f} TFLOP/s")
    print(f"card after: {card()['nvidia_smi']}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
