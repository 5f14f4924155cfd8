"""Time one BDGCN layer's backward with and without the support gradient (dL/dG), and the dG stages on their own.

    python tools/support_grad_timing.py [--nodes 1000] [--supports 3] [--hidden 32] [--batch 8] [--reps 20]

For static and dynamic supports, at precision 1 (tensor cores): the backward call alone (mpgcn_bdgcn_backward_x vs
mpgcn_bdgcn_backward_supports, same inputs, CUDA events around each call, alternated), and the per-tag kernel time of the
BWD_DG launches (U16 recompute, BWD_DGO / BWD_DGD, their reductions) from the library's event profiler in a separate pass.
The dG stages' algorithmic rate is 2 K B N^3 (C + H) over the BWD_DG kernel time.  Prints the card's name and power limit;
needs a GPU.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mpgcn_b200 import _lib  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1000)
    ap.add_argument("--supports", type=int, default=3)
    ap.add_argument("--hidden", type=int, default=32)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lib = _lib.load()
    dev = torch.device("cuda:0")
    B, N, K, C, H, prec = a.batch, a.nodes, a.supports, a.hidden, a.hidden, _lib.PREC_FP16_TC
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: None if t is None else t.data_ptr()
    res = {"card": card, "B": B, "N": N, "K": K, "C": C, "H": H}
    for dyn in (0, 1):
        g = torch.Generator(device=dev).manual_seed(dyn)
        X = torch.tanh(torch.randn(B, N, N, C, device=dev, generator=g))
        shape = (B, K, N, N) if dyn else (K, N, N)
        Go = torch.randn(shape, device=dev, generator=g) / N ** 0.5
        Gd = torch.randn(shape, device=dev, generator=g) / N ** 0.5 if dyn else Go
        W = torch.randn(K * K * C, H, device=dev, generator=g) * (2.0 / (K * K * C + H)) ** 0.5
        bias = torch.zeros(H, device=dev)
        out = torch.empty(B, N, N, H, device=dev)
        saved = torch.empty(lib.mpgcn_bdgcn_saved_bytes(B, N, K, C, H, prec), dtype=torch.uint8, device=dev)
        fws = torch.empty(lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, C, H, dyn, prec), dtype=torch.uint8, device=dev)
        _lib.check(lib.mpgcn_bdgcn_forward(p(X), p(Go), p(Gd), dyn, p(W), p(bias), 1, p(out), p(saved), p(fws), fws.numel(), B, N, K, C, H,
                                           prec, st), "forward")
        d_out = torch.randn(B, N, N, H, device=dev, generator=g) * 1e-3
        dX, dW, db = torch.empty_like(X), torch.empty_like(W), torch.empty_like(bias)
        dGo = torch.empty(shape, device=dev)
        dGd = torch.empty(shape, device=dev) if dyn else None
        ws = torch.empty(lib.mpgcn_bdgcn_support_grad_workspace_bytes(B, N, K, C, H, dyn, prec), dtype=torch.uint8, device=dev)

        def plain():
            _lib.check(lib.mpgcn_bdgcn_backward_x(p(d_out), p(out), p(Go), p(Gd), dyn, p(W), 1, p(saved), p(dX), p(dW), p(db), p(ws), ws.numel(),
                                                  B, N, K, C, H, prec, None, st), "backward_x")

        def with_dg():
            _lib.check(lib.mpgcn_bdgcn_backward_supports(p(d_out), p(out), p(Go), p(Gd), dyn, p(W), 1, p(saved), p(dX), p(dW), p(db), p(ws),
                                                         ws.numel(), B, N, K, C, H, prec, None, p(X), p(dGo), p(dGd), st), "backward_supports")

        for f in (plain, with_dg):          # warm-up: module load, tensor-map encoder, smem opt-in
            f()
        torch.cuda.synchronize()
        ms = {"plain": [], "with_dg": []}
        for _ in range(a.reps):
            for name, f in (("plain", plain), ("with_dg", with_dg)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                f()
                e1.record()
                torch.cuda.synchronize()
                ms[name].append(e0.elapsed_time(e1))
        lib.mpgcn_profile_reset()
        lib.mpgcn_profile_enable(1)
        for _ in range(a.reps):
            with_dg()
        torch.cuda.synchronize()
        prof = _lib.profile_read()
        lib.mpgcn_profile_enable(0)
        lib.mpgcn_profile_reset()
        med = lambda v: sorted(v)[len(v) // 2]
        n3 = {t: prof[t]["ms"] / a.reps for t in ("BWD_V", "BWD_DX")}
        dg_ms = prof["BWD_DG"]["ms"] / a.reps
        dg_flops = 2.0 * K * B * N ** 3 * (C + H)
        res["dynamic" if dyn else "static"] = {
            "backward_ms": med(ms["plain"]), "backward_with_dG_ms": med(ms["with_dg"]), "ratio": med(ms["with_dg"]) / med(ms["plain"]),
            "n3_kernels_ms": n3, "dG_kernels_ms": dg_ms, "dG_launches_per_call": prof["BWD_DG"]["launches"] / a.reps,
            "dG_algorithmic_tflops": dg_flops / (dg_ms * 1e-3) / 1e12 if dg_ms > 0 else None}
        del saved, fws, ws
        torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
