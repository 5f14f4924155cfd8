"""Time the support-matrix builder's forward and backward: `Adj_Processor.process(flow)` and the gradient it sends to the flow.

    python tools/adj_grad_timing.py [--nodes 1000] [--order 3] [--batch 1 8] [--reps 20]

For each kernel type and batch size: the forward (`mpgcn_adj_process`) and the backward (`mpgcn_adj_process_backward`) called
through the C ABI on preallocated buffers, CUDA events around each call, medians over the repetitions.  The backward's N^3 work
is 2 (K - 1) SGEMMs per series per batch element (localpool has none); its algorithmic rate is reported against that count.
Prints the card's name and power limit; needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mpgcn_b200 import _lib  # noqa: E402

KINDS = ("localpool", "chebyshev", "random_walk_diffusion", "dual_random_walk_diffusion")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=1000)
    ap.add_argument("--order", type=int, default=3, help="K of Adj_Processor (chebyshev order / diffusion steps)")
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lib = _lib.load()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    N = a.nodes
    res = {"card": card, "N": N, "K": a.order, "ms": {}}
    med = lambda v: sorted(v)[len(v) // 2]
    for B in a.batch:
        for kt, kind in enumerate(KINDS):
            K = 1 if kind == "localpool" else a.order
            Ks = lib.mpgcn_adj_num_supports(kt, K)
            g = torch.Generator(device=dev).manual_seed(kt)
            flow = torch.rand(B, N, N, device=dev, generator=g) + 0.05
            sup = torch.empty(B, Ks, N, N, device=dev)
            d_sup = torch.randn(B, Ks, N, N, device=dev, generator=g)
            d_flow = torch.empty_like(flow)
            fws = torch.empty(lib.mpgcn_adj_workspace_bytes(B, N, kt, K), dtype=torch.uint8, device=dev)
            bws = torch.empty(lib.mpgcn_adj_backward_workspace_bytes(B, N, kt, K), dtype=torch.uint8, device=dev)

            def fwd():
                _lib.check(lib.mpgcn_adj_process(flow.data_ptr(), sup.data_ptr(), B, N, kt, K, fws.data_ptr(), fws.numel(), st), "adj_process")

            def bwd():
                _lib.check(lib.mpgcn_adj_process_backward(flow.data_ptr(), sup.data_ptr(), d_sup.data_ptr(), d_flow.data_ptr(), B, N, kt, K,
                                                          bws.data_ptr(), bws.numel(), st), "adj_process_backward")

            fwd()
            bwd()
            torch.cuda.synchronize()
            ms = {"forward": [], "backward": []}
            for _ in range(a.reps):
                for name, f in (("forward", fwd), ("backward", bwd)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    f()
                    e1.record()
                    torch.cuda.synchronize()
                    ms[name].append(e0.elapsed_time(e1))
            nser = 2 if kind == "dual_random_walk_diffusion" else 1
            gemm_flops = 0 if kind == "localpool" else 2.0 * (K - 1) * nser * B * 2.0 * N ** 3
            b_ms = med(ms["backward"])
            res["ms"][f"{kind} B={B}"] = {"forward_ms": med(ms["forward"]), "backward_ms": b_ms,
                                          "backward_gemm_tflops": gemm_flops / (b_ms * 1e-3) / 1e12 if gemm_flops else None}
            del flow, sup, d_sup, d_flow, fws, bws
            torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
