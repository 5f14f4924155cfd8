#!/usr/bin/env python
"""Time the BDGCN layer on sparse static supports against the dense fp32 (precision 0) and fp16 tensor-core (precision 1) layers.

    python tools/sparse_timing.py [--reps 20] [--out results.json]

Workloads: N = 500 / 1000 / 2000 with the batch of bench.py's cfg3 / headline / cfg5 (BASELINE.json configs: 32, 8, 2), K = 3
random-walk diffusion supports (T_0 = I, T_1, T_2) of a symmetric 6-nearest-neighbour adjacency of random points in the plane,
C = H = 32, ReLU and bias.  Every shape is warmed up; forward and backward are timed separately with CUDA events, median of
`reps`.  Each sparse stage (the four gather launches of one forward + backward, in the order FWD_A, FWD_B, BWD_V, BWD_DX) is timed
with torch.profiler in a run of its own, and its achieved bytes/s is reported against the bytes it must move (its dense input read
once, its output written once).  The card's name and power limit are read in the same run.  One JSON line per workload goes to
stdout; `--out` also writes the whole run as one JSON file.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mpgcn_b200 import ops  # noqa: E402
from oracle import mpgcn_oracle as orc  # noqa: E402

WORKLOADS = [(500, 32), (1000, 8), (2000, 2)]
K, C, H = 3, 32, 32
HBM_PEAK = 3.35e12        # H100 SXM data sheet, bytes/s


def knn_supports(N, seed=0):
    rng = np.random.default_rng(seed)
    p = rng.random((N, 2))
    d = ((p[:, None] - p[None]) ** 2).sum(-1)
    A = np.zeros((N, N))
    nb = np.argsort(d, axis=1)[:, 1:7]
    A[np.repeat(np.arange(N), 6), nb.ravel()] = 1.0
    A = np.maximum(A, A.T)
    return orc.adj_process(A[None], "random_walk_diffusion", K - 1)[0].astype(np.float32)


def time_layer(X, G, W, b, d_out, precision, reps):
    def once():
        Xg = X.detach().requires_grad_(True)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        out = ops.bdgcn(Xg, G, W, b, True, precision=precision)
        e[1].record()
        out.backward(d_out)
        e[2].record()
        torch.cuda.synchronize()
        return e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])
    for _ in range(2):
        once()
    t = [once() for _ in range(reps)]
    return statistics.median(a for a, _ in t), statistics.median(b for _, b in t)


def sparse_stage_times(X, G, W, b, d_out):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):      # the last forward + backward is read: the profiler may miss the first launches of a session
            ops.bdgcn(X.detach().requires_grad_(True), G, W, b, True, precision="fp32").backward(d_out)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if "sparse_gather_kernel" in e.name and e.device_type.name == "CUDA"),
                key=lambda e: e.time_range.start)
    assert len(ev) >= 4, f"expected the four gather launches of a forward + backward, saw {len(ev)}"
    return [e.time_range.elapsed_us() / 1e3 for e in ev[-4:]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sparse_timing.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = {"torch_name": torch.cuda.get_device_name(dev), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}
    print("card:", card)
    rows = []
    for N, B in WORKLOADS:
        torch.manual_seed(0)
        Gd = torch.from_numpy(knn_supports(N)).to(dev)
        Gs = Gd.to_sparse()
        nnz = Gs._nnz()
        X = torch.randn(B, N, N, C, device=dev)
        W = torch.randn(K * K * C, H, device=dev) / (K * K * C) ** 0.5
        b = torch.randn(H, device=dev)
        d_out = torch.randn(B, N, N, H, device=dev)
        r = {"N": N, "B": B, "K": K, "C": C, "H": H, "nnz": nnz, "density": nnz / (K * N * N)}
        for name, G, prec in (("sparse", Gs, "fp32"), ("dense_fp32", Gd, "fp32"), ("dense_fp16", Gd, "fp16")):
            f, bw = time_layer(X, G, W, b, d_out, prec, a.reps)
            r[name] = {"fwd_ms": f, "bwd_ms": bw}
            torch.cuda.empty_cache()
        a4 = 4.0 * B * N * N
        need = {"FWD_A": a4 * C * (1 + K), "FWD_B": a4 * H * (K + 1), "BWD_V": a4 * H * (1 + K), "BWD_DX": a4 * C * (K + 1)}
        st = sparse_stage_times(X, Gs, W, b, d_out)
        r["stages"] = {k: {"ms": t, "bytes": need[k], "GB_per_s": need[k] / t / 1e6, "of_hbm_peak": need[k] * 1e3 / t / HBM_PEAK}
                       for k, t in zip(need, st)}
        r["speedup_vs_dense_fp32"] = (r["dense_fp32"]["fwd_ms"] + r["dense_fp32"]["bwd_ms"]) / (r["sparse"]["fwd_ms"] + r["sparse"]["bwd_ms"])
        r["speedup_vs_dense_fp16"] = (r["dense_fp16"]["fwd_ms"] + r["dense_fp16"]["bwd_ms"]) / (r["sparse"]["fwd_ms"] + r["sparse"]["bwd_ms"])
        print(json.dumps(r))
        rows.append(r)
        del X, d_out, Gd, Gs
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": card, "reps": a.reps, "rows": rows}, f, indent=1)
    print(f"{'N':>5} {'B':>3} {'sparse f/b ms':>16} {'dense fp32 f/b ms':>20} {'dense fp16 f/b ms':>20} {'x fp32':>7} {'x fp16':>7}")
    for r in rows:
        s, d, h = r["sparse"], r["dense_fp32"], r["dense_fp16"]
        print(f"{r['N']:>5} {r['B']:>3} {s['fwd_ms']:>7.2f}/{s['bwd_ms']:<8.2f} {d['fwd_ms']:>9.2f}/{d['bwd_ms']:<10.2f} "
              f"{h['fwd_ms']:>9.2f}/{h['bwd_ms']:<10.2f} {r['speedup_vs_dense_fp32']:>7.1f} {r['speedup_vs_dense_fp16']:>7.2f}")
        print("      stages: " + ", ".join(f"{k} {v['ms']:.3f} ms {v['GB_per_s']:.0f} GB/s" for k, v in r["stages"].items()))


if __name__ == "__main__":
    main()
