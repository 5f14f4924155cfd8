"""Generate the support-builder gradient fixtures `tests/golden/agrad_*.npz` by running the UNMODIFIED reference.

TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose loader it reuses.  The reference's `Adj_Processor.process` is plain
torch algebra, so a float64 flow that requires grad receives dL/dflow from autograd (its float32 `torch.eye` promotes).  Run where
a checkout of the reference is available (MPGCN_REFERENCE_DIR):

    python tools/gen_golden_adj_grad.py

Each fixture stores `flow` [B,N,N] (float32-representable values, in float64), the upstream `d_supports` [B,Ks,N,N], the
reference's `supports` and `d_flow`, plus `kernel_type` and `K`.  The `_zero` cases have an all-zero row (and, for the dual
kernel, an all-zero column) in the flow: the reference's `d_flow` holds NaN rows there.  Seeds are 9700 + i.  The `agrad_`
prefix keeps them out of the tests that collect `adj_*` fixtures.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.gen_golden import OUT, REF, _load_ref  # noqa: E402

SHORT = {"localpool": "lp", "chebyshev": "cheb", "random_walk_diffusion": "rw", "dual_random_walk_diffusion": "drw"}
CASES = []       # kernel type, K, B, N, zero rows [(b, i)], zero columns [(b, j)]
for _kt in SHORT:
    CASES += [(_kt, 1, 2, 1, [], []), (_kt, 2, 1, 5, [], []), (_kt, 3, 3, 12, [], []), (_kt, 3, 2, 33, [], [])]
CASES = [c for c in CASES if not (c[0] == "localpool" and c[1] != 1)] + [("localpool", 1, 3, 33, [], [])]
CASES += [("random_walk_diffusion", 2, 2, 12, [(0, 3)], []),
          ("dual_random_walk_diffusion", 2, 2, 12, [(1, 5)], [(0, 2)])]


def name_of(kt, K, B, N, zr, zc):
    return f"agrad_{SHORT[kt]}_k{K}_b{B}_n{N}" + ("_zero" if zr or zc else "")


def main():
    if not os.path.isdir(REF):
        sys.exit(f"reference not found at {REF}; set MPGCN_REFERENCE_DIR to a checkout of it")
    ref_gcn = _load_ref("GCN")
    for idx, (kt, K, B, N, zr, zc) in enumerate(CASES):
        rng = np.random.default_rng(9700 + idx)
        flow = (rng.random((B, N, N)) + 0.05).astype(np.float32).astype(np.float64)
        for b, i in zr:
            flow[b, i, :] = 0
        for b, j in zc:
            flow[b, :, j] = 0
        proc = ref_gcn.Adj_Processor(kt, K)
        f = torch.from_numpy(flow).requires_grad_(True)
        sup = proc.process(f)
        assert sup.dtype == torch.float64, sup.dtype
        d_sup = rng.standard_normal(tuple(sup.shape))
        sup.backward(torch.from_numpy(d_sup))
        rec = dict(flow=flow, d_supports=d_sup, supports=sup.detach().numpy(), d_flow=f.grad.numpy(), kernel_type=kt, K=proc.K)
        name = name_of(kt, K, B, N, zr, zc)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print("wrote", name, "supports", tuple(sup.shape), "NaN rows in d_flow:", int(np.isnan(rec["d_flow"]).any(axis=2).sum()))


if __name__ == "__main__":
    main()
