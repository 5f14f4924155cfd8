"""Generate the many-support layer fixtures `tests/golden/many_bdgcn_*.npz` by running the UNMODIFIED reference.

TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose helpers it reuses.  These are BDGCN layers at C = H = 32 with more
than 8 supports, built the way the trainer builds them: `Adj_Processor('dual_random_walk_diffusion', k)` gives 2k + 1
supports (Model_Trainer.py:32).  Run where a checkout of the reference is available (MPGCN_REFERENCE_DIR):

    python tools/gen_golden_many.py

Seeds are their own (7000 + i, inputs 7100 + i), so no other fixture changes.  X and d_out are regenerated from the seed by
`oracle.gen_golden.layer_fixture`; W, the supports and the reference's outputs and gradients are stored.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.gen_golden import OUT, REF, _load_ref, _np, layer_case_inputs  # noqa: E402

MANY_CASES = [
    # name, dynamic, diffusion order k (K = 2k + 1 supports), N, B
    ("many_bdgcn_s_k9_n20_dual", False, 4, 20, 2),
    ("many_bdgcn_d_k9_n12_dual", True, 4, 12, 2),
    ("many_bdgcn_s_k11_n14_dual", False, 5, 14, 1),
]


def dual_supports(ref_gcn, order, N, batch, rng):
    """reference Adj_Processor('dual_random_walk_diffusion', order) on a U[0,1) flow -> [2*order+1, N, N] (batch 0) or
    [batch, 2*order+1, N, N] (GCN.py:84-92)."""
    flow = torch.from_numpy(rng.random((max(batch, 1), N, N)).astype(np.float32))
    g = _np(ref_gcn.Adj_Processor("dual_random_walk_diffusion", order).process(flow))
    assert g.shape[1] == 2 * order + 1, g.shape
    return g if batch else g[0]


def gen_many(ref_mpgcn, ref_gcn):
    for idx, (name, dyn, order, N, B) in enumerate(MANY_CASES):
        K, C = 2 * order + 1, 32
        seed, in_seed = 7000 + idx, 7100 + idx
        rng = np.random.default_rng(seed)
        torch.manual_seed(seed)
        layer = ref_mpgcn.BDGCN(K=K, input_dim=C, hidden_dim=C, use_bias=True, activation=torch.nn.ReLU)
        with torch.no_grad():
            layer.b.copy_(torch.from_numpy(rng.standard_normal(C).astype(np.float32) * 0.1))
        X, d_out = layer_case_inputs(in_seed, B, N, C, C)
        Xt = torch.from_numpy(X).requires_grad_(True)
        if dyn:
            go, gd = dual_supports(ref_gcn, order, N, B, rng), dual_supports(ref_gcn, order, N, B, rng)
            G = (torch.from_numpy(go), torch.from_numpy(gd))
        else:
            g = dual_supports(ref_gcn, order, N, 0, rng)
            G = torch.from_numpy(g)
        out = layer(Xt, G)
        out.backward(torch.from_numpy(d_out))
        rec = dict(W=_np(layer.W), b=_np(layer.b), out=_np(out), dX=_np(Xt.grad), dW=_np(layer.W.grad), db=_np(layer.b.grad), K=K,
                   act="relu", dynamic=int(dyn), seed=in_seed, B=B, N=N, C=C, H=C, x_checksum=np.float64(X.astype(np.float64).sum()),
                   d_out_checksum=np.float64(d_out.astype(np.float64).sum()))
        rec.update(dict(G_o=go, G_d=gd) if dyn else dict(G=g))
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print("wrote", name, "K", K, "out", tuple(out.shape))


def main():
    if not os.path.isdir(REF):
        sys.exit(f"reference not found at {REF}; set MPGCN_REFERENCE_DIR to a checkout of it")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    gen_many(_load_ref("MPGCN"), _load_ref("GCN"))


if __name__ == "__main__":
    main()
