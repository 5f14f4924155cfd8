"""Generate the support-gradient fixtures `tests/golden/sgrad_*.npz` by running the UNMODIFIED reference.

TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose helpers it reuses.  The reference computes BDGCN with einsums, so a
support stack that requires grad receives dL/dG from autograd; these fixtures record it.  Run where a checkout of the reference
is available (MPGCN_REFERENCE_DIR):

    python tools/gen_golden_support_grad.py

Seeds are their own (9000 + i, inputs 9100 + i, model 9500 + 100 j), so no other fixture changes.  Layer X and d_out are
regenerated from the seed by `oracle.gen_golden.layer_fixture`; W, b, the supports, the output and the support gradients are
stored (static: `dG` [K,N,N]; dynamic: `dG_o`, `dG_d` [B,K,N,N]).  The model fixture is the whole model with a learnable static
support in G_list[0]: the three layers of that branch add into one `dG_static`.  The `sgrad_` prefix keeps them out of the tests
that collect `bdgcn_*` / `mpgcn_*` / `wide_*` / `many_*` / `big_*` fixtures.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.gen_golden import OUT, REF, _load_ref, _np, layer_case_inputs, make_supports  # noqa: E402

SGRAD_LAYER_CASES = [
    # name, dynamic, K, N, B, C, H, support kind (oracle.gen_golden.make_supports)
    ("sgrad_bdgcn_s_k1_n7_c32_h32", False, 1, 7, 2, 32, 32, "dense"),
    ("sgrad_bdgcn_s_k3_n47_c32_h32", False, 3, 47, 1, 32, 32, "rw"),
    ("sgrad_bdgcn_s_k9_n20_c32_h32", False, 9, 20, 2, 32, 32, "dense"),
    ("sgrad_bdgcn_s_k3_n20_c64_h96", False, 3, 20, 2, 64, 96, "rw"),
    ("sgrad_bdgcn_d_k3_n20_c96_h32", True, 3, 20, 2, 96, 32, "dense"),
    ("sgrad_bdgcn_d_k9_n7_c32_h32", True, 9, 7, 2, 32, 32, "dense"),
    ("sgrad_bdgcn_d_k1_n47_c64_h96", True, 1, 47, 1, 64, 96, "dense"),
]

SGRAD_MODEL_CASES = [
    # name, N, K, support kind, T, B, hidden
    ("sgrad_mpgcn_n9_k3_h32", 9, 3, "rw", 4, 2, 32),
]


def gen_layers(ref_mpgcn, ref_gcn):
    for idx, (name, dyn, K, N, B, C, H, gk) in enumerate(SGRAD_LAYER_CASES):
        seed, in_seed = 9000 + idx, 9100 + idx
        rng = np.random.default_rng(seed)
        torch.manual_seed(seed)
        layer = ref_mpgcn.BDGCN(K=K, input_dim=C, hidden_dim=H, use_bias=True, activation=torch.nn.ReLU)
        with torch.no_grad():
            layer.b.copy_(torch.from_numpy(rng.standard_normal(H).astype(np.float32) * 0.1))
        X, d_out = layer_case_inputs(in_seed, B, N, C, H)
        Xt = torch.from_numpy(X).requires_grad_(True)
        if dyn:
            go, gd = make_supports(ref_gcn, gk, K, N, B, rng), make_supports(ref_gcn, gk, K, N, B, rng)
            G = (torch.from_numpy(go).requires_grad_(True), torch.from_numpy(gd).requires_grad_(True))
        else:
            g = make_supports(ref_gcn, gk, K, N, 0, rng)
            G = torch.from_numpy(g).requires_grad_(True)
        out = layer(Xt, G)
        out.backward(torch.from_numpy(d_out))
        rec = dict(W=_np(layer.W), b=_np(layer.b), out=_np(out), K=K, act="relu", dynamic=int(dyn), seed=in_seed, B=B, N=N, C=C, H=H,
                   x_checksum=np.float64(X.astype(np.float64).sum()), d_out_checksum=np.float64(d_out.astype(np.float64).sum()))
        if dyn:
            rec.update(G_o=go, G_d=gd, dG_o=_np(G[0].grad), dG_d=_np(G[1].grad))
        else:
            rec.update(G=g, dG=_np(G.grad))
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print("wrote", name, "out", tuple(out.shape))


def _one_model(ref_mpgcn, ref_gcn, seed, N, K, gk, T, B, hid):
    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    model = ref_mpgcn.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                            num_nodes=N, user_bias=True, activation=torch.nn.ReLU)
    x_seq = (rng.random((B, T, N, N, 1)) * 8).astype(np.float32)
    g_static = make_supports(ref_gcn, gk, K, N, 0, rng)
    g_o = make_supports(ref_gcn, gk, K, N, B, rng)
    g_d = make_supports(ref_gcn, gk, K, N, B, rng)
    d_y = rng.standard_normal((B, 1, N, N, 1)).astype(np.float32)
    gs = torch.from_numpy(g_static).requires_grad_(True)
    y = model(x_seq=torch.from_numpy(x_seq), G_list=[gs, (torch.from_numpy(g_o), torch.from_numpy(g_d))])
    y.backward(torch.from_numpy(d_y))
    if not all(float(p.grad.abs().max()) > 0 for p in model.parameters()) or float(gs.grad.abs().max()) == 0:
        return None
    rec = dict(x_seq=x_seq, G_static=g_static, G_o=g_o, G_d=g_d, d_y=d_y, y=_np(y), dG_static=_np(gs.grad), K=K, hidden=hid, seed=seed)
    for k, v in model.state_dict().items():
        rec["param:" + k] = _np(v)
    for k, p in model.named_parameters():
        rec["grad:" + k] = _np(p.grad)
    return rec


def gen_models(ref_mpgcn, ref_gcn):
    for idx, (name, N, K, gk, T, B, hid) in enumerate(SGRAD_MODEL_CASES):
        for seed in range(9500 + idx, 12000, 100):     # the first seed whose two branches both receive gradients
            rec = _one_model(ref_mpgcn, ref_gcn, seed, N, K, gk, T, B, hid)
            if rec is not None:
                break
        else:
            raise RuntimeError(f"{name}: no seed with two live branches")
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print("wrote", name, "y", rec["y"].shape, "seed", seed)


def main():
    if not os.path.isdir(REF):
        sys.exit(f"reference not found at {REF}; set MPGCN_REFERENCE_DIR to a checkout of it")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    ref_mpgcn, ref_gcn = _load_ref("MPGCN"), _load_ref("GCN")
    gen_layers(ref_mpgcn, ref_gcn)
    gen_models(ref_mpgcn, ref_gcn)


if __name__ == "__main__":
    main()
