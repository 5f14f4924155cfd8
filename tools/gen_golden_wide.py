"""Generate the wide-channel fixtures `tests/golden/wide_*.npz` by running the UNMODIFIED reference.

TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py, whose helpers it reuses.  These are BDGCN layers and one whole model at
channel widths other than 32 (multiples of 32, C != H included: the first layer of a branch has C = lstm_hidden_dim).  Run
where a checkout of the reference is available (MPGCN_REFERENCE_DIR):

    python tools/gen_golden_wide.py

Seeds are their own (8000 + i, inputs 8100 + i, model 8500 + 100 j), so no other fixture changes.  Layer X and d_out are
regenerated from the seed by `oracle.gen_golden.layer_fixture`; W, the supports and the reference's outputs and gradients are
stored.  The model fixture keeps under 1 MB the way the at-size layer fixtures do: its parameters are drawn from the seed
(`wide_model_params`, loaded into the reference model; a checksum is stored) instead of stored, and of each BDGCN W gradient
(576 x 64 at hidden 64) only `W_ROWS` rows and the norm of the whole tensor are kept; every other gradient is stored in full.
The `wide_` prefix keeps them out of the tests that collect `bdgcn_*` / `mpgcn_*` fixtures.
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

WIDE_LAYER_CASES = [
    # name, dynamic, K, N, B, C, H, support kind (oracle.gen_golden.make_supports)
    ("wide_bdgcn_s_k3_n20_c64_h64", False, 3, 20, 2, 64, 64, "rw"),
    ("wide_bdgcn_d_k3_n12_c64_h96", True, 3, 12, 2, 64, 96, "rw"),
    ("wide_bdgcn_s_k2_n16_c32_h64", False, 2, 16, 2, 32, 64, "cheb"),
    ("wide_bdgcn_s_k1_n9_c128_h128", False, 1, 9, 2, 128, 128, "dense"),
]

WIDE_MODEL_CASES = [
    # name, N, K, support kind, T, B, hidden
    ("wide_mpgcn_n20_k3_h64", 20, 3, "rw", 5, 2, 64),
]


def gen_wide_layers(ref_mpgcn, ref_gcn):
    for idx, (name, dyn, K, N, B, C, H, gk) in enumerate(WIDE_LAYER_CASES):
        seed, in_seed = 8000 + idx, 8100 + idx
        rng = np.random.default_rng(seed)
        torch.manual_seed(seed)
        layer = ref_mpgcn.BDGCN(K=K, input_dim=C, hidden_dim=H, use_bias=True, activation=torch.nn.ReLU)
        with torch.no_grad():
            layer.b.copy_(torch.from_numpy(rng.standard_normal(H).astype(np.float32) * 0.1))
        X, d_out = layer_case_inputs(in_seed, B, N, C, H)
        Xt = torch.from_numpy(X).requires_grad_(True)
        if dyn:
            go, gd = make_supports(ref_gcn, gk, K, N, B, rng), make_supports(ref_gcn, gk, K, N, B, rng)
            G = (torch.from_numpy(go), torch.from_numpy(gd))
        else:
            g = make_supports(ref_gcn, gk, K, N, 0, rng)
            G = torch.from_numpy(g)
        out = layer(Xt, G)
        out.backward(torch.from_numpy(d_out))
        rec = dict(W=_np(layer.W), b=_np(layer.b), out=_np(out), dX=_np(Xt.grad), dW=_np(layer.W.grad), db=_np(layer.b.grad), K=K,
                   act="relu", dynamic=int(dyn), seed=in_seed, B=B, N=N, C=C, H=H, x_checksum=np.float64(X.astype(np.float64).sum()),
                   d_out_checksum=np.float64(d_out.astype(np.float64).sum()))
        rec.update(dict(G_o=go, G_d=gd) if dyn else dict(G=g))
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print("wrote", name, "out", tuple(out.shape))


W_ROWS = 48        # rows of each BDGCN W gradient kept in the model fixture


def wide_model_params(seed, shapes):
    """Parameters of the wide model fixture from its seed alone.  shapes: {state_dict key: shape} -> {key: float32 array}.
    BDGCN W [K*K*C, H]: Xavier normal; other matrices (LSTM, FC): U(+-1/sqrt(fan_in)); vectors (biases): U(+-0.1)."""
    rng = np.random.default_rng(seed)
    params = {}
    for k in sorted(shapes):
        shape = tuple(int(d) for d in shapes[k])
        if k.endswith(".W"):
            v = rng.standard_normal(shape) * np.sqrt(2.0 / (shape[0] + shape[1]))
        elif len(shape) == 2:
            a = 1.0 / np.sqrt(shape[1])
            v = rng.uniform(-a, a, shape)
        else:
            v = rng.uniform(-0.1, 0.1, shape)
        params[k] = v.astype(np.float32)
    return params


def params_checksum(params):
    return np.float64(sum(float(v.astype(np.float64).sum()) for v in params.values()))


def w_grad_rows(n, count=W_ROWS):
    """Rows of a W gradient kept in the fixture: evenly spread, first and last included."""
    return np.unique(np.linspace(0, n - 1, count).round().astype(np.int64))


def _gen_one_wide_model(ref_mpgcn, ref_gcn, seed, N, K, gk, T, B, hid):
    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    model = ref_mpgcn.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                            num_nodes=N, user_bias=True, activation=torch.nn.ReLU)
    params = wide_model_params(seed, {k: v.shape for k, v in model.state_dict().items()})
    model.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    x_seq = (rng.random((B, T, N, N, 1)) * 8).astype(np.float32)
    g_static = make_supports(ref_gcn, gk, K, N, 0, rng)
    g_o = make_supports(ref_gcn, gk, K, N, B, rng)
    g_d = make_supports(ref_gcn, gk, K, N, B, rng)
    d_y = rng.standard_normal((B, 1, N, N, 1)).astype(np.float32)
    y = model(x_seq=torch.from_numpy(x_seq), G_list=[torch.from_numpy(g_static), (torch.from_numpy(g_o), torch.from_numpy(g_d))])
    y.backward(torch.from_numpy(d_y))
    if not all(float(p.grad.abs().max()) > 0 for p in model.parameters()):
        return None
    rows = w_grad_rows(K * K * hid)
    rec = dict(x_seq=x_seq, G_static=g_static, G_o=g_o, G_d=g_d, d_y=d_y, y=_np(y), K=K, hidden=hid, seed=seed, W_rows=rows,
               params_checksum=params_checksum(params))
    for k, p in model.named_parameters():
        g = _np(p.grad)
        if k.endswith(".W"):
            rec["grad_rows:" + k] = g[rows]
            rec["grad_norm:" + k] = np.float64(np.linalg.norm(g.astype(np.float64)))
        else:
            rec["grad:" + k] = g
    return rec


def gen_wide_models(ref_mpgcn, ref_gcn):
    """As oracle.gen_golden.gen_model: the first seed whose run gives every parameter of both branches a gradient."""
    for idx, (name, N, K, gk, T, B, hid) in enumerate(WIDE_MODEL_CASES):
        for seed in range(8500 + idx, 12000, 100):
            rec = _gen_one_wide_model(ref_mpgcn, ref_gcn, seed, N, K, gk, T, B, hid)
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
    gen_wide_layers(ref_mpgcn, ref_gcn)
    gen_wide_models(ref_mpgcn, ref_gcn)


if __name__ == "__main__":
    main()
