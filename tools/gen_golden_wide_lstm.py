"""Generate the wide-LSTM fixtures `tests/golden/lstmw_*.npz` and `tests/golden/mpgcnw_*.npz` by running the UNMODIFIED reference.

TEST INFRASTRUCTURE ONLY, like oracle/gen_golden.py and tools/gen_golden_wide.py, whose helpers it reuses.  These pin the
per-cell LSTM (the reference's nn.LSTM) and one whole model at hidden sizes 96 and 128.  Run where a checkout of the reference
is available (MPGCN_REFERENCE_DIR):

    python tools/gen_golden_wide_lstm.py

Seeds are their own (LSTM 9000 + i, model 9500 + 100 j), so no other fixture changes.  To keep the files small, parameters are
drawn from the seed (`lstm_params`, `wide_model_params`) and only their checksum is stored; of each gradient with more than
`W_ROWS` rows of width >= 96 (BDGCN W, LSTM weight_hh) only `W_ROWS` rows and the norm of the whole tensor are kept, in the
LSTM fixtures (`dw_hh_rows`, `dw_hh_row_ids`, `dw_hh_norm`) as in the model fixture.  The prefixes `lstmw_` / `mpgcnw_` keep them out of the tests that collect `lstm_*` / `mpgcn_*` fixtures (those run
the fp32 LSTM kernels, which stop at hidden 64).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.gen_golden import OUT, REF, _load_ref, _np, make_supports  # noqa: E402
from tools.gen_golden_wide import W_ROWS, params_checksum, w_grad_rows, wide_model_params  # noqa: E402

LSTM_CASES = [
    # name, cells S (not a multiple of 128), T, hidden
    ("lstmw_s50_t1_c96", 50, 1, 96),
    ("lstmw_s50_t7_c96", 50, 7, 96),
    ("lstmw_s37_t1_c128", 37, 1, 128),
    ("lstmw_s37_t7_c128", 37, 7, 128),
]

MODEL_CASES = [
    # name, N, K, support kind, T, B, hidden
    ("mpgcnw_n8_k2_h128", 8, 2, "rw", 5, 2, 128),
]


def lstm_params(seed, C):
    """nn.LSTM(1, C) parameters from the seed alone, in nn.LSTM's default range U(+-1/sqrt(C)) -> {name: float32 array}."""
    rng = np.random.default_rng(seed)
    a = 1.0 / np.sqrt(C)
    shapes = {"w_ih": (4 * C, 1), "w_hh": (4 * C, C), "b_ih": (4 * C,), "b_hh": (4 * C,)}
    return {k: rng.uniform(-a, a, s).astype(np.float32) for k, s in shapes.items()}


def gen_lstm():
    for idx, (name, S, T, C) in enumerate(LSTM_CASES):
        seed = 9000 + idx
        params = lstm_params(seed, C)
        rng = np.random.default_rng(seed + 50)
        lstm = torch.nn.LSTM(input_size=1, hidden_size=C, num_layers=1, batch_first=True)   # MPGCN.py:69
        with torch.no_grad():
            for k, attr in (("w_ih", "weight_ih_l0"), ("w_hh", "weight_hh_l0"), ("b_ih", "bias_ih_l0"), ("b_hh", "bias_hh_l0")):
                getattr(lstm, attr).copy_(torch.from_numpy(params[k]))
        x = (rng.random((S, T, 1)) * 8).astype(np.float32)       # log1p(flow)-like range
        d_h = rng.standard_normal((S, C)).astype(np.float32)
        xt = torch.from_numpy(x).requires_grad_(True)
        h0 = torch.zeros(1, S, C)
        out, _ = lstm(xt, (h0, h0.clone()))                      # MPGCN.py:80-87,103
        hT = out[:, -1, :]                                       # MPGCN.py:104
        hT.backward(torch.from_numpy(d_h))
        dw_hh = _np(lstm.weight_hh_l0.grad)
        rows = w_grad_rows(dw_hh.shape[0])
        np.savez_compressed(os.path.join(OUT, name + ".npz"), x=x, d_hT=d_h, hT=_np(hT), dx=_np(xt.grad), seed=seed, C=C,
                            params_checksum=params_checksum(params), dw_ih=_np(lstm.weight_ih_l0.grad),
                            dw_hh_rows=dw_hh[rows], dw_hh_row_ids=rows, dw_hh_norm=np.float64(np.linalg.norm(dw_hh.astype(np.float64))),
                            db_ih=_np(lstm.bias_ih_l0.grad), db_hh=_np(lstm.bias_hh_l0.grad))
        print("wrote", name)


def _gen_one_model(ref_mpgcn, ref_gcn, seed, N, K, gk, T, B, hid, lstm_num_layers=1):
    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    model = ref_mpgcn.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=lstm_num_layers, gcn_hidden_dim=hid, gcn_num_layers=3,
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
    rec = dict(x_seq=x_seq, G_static=g_static, G_o=g_o, G_d=g_d, d_y=d_y, y=_np(y), K=K, hidden=hid, seed=seed,
               params_checksum=params_checksum(params))
    for k, p in model.named_parameters():
        g = _np(p.grad)
        if g.ndim == 2 and g.shape[0] > W_ROWS and g.shape[1] >= 96:
            rows = w_grad_rows(g.shape[0])
            rec["grad_rows:" + k] = g[rows]
            rec["grad_row_ids:" + k] = rows
            rec["grad_norm:" + k] = np.float64(np.linalg.norm(g.astype(np.float64)))
        else:
            rec["grad:" + k] = g
    return rec


def gen_models(ref_mpgcn, ref_gcn):
    """As tools.gen_golden_wide.gen_wide_models: the first seed whose run gives every parameter of both branches a gradient."""
    for idx, (name, N, K, gk, T, B, hid) in enumerate(MODEL_CASES):
        for seed in range(9500 + idx, 12000, 100):
            rec = _gen_one_model(ref_mpgcn, ref_gcn, seed, N, K, gk, T, B, hid)
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
    gen_lstm()
    gen_models(ref_mpgcn, ref_gcn)


if __name__ == "__main__":
    main()
