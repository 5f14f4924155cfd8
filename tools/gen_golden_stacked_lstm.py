"""Generate the stacked-LSTM fixtures `tests/golden/lstms_*.npz` and `tests/golden/mpgcns_*.npz` by running the UNMODIFIED reference.

TEST INFRASTRUCTURE ONLY, like tools/gen_golden_wide_lstm.py, whose helpers it reuses.  These pin nn.LSTM(1, H, L) alone and
one whole model with lstm_num_layers = 2, at hidden 32 and 96.  Run where a checkout of the reference is available
(MPGCN_REFERENCE_DIR):

    python tools/gen_golden_stacked_lstm.py

Seeds are their own (LSTM 9600 + i, model 9800 + 100 j), so no other fixture changes.  Parameters are drawn from the seed
(`stacked_lstm_params`, `wide_model_params`) and only their checksum is stored; of each gradient with more than `W_ROWS` rows
of width >= 96 only `W_ROWS` rows and the norm of the whole tensor are kept (`dw_hh_l{l}_rows`, ... as in the wide fixtures).
The prefixes `lstms_` / `mpgcns_` keep them out of the tests that collect `lstm_*` / `mpgcn_*` fixtures.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.gen_golden import OUT, REF, _load_ref, _np  # noqa: E402
from tools.gen_golden_wide import W_ROWS, params_checksum, w_grad_rows, wide_model_params  # noqa: E402
from tools.gen_golden_wide_lstm import _gen_one_model  # noqa: E402

LSTM_CASES = [
    # name, cells S (not a multiple of the 128 / 64-cell tiles), T, hidden, layers
    ("lstms_s150_t1_c32_l2", 150, 1, 32, 2),
    ("lstms_s150_t7_c32_l3", 150, 7, 32, 3),
    ("lstms_s70_t1_c96_l3", 70, 1, 96, 3),
    ("lstms_s70_t7_c96_l2", 70, 7, 96, 2),
]

MODEL_CASES = [
    # name, N, K, support kind, T, B, hidden, layers
    ("mpgcns_n9_k2_h32_l2", 9, 2, "rw", 5, 2, 32, 2),
    ("mpgcns_n8_k2_h96_l2", 8, 2, "rw", 4, 2, 96, 2),
]

KEYS = ("w_ih", "w_hh", "b_ih", "b_hh")


def stacked_lstm_params(seed, C, L):
    """nn.LSTM(1, C, L) parameters from the seed alone, in nn.LSTM's default range U(+-1/sqrt(C)) -> {"w_ih_l0": ..., ...}."""
    rng = np.random.default_rng(seed)
    a = 1.0 / np.sqrt(C)
    out = {}
    for l in range(L):
        shapes = {"w_ih": (4 * C, 1 if l == 0 else C), "w_hh": (4 * C, C), "b_ih": (4 * C,), "b_hh": (4 * C,)}
        for k, s in shapes.items():
            out[f"{k}_l{l}"] = rng.uniform(-a, a, s).astype(np.float32)
    return out


def _store_grad(rec, key, g):
    if g.ndim == 2 and g.shape[0] > W_ROWS and g.shape[1] >= 96:
        rows = w_grad_rows(g.shape[0])
        rec[key + "_rows"] = g[rows]
        rec[key + "_row_ids"] = rows
        rec[key + "_norm"] = np.float64(np.linalg.norm(g.astype(np.float64)))
    else:
        rec[key] = g


def gen_lstm():
    for idx, (name, S, T, C, L) in enumerate(LSTM_CASES):
        seed = 9600 + idx
        params = stacked_lstm_params(seed, C, L)
        rng = np.random.default_rng(seed + 50)
        lstm = torch.nn.LSTM(input_size=1, hidden_size=C, num_layers=L, batch_first=True)   # MPGCN.py:69
        attrs = {"w_ih": "weight_ih", "w_hh": "weight_hh", "b_ih": "bias_ih", "b_hh": "bias_hh"}
        with torch.no_grad():
            for k, v in params.items():
                base, l = k.rsplit("_l", 1)
                getattr(lstm, f"{attrs[base]}_l{l}").copy_(torch.from_numpy(v))
        x = (rng.random((S, T, 1)) * 8).astype(np.float32)       # log1p(flow)-like range
        d_h = rng.standard_normal((S, C)).astype(np.float32)
        xt = torch.from_numpy(x).requires_grad_(True)
        h0 = torch.zeros(L, S, C)
        out, _ = lstm(xt, (h0, h0.clone()))                      # MPGCN.py:80-87,103
        hT = out[:, -1, :]                                       # MPGCN.py:104
        hT.backward(torch.from_numpy(d_h))
        rec = dict(x=x, d_hT=d_h, hT=_np(hT), dx=_np(xt.grad), seed=seed, C=C, L=L, params_checksum=params_checksum(params))
        for l in range(L):
            for k in KEYS:
                _store_grad(rec, f"d{k}_l{l}", _np(getattr(lstm, f"{attrs[k]}_l{l}").grad))
        np.savez_compressed(os.path.join(OUT, name + ".npz"), **rec)
        print("wrote", name)


def gen_models(ref_mpgcn, ref_gcn):
    """As tools.gen_golden_wide_lstm.gen_models, with lstm_num_layers = L."""
    for idx, (name, N, K, gk, T, B, hid, L) in enumerate(MODEL_CASES):
        for seed in range(9800 + idx, 12000, 100):
            rec = _gen_one_model(ref_mpgcn, ref_gcn, seed, N, K, gk, T, B, hid, lstm_num_layers=L)
            if rec is not None:
                break
        else:
            raise RuntimeError(f"{name}: no seed with two live branches")
        rec["lstm_num_layers"] = L
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
