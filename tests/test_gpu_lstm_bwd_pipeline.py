"""The hidden-32 tensor-core LSTM backward without d_x, and the edges of its pipelined walk.

lstm_bwd_saved_tc_kernel has two instances: one writes d_x, the other (taken when d_x is null, as in a model's training step,
where x needs no gradient) skips that sum.  Both are held to the stage bounds of tests/test_gpu_lstm_stages.py.

The kernel streams the saved state and x of a CTA's walk through a ring of 3 slots, two steps ahead, and hands each step's gate
gradients and operand rows between its warps through a ring of the same depth, so the walk's sequence of (tile, step) entries
crosses tile boundaries inside both rings.  The edge cases run one cell past two full backward grids of tiles (one CTA per SM:
every CTA walks two tiles, CTA 0 a third with one live cell) at T = 1, the ring depth and the ring depth + 1.
"""
import math

import numpy as np
import pytest
import torch

from mpgcn_b200 import _lib
from oracle import lstm_tc_oracle as emu
from test_gpu_lstm_stages import TC_TILE, _assert_and_record, _garbage, _tc_cases, check_tc, run_tc, tc_inputs

C = 32
RING = 3                   # lstm_tc.cu kBwdRing


def run_saved_without_dx(x, ws, d_hT, dev):
    """Training forward + backward_saved with d_x = nullptr -> the weight gradients, the gradient scale and the saved state."""
    lib = _lib.load()
    B, T, NN = x.shape
    st = torch.cuda.current_stream().cuda_stream
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    p = lambda a: a.data_ptr()
    xt, wt, dh = t(x), [t(w) for w in ws], t(d_hT)
    hT = torch.empty((B * NN, C), device=dev)
    nsave = lib.mpgcn_lstm_saved_bytes(B, T, NN, C, 1)
    saved = _garbage(nsave, dev)
    _lib.check(lib.mpgcn_lstm_last_forward_train(p(xt), *[p(w) for w in wt], p(hT), p(saved), nsave, B, T, NN, C, 1, st), "fwd_train")
    g = [torch.full_like(w, math.nan) for w in wt]
    wsb = _garbage(lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, 1) - nsave, dev)
    _lib.check(lib.mpgcn_lstm_last_backward_saved(p(xt), *[p(w) for w in wt], p(dh), *[p(a) for a in g], None, p(saved), nsave,
                                                  p(wsb), wsb.numel(), B, T, NN, C, 1, None, st), "bwd_saved without d_x")
    torch.cuda.synchronize()
    return dict(scale2=wsb[:8].view(torch.float32).cpu().numpy().astype(np.float64),
                dw_ih=g[0].cpu().numpy()[:, 0].astype(np.float64), dw_hh=g[1].cpu().numpy().astype(np.float64),
                db=g[2].cpu().numpy().astype(np.float64), db_hh=g[3].cpu().numpy().astype(np.float64),
                state=saved.view(torch.float16).cpu().numpy())


def check_both_instances(B, NN, T, xmag, gmag, dev, tag):
    x, x_cells, ws, d_hT = tc_inputs(C, B, NN, T, xmag, gmag, seed=C * 7 + B * NN + T)
    r = run_tc(x, ws, d_hT, C, "saved", dev)
    res, l2 = check_tc(r, x_cells, ws, d_hT, C, f"{tag} with d_x")
    _assert_and_record(res, l2, f"{tag} with d_x")
    n = run_saved_without_dx(x, ws, d_hT, dev)
    # the same forward ran before both: the stages other than the weight gradients are those of the run with d_x
    _, h_n = emu.decode_saved(n["state"], B * NN, T, C)
    assert np.array_equal(h_n, r["h"]), f"{tag}: the training forward is not deterministic"
    res, l2 = check_tc(dict(r, **{k: n[k] for k in ("scale2", "dw_ih", "dw_hh", "db", "db_hh")}), x_cells, ws, d_hT, C, f"{tag} without d_x")
    l2.pop("dx")                  # dx of the run with d_x, checked above
    _assert_and_record(res, l2, f"{tag} without d_x")


@pytest.mark.gpu
@pytest.mark.parametrize("C_,B,NN,T,xmag,gmag", [row for row in _tc_cases() if row[0] == C])
def test_backward_without_dx_meets_the_stage_bounds(C_, B, NN, T, xmag, gmag, cuda_device):
    if NN == "grid":
        sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
        NN = (sms * 2 * TC_TILE[C]) // 2 + 1
    check_both_instances(B, NN, T, xmag, gmag, cuda_device, f"C={C} B={B} NN={NN} T={T} |x|~{xmag:g} |dh|~{gmag:g}")


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, RING, RING + 1])
def test_walk_crosses_tiles_inside_the_rings(T, cuda_device):
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    NN = 2 * sms * TC_TILE[C] + 1
    check_both_instances(1, NN, T, 8.0, 1.0, cuda_device, f"C={C} NN={NN} (2 grids + 1) T={T}")
