"""Precision 2, "bf16x3", of the BDGCN layer (DESIGN.md section 3) without a GPU: the numpy emulation of its pair arithmetic
(tests/bf16x3_oracle.py) against the layer fixtures, the refusals of the Python layer, the names that keep their meaning, and the
C ABI's answers and refusals before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

import bf16x3_oracle as em
from conftest import golden_names, load_golden
from oracle import mpgcn_oracle as orc
from oracle.gen_golden import layer_fixture

from mpgcn_b200 import _lib, ops

FWD_BAR, GRAD_BAR = 1e-4, 2e-4       # the GPU bars of tests/test_gpu_bf16x3.py


def _graph(g):
    return (g["G_o"], g["G_d"]) if int(g["dynamic"]) else g["G"]


def _f64(a):
    return tuple(x.astype(np.float64) for x in a) if isinstance(a, tuple) else a.astype(np.float64)


@pytest.mark.parametrize("name", golden_names("bdgcn_") + golden_names("wide_bdgcn_") + golden_names("many_bdgcn_"))
def test_emulated_pair_arithmetic_meets_the_gpu_bars(name):
    """The pair scheme itself reaches the bars: forward against the reference's output, gradients against the float64 oracle on the
    emulation's own ReLU mask (the convention of DESIGN.md section 3)."""
    g = layer_fixture(load_golden(name))
    act = str(g["act"])
    b = g.get("b")
    out, dX, dW, db = em.backward(g["X"], _graph(g), g["W"], b, g["d_out"], act == "relu")
    linf, l2 = orc.rel_errors(out, g["out"])
    assert max(linf, l2) <= FWD_BAR, f"{name}: out rel_Linf={linf:.2e} rel_L2={l2:.2e}"
    refs = orc.bdgcn_backward_factored(_f64(g["X"]), _f64(_graph(g)), _f64(g["W"]), None if b is None else _f64(b), act,
                                       _f64(g["d_out"]), mask_from=out)[1:]
    for a, r, k in zip((dX, dW, db), refs, ("dX", "dW", "db")):
        if r is None:
            continue
        linf, l2 = orc.rel_errors(a, r)
        assert max(linf, l2) <= GRAD_BAR, f"{name}: {k} rel_Linf={linf:.2e} rel_L2={l2:.2e}"


def test_emulated_rounding_is_round_to_nearest_even():
    x = np.array([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 1.0 + 2.0 ** -8 + 2.0 ** -20], dtype=np.float32)
    assert em.bf16_rn(x).tolist() == [1.0, 1.0, 1.0 + 2.0 ** -6, -1.0, 1.0 + 2.0 ** -7]
    hi, lo = em.split(np.float32(np.pi))
    assert abs(float(hi) + float(lo) - np.pi) < 2.0 ** -15


def test_names_keep_their_meaning(monkeypatch):
    """"bf16" stays unknown, "auto" never picks bf16x3, and the LSTM reads "bf16x3" as "auto"."""
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    with pytest.raises(ValueError, match="unknown precision"):
        ops.resolve_precision("bf16", 2, 50, 3, 32, 32)
    assert ops.resolve_precision("auto", 2, 50, 3, 32, 32) == _lib.PREC_FP16_TC
    assert ops.resolve_precision("auto", 2, 50, 3, 16, 32) == _lib.PREC_FP32
    assert ops.resolve_precision("bf16x3", 2, 50, 3, 64, 96) == _lib.PREC_BF16X3
    with pytest.raises(RuntimeError, match="does not support"):
        ops.resolve_precision("bf16x3", 2, 50, 3, 16, 32)
    for T, C in ((8, 32), (8, 128), (20, 64)):
        assert ops.resolve_lstm_precision("bf16x3", T, C) == ops.resolve_lstm_precision("auto", T, C)
        assert ops.lstm_stack_supports("bf16x3", T, C, 2) == ops.lstm_stack_supports("auto", T, C, 2)
    monkeypatch.setenv("MPGCN_B200_PRECISION", "bf16x3")
    assert ops.resolve_precision(None, 2, 50, 3, 32, 32) == _lib.PREC_BF16X3
    assert ops.resolve_lstm_precision(None, 8, 32) == ops.resolve_lstm_precision("auto", 8, 32)
    lstm = torch.nn.LSTM(1, 32, batch_first=True)
    assert ops.lstm_runs_on_engine(lstm, 8, "bf16x3") == ops.lstm_runs_on_engine(lstm, 8, "auto")


def test_python_refusals():
    X = torch.zeros(1, 4, 4, 32)
    G = torch.zeros(2, 4, 4)
    W = torch.zeros(2 * 2 * 32, 32)
    with pytest.raises(RuntimeError, match="no bf16x3 sparse kernels"):
        ops.bdgcn(X, G.to_sparse(), W, None, True, precision="bf16x3")
    with pytest.raises(NotImplementedError, match="no support gradient"):
        ops.bdgcn(X, G, W, None, True, precision="bf16x3", support_grad=True)


def test_sharded_layer_refuses_bf16x3(monkeypatch):
    from mpgcn_b200 import shard

    class Ctx:
        needs_input_grad = (True, False, False, True, False)

    monkeypatch.setattr(shard._ENGINE, "resolve_precision", lambda name, *shape: ops._PREC_NAMES[name])
    with pytest.raises(NotImplementedError, match="bf16x3"):
        shard._begin_forward(Ctx(), torch.zeros(1, 1, 4, 32), torch.zeros(2, 4, 4), torch.zeros(2, 4, 4), torch.zeros(128, 32), None,
                             False, 1, "bf16x3", None, True, 1)


def _err(lib):
    return lib.mpgcn_last_error().decode()


def test_c_abi_answers_and_refusals_before_any_cuda_call():
    lib = _lib.load()
    for shape in ((2, 50, 3, 32, 32), (2, 50, 3, 16, 32), (1, 9, 11, 64, 96), (2, 50, 3, 32, 2048)):
        assert lib.mpgcn_bdgcn_precision_supported(*shape, 2) == lib.mpgcn_bdgcn_precision_supported(*shape, 1)
    assert lib.mpgcn_bdgcn_precision_supported(2, 50, 3, 32, 32, 7) == 0
    # the whole layer: sizes; the stash is twice the fp16 one
    assert lib.mpgcn_bdgcn_saved_bytes(2, 50, 3, 32, 32, 2) == 2 * lib.mpgcn_bdgcn_saved_bytes(2, 50, 3, 32, 32, 1)
    for dyn in (0, 1):
        assert lib.mpgcn_bdgcn_fwd_workspace_bytes(2, 50, 3, 32, 32, dyn, 2) > lib.mpgcn_bdgcn_fwd_workspace_bytes(2, 50, 3, 32, 32, dyn, 1)
        assert lib.mpgcn_bdgcn_bwd_workspace_bytes(2, 50, 3, 32, 32, dyn, 2) > lib.mpgcn_bdgcn_bwd_workspace_bytes(2, 50, 3, 32, 32, dyn, 1)
        assert lib.mpgcn_bdgcn_support_grad_workspace_bytes(2, 50, 3, 32, 32, dyn, 2) == 0
    assert lib.mpgcn_bdgcn_supports_prepared_bytes_ex(3, 50, 2) == -(-2 * 3 * 50 * 56 * 2 // 256) * 256     # the pair, 256-byte aligned
    assert lib.mpgcn_bdgcn_supports_prepared_bytes_ex(3, 50, 1) == lib.mpgcn_bdgcn_supports_prepared_bytes(3, 50)
    assert lib.mpgcn_bdgcn_supports_prepared_bytes_ex(3, 50, 0) == 0
    part = _lib.BdgcnPart(row0=0, rows=25, Ko=3, Kd=3)
    pp = ctypes.byref(part)
    assert lib.mpgcn_bdgcn_part_saved_bytes(2, 50, 32, 32, 2, pp) == 0
    assert lib.mpgcn_bdgcn_part_fwd_workspace_bytes(2, 50, 32, 32, 0, 2, pp) == 0
    assert lib.mpgcn_bdgcn_part_bwd_workspace_bytes(2, 50, 32, 32, 0, 2, pp) == 0
    # refusals: dangling (non-null, never dereferenced) pointers show that nothing reaches the device
    one = 1 << 20
    assert lib.mpgcn_bdgcn_forward_part(one, one, one, 0, one, one, None, one, 1 << 30, 2, 50, 32, 32, 2, pp, None, None) != 0
    assert "bf16x3" in _err(lib)
    assert lib.mpgcn_bdgcn_backward_part(one, one, one, 0, one, one, one, one, one, 1 << 30, 2, 50, 32, 32, 2, pp, None, None) != 0
    assert "bf16x3" in _err(lib)
    assert lib.mpgcn_bdgcn_backward_supports(one, one, one, one, 0, one, 1, one, one, one, one, one, 1 << 30, 2, 50, 3, 32, 32, 2, None,
                                             one, one, None, None) != 0
    assert "support gradient" in _err(lib)
    for field in ("x_f16", "out_f16"):
        ex = _lib.BdgcnExtras()
        setattr(ex, field, one)
        assert lib.mpgcn_bdgcn_forward_x(one, one, one, 0, one, None, 1, one, None, one, 1 << 30, 2, 8, 3, 32, 32, 2,
                                         ctypes.addressof(ex), None) != 0 and "bf16x3" in _err(lib)
        assert lib.mpgcn_bdgcn_backward_x(one, one, one, one, 0, one, 1, one, one, one, one, one, 1 << 30, 2, 8, 3, 32, 32, 2,
                                          ctypes.addressof(ex), None) != 0 and "bf16x3" in _err(lib)
    assert lib.mpgcn_bdgcn_prepare_supports_ex(one, one, 1 << 30, 3, 50, 0, None) != 0
    assert lib.mpgcn_bdgcn_forward(one, one, one, 0, one, None, 1, one, None, one, 1 << 20, 2, 8, 3, 16, 32, 2, None) != 0
    assert "precision 2" in _err(lib)
    # the LSTM entry points do not take it
    assert lib.mpgcn_lstm_precision_supported(8, 32, 2) == 0
