"""The deterministic mode's host surface, without a GPU: the per-thread switch, the workspace each affected query adds for its
slots (DESIGN.md section 11), the refusals before any CUDA call, and an audit of every floating-point atomicAdd in the sources."""
import ctypes
import os
import re
import threading

import pytest
import torch

from mpgcn_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "mpgcn_b200", "csrc")
P = 1 << 20                      # a plausible, aligned, never dereferenced device address


def sms():
    """The SM count the library sizes its slots with: the current device's, or 132 when there is none."""
    if torch.cuda.is_available():
        return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return 132


def a256(x):
    return (x + 255) // 256 * 256


@pytest.fixture
def det():
    """Runs the test body's queries in both modes: det(True) / det(False); always leaves the thread's mode off."""
    lib = _lib.load()
    yield lambda on: lib.mpgcn_set_deterministic(int(on))
    lib.mpgcn_set_deterministic(0)
    _lib._DET.on = False


def test_switch_is_per_thread(det):
    lib = _lib.load()
    assert lib.mpgcn_get_deterministic() == 0
    assert lib.mpgcn_set_deterministic(1) == 0
    assert lib.mpgcn_get_deterministic() == 1
    seen = []
    t = threading.Thread(target=lambda: seen.append(lib.mpgcn_get_deterministic()))
    t.start()
    t.join()
    assert seen == [0], "another host thread sees the default"
    assert lib.mpgcn_set_deterministic(0) == 1
    assert lib.mpgcn_get_deterministic() == 0


def test_python_cache_sets_the_mode_only_when_it_changes(det, monkeypatch):
    lib = _lib.load()
    calls = []
    real = lib.mpgcn_set_deterministic
    monkeypatch.setattr(lib, "mpgcn_set_deterministic", lambda on: calls.append(on) or real(on))
    assert _lib.sync_deterministic() is False and calls == [], "the default path makes no call"
    torch.use_deterministic_algorithms(True)
    try:
        assert _lib.sync_deterministic() is True and _lib.sync_deterministic() is True
    finally:
        torch.use_deterministic_algorithms(False)
    assert calls == [1] and lib.mpgcn_get_deterministic() == 1
    assert _lib.sync_deterministic() is False and calls == [1, 0]


# ------------------------------------------------------------------------------------------------------------------------------
# slot sizes: mode off = what the query always returned, mode on = that + the documented slots
# ------------------------------------------------------------------------------------------------------------------------------
def lstm_slots(C, up=False):
    G4 = 4 * C
    image = G4 * C + G4 * (C if up else 1) + G4
    n = sms() if (C == 32 and not up) else 4 * sms() // (C // 32)
    return a256(n * image * 4)


def bias_slots(H):
    return a256(16 * sms() * H * 4)


def simt_dw_slices(R, N, Ko, Kd, C, H):
    ks = min(max(R * N // 2048, 1), 256)
    return a256(ks * ((Kd * C + 127) // 128) * 128 * Ko * H * 4) if ks > 1 else 0


def head_slots(cells, C, M):
    grid = min(max((cells + 31) // 32, 1), 8 * sms())
    return a256(grid * M * (C + 1) * 4)


def both(det, q):
    det(False)
    off = q()
    det(True)
    on = q()
    det(False)
    assert q() == off
    return off, on


@pytest.mark.parametrize("B,T,NN,C", [(2, 12, 10000, 32), (1, 7, 3600, 96), (4, 3, 999, 128)])
def test_lstm_tc_workspace(det, B, T, NN, C):
    lib = _lib.load()
    off, on = both(det, lambda: lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, 1))
    assert on - off == lstm_slots(C)


@pytest.mark.parametrize("C", [1, 16, 48, 64])
def test_lstm_fp32_workspace(det, C):
    lib = _lib.load()
    off, on = both(det, lambda: lib.mpgcn_lstm_bwd_workspace_bytes(2, 5, 100, C, 0))
    assert off == 256 and on == 256 + a256(sms() * (4 * C * C + 8 * C) * 4)


@pytest.mark.parametrize("B,T,NN,C,L", [(2, 12, 10000, 32, 2), (1, 7, 3600, 96, 2), (1, 4, 500, 96, 3)])
def test_lstm_stack_workspace(det, B, T, NN, C, L):
    lib = _lib.load()
    off, on = both(det, lambda: lib.mpgcn_lstm_stack_bwd_workspace_bytes(B, T, NN, C, L, 1))
    assert on - off == lstm_slots(C, up=True)


@pytest.mark.parametrize("B,N,K,C,H,dyn", [(2, 60, 3, 32, 32, 0), (1, 200, 2, 64, 96, 1), (3, 47, 1, 32, 64, 0), (1, 17, 3, 8, 12, 1)])
def test_bdgcn_workspaces(det, B, N, K, C, H, dyn):
    lib = _lib.load()
    for prec in (0, 1):
        if not lib.mpgcn_bdgcn_precision_supported(B, N, K, C, H, prec):
            continue
        extra = bias_slots(H) + (simt_dw_slices(N, N, K, K, C, H) if prec == 0 else 0)
        off, on = both(det, lambda: lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, dyn, prec))
        assert on - off == extra, prec
        off, on = both(det, lambda: lib.mpgcn_bdgcn_support_grad_workspace_bytes(B, N, K, C, H, dyn, prec))
        assert on - off == extra, prec
        for row0, rows, Ko, Kd in ((0, N, K, K), (N // 3, N - N // 3, K, K), (0, N, K, 1)):
            part = _lib.BdgcnPart(row0, rows, Ko, Kd)
            off, on = both(det, lambda: lib.mpgcn_bdgcn_part_bwd_workspace_bytes(B, N, C, H, dyn, prec, ctypes.addressof(part)))
            assert on - off == bias_slots(H) + (simt_dw_slices(rows, N, Ko, Kd, C, H) if prec == 0 else 0), (prec, row0, rows, Kd)


def test_dyn_graph_and_head_workspace(det):
    lib = _lib.load()
    for P_, N in ((7, 500), (3, 33)):
        off, on = both(det, lambda: lib.mpgcn_dyn_graph_workspace_bytes(P_, N))
        assert on == off, "the fixed-order column norms read the average directly: no slots"
    for cells, C, M in ((10 ** 6, 32, 2), (1000, 256, 8), (1, 4, 1)):
        off, on = both(det, lambda: lib.mpgcn_head_backward_workspace_bytes(cells, C, M))
        assert off == 0 and on == head_slots(cells, C, M)


# ------------------------------------------------------------------------------------------------------------------------------
# refusals, all before any CUDA call (fake addresses)
# ------------------------------------------------------------------------------------------------------------------------------
def _err(lib):
    return lib.mpgcn_last_error().decode()


def test_refusals_before_any_cuda_call(det):
    lib = _lib.load()
    M, C, cells = 2, 32, 1000
    g = (ctypes.c_void_p * M)(P, P)
    det(True)
    assert lib.mpgcn_head_backward(g, P, P, P, g, P, P, P, cells, C, M, None) != 0
    assert "mpgcn_head_backward_ex" in _err(lib)
    need = lib.mpgcn_head_backward_workspace_bytes(cells, C, M)
    assert lib.mpgcn_head_backward_ex(g, P, P, P, g, P, P, P, cells, C, M, P, need - 256, None) != 0
    assert "workspace too small" in _err(lib)
    assert lib.mpgcn_head_backward_ex(g, P, P, P, g, P, P, P, cells, C, M, None, need, None) != 0
    assert lib.mpgcn_relu_backward(P, P, 1, P, P, 1024, 32, None) != 0 and "no deterministic implementation" in _err(lib)
    arr = (ctypes.c_void_p * 2)(P, P)
    assert lib.mpgcn_relu_backward_scatter(P, P, 1, arr, 2, P, 1, 8, 0, 4, 32, None) != 0
    assert "no deterministic implementation" in _err(lib)
    assert lib.mpgcn_relu_backward_scatter_f16(P, P, 1, arr, 2, P, P, P, 1, 8, 0, 4, 32, None) != 0
    assert "no deterministic implementation" in _err(lib)
    # a workspace sized in the default mode is refused in the deterministic one
    B, T, NN = 1, 4, 1000
    for Cl, prec in ((32, 1), (96, 1), (16, 0)):
        det(False)
        small = lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, Cl, prec)
        det(True)
        r = lib.mpgcn_lstm_last_backward(*([P] * 11), P, small, B, T, NN, Cl, prec, None)
        assert r != 0 and "workspace too small" in _err(lib), (Cl, prec)
    det(False)
    small = lib.mpgcn_lstm_stack_bwd_workspace_bytes(B, T, NN, 32, 2, 1)
    det(True)
    arr4 = (ctypes.c_void_p * 2)(P, P)
    r = lib.mpgcn_lstm_stack_backward(P, 2, arr4, arr4, arr4, arr4, P, arr4, arr4, arr4, arr4, P, P,
                                      lib.mpgcn_lstm_stack_saved_bytes(B, T, NN, 32, 2, 1), P, small, B, T, NN, 32, 1, None, None)
    assert r != 0 and "workspace too small" in _err(lib)
    for prec, (Cb, Hb) in ((0, (8, 12)), (1, (32, 32))):
        det(False)
        small = lib.mpgcn_bdgcn_bwd_workspace_bytes(2, 40, 2, Cb, Hb, 0, prec)
        det(True)
        r = lib.mpgcn_bdgcn_backward(P, P, P, P, 0, P, 1, P, P, P, P, P, small, 2, 40, 2, Cb, Hb, prec, None)
        assert r != 0 and "workspace too small" in _err(lib), prec


# ------------------------------------------------------------------------------------------------------------------------------
# source audit: a kernel that adds a floating-point atomicAdd has to say whether it breaks the deterministic mode
# ------------------------------------------------------------------------------------------------------------------------------
# function -> why it is allowed: each has a fixed-order alternative that the deterministic mode runs instead
AUDITED = {
    ("lstm_tc.cu", "lstm_bwd_saved_tc_kernel"): "DET = false only; DET = true stores to its slot",
    ("lstm_tc.cu", "lstm_dw_tcw_kernel"): "DET = false only; DET = true stores to its split's slot",
    ("lstm_kernels.cu", "lstm_bwd_kernel"): "DET = false only; DET = true stores to its slot",
    ("head_kernels.cu", "head_bwd_kernel"): "the deterministic mode runs head_bwd_det_kernel",
    ("simt_kernels.cu", "sgemm_kernel"): "ksplit > 1 with d_sslice == 0 only; the deterministic dW sets d_sslice",
    ("simt_kernels.cu", "block_bias_grad"): "without slots only; the deterministic mode passes them",
    ("dyn_graph_kernels.cu", "norms_kernel"): "COLS = true only; the deterministic mode runs COLS = false + col_norms_kernel",
}
_HEADER = re.compile(r"^(?!\s)(?!//)(?!#).*?\b(\w+)\s*\(")
_SKIP = {"__launch_bounds__", "__align__", "if", "for", "while", "switch", "return", "sizeof"}


def _atomic_sites():
    sites = []
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh", ".h")):
            continue
        func = None
        for ln, line in enumerate(open(os.path.join(CSRC, name)), 1):
            if not line.startswith((" ", "\t", "/", "#", "}")) and "(" in line:
                idents = [m for m in re.findall(r"\b(\w+)\s*\(", line) if m not in _SKIP]
                if idents:
                    func = idents[0]
            code = line.split("//")[0]
            for _ in re.finditer(r"\batomicAdd\s*\(", code):
                sites.append((name, func, ln))
    return sites


def test_every_float_atomic_add_is_audited():
    sites = _atomic_sites()
    assert sites, "the scan found no atomicAdd at all: the scanner is broken"
    unaudited = [s for s in sites if (s[0], s[1]) not in AUDITED]
    assert not unaudited, f"atomicAdd outside the audited functions (does it break the deterministic mode?): {unaudited}"
    assert {(s[0], s[1]) for s in sites} == set(AUDITED), "an audited function no longer has an atomicAdd: drop it from the list"
