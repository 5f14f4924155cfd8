"""ctypes binding of libmpgcn_b200.so (C ABI: include/mpgcn_b200.h).

The shared library is built in-tree by `mpgcn_b200/csrc/Makefile` (`__graft_entry__.build()`),
for sm_90a only.  There is deliberately no fallback: if the library is missing or a call
fails, a RuntimeError is raised -- the product never silently computes on another path.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmpgcn_b200.so")
CSRC = os.path.join(_HERE, "csrc")

PREC_FP32 = 0      # exact fp32 CUDA-core kernels
PREC_FP16_TC = 1   # fp16 operands / fp32 accumulate on tensor cores (wgmma / mma.sync)

_lib = None

_c_f = ctypes.c_void_p   # device pointers travel as void*
_SIGS = {
    "mpgcn_abi_version": (ctypes.c_int, []),
    "mpgcn_last_error": (ctypes.c_char_p, []),
    "mpgcn_bdgcn_precision_supported": (ctypes.c_int, [ctypes.c_int] * 6),
    "mpgcn_bdgcn_saved_bytes": (ctypes.c_size_t, [ctypes.c_int] * 6),
    "mpgcn_bdgcn_fwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int] * 7),
    "mpgcn_bdgcn_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int] * 7),
    "mpgcn_bdgcn_forward": (ctypes.c_int, [_c_f, _c_f, _c_f, ctypes.c_int, _c_f, _c_f, ctypes.c_int, _c_f, _c_f, _c_f, ctypes.c_size_t]
                            + [ctypes.c_int] * 6 + [ctypes.c_void_p]),
    "mpgcn_bdgcn_backward": (ctypes.c_int, [_c_f, _c_f, _c_f, _c_f, ctypes.c_int, _c_f, ctypes.c_int, _c_f, _c_f, _c_f, _c_f, _c_f,
                                            ctypes.c_size_t] + [ctypes.c_int] * 6 + [ctypes.c_void_p]),
    "mpgcn_adj_num_supports": (ctypes.c_int, [ctypes.c_int, ctypes.c_int]),
    "mpgcn_adj_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int] * 4),
    "mpgcn_adj_process": (ctypes.c_int, [_c_f, _c_f, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_f, ctypes.c_size_t, ctypes.c_void_p]),
    "mpgcn_head_forward": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), _c_f, _c_f, _c_f, _c_f, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_void_p]),
    "mpgcn_head_backward": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), _c_f, _c_f, _c_f, ctypes.POINTER(ctypes.c_void_p), _c_f, _c_f, _c_f,
                                           ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "mpgcn_profile_enable": (None, [ctypes.c_int]),
    "mpgcn_profile_reset": (None, []),
    "mpgcn_profile_read": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)]),
    "mpgcn_debug_tc_workspace_offset": (ctypes.c_longlong, [ctypes.c_int] * 5),
    "mpgcn_bdgcn_supports_prepared_bytes": (ctypes.c_size_t, [ctypes.c_longlong, ctypes.c_int]),
    "mpgcn_bdgcn_prepare_supports": (ctypes.c_int, [_c_f, _c_f, ctypes.c_size_t, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]),
    "mpgcn_bdgcn_forward_x": (ctypes.c_int, [_c_f, _c_f, _c_f, ctypes.c_int, _c_f, _c_f, ctypes.c_int, _c_f, _c_f, _c_f, ctypes.c_size_t] +
                              [ctypes.c_int] * 6 + [ctypes.c_void_p, ctypes.c_void_p]),
    "mpgcn_bdgcn_backward_x": (ctypes.c_int, [_c_f, _c_f, _c_f, _c_f, ctypes.c_int, _c_f, ctypes.c_int, _c_f, _c_f, _c_f, _c_f, _c_f,
                                              ctypes.c_size_t] + [ctypes.c_int] * 6 + [ctypes.c_void_p, ctypes.c_void_p]),
    "mpgcn_bdgcn_backward_ex": (ctypes.c_int, [_c_f, _c_f, _c_f, _c_f, ctypes.c_int, _c_f, ctypes.c_int, _c_f, _c_f, _c_f, _c_f, _c_f,
                                               ctypes.c_size_t] + [ctypes.c_int] * 6 + [_c_f, _c_f, ctypes.c_void_p]),
    "mpgcn_lstm_last_backward_ex": (ctypes.c_int, [_c_f] * 12 + [ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int,
                                                   ctypes.c_int, _c_f, ctypes.c_void_p]),
    "mpgcn_dyn_graph_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int]),
    "mpgcn_dyn_graph_build": (ctypes.c_int, [_c_f, ctypes.c_int, _c_f, _c_f, ctypes.c_int, ctypes.c_int, _c_f, ctypes.c_size_t, ctypes.c_void_p]),
    "mpgcn_lstm_saved_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int]),
    "mpgcn_lstm_last_forward_train": (ctypes.c_int, [_c_f] * 7 + [ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int,
                                                     ctypes.c_int, ctypes.c_void_p]),
    "mpgcn_lstm_last_backward_saved": (ctypes.c_int, [_c_f] * 12 + [ctypes.c_size_t, _c_f, ctypes.c_size_t, ctypes.c_int, ctypes.c_int,
                                                      ctypes.c_longlong, ctypes.c_int, ctypes.c_int, _c_f, ctypes.c_void_p]),
    "mpgcn_lstm_precision_supported": (ctypes.c_int, [ctypes.c_int] * 3),
    "mpgcn_lstm_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int]),
    "mpgcn_lstm_last_forward": (ctypes.c_int, [_c_f] * 6 + [ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_void_p]),
    "mpgcn_bdgcn_part_saved_bytes": (ctypes.c_size_t, [ctypes.c_int] * 5 + [ctypes.c_void_p]),
    "mpgcn_bdgcn_part_fwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int] * 6 + [ctypes.c_void_p]),
    "mpgcn_bdgcn_part_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int] * 6 + [ctypes.c_void_p]),
    "mpgcn_bdgcn_forward_part": (ctypes.c_int, [_c_f, _c_f, _c_f, ctypes.c_int, _c_f, _c_f, _c_f, _c_f, ctypes.c_size_t] + [ctypes.c_int] * 5 +
                                 [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "mpgcn_bdgcn_backward_part": (ctypes.c_int, [_c_f, _c_f, _c_f, ctypes.c_int, _c_f, _c_f, _c_f, _c_f, _c_f, ctypes.c_size_t] + [ctypes.c_int] * 5 +
                                  [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "mpgcn_relu_backward_scatter_f16": (ctypes.c_int, [_c_f, _c_f, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, _c_f, _c_f, _c_f] +
                                        [ctypes.c_int] * 5 + [ctypes.c_void_p]),
    "mpgcn_absmax": (ctypes.c_int, [_c_f, ctypes.c_longlong, _c_f, ctypes.c_void_p]),
    "mpgcn_rows_reduce_bias_act": (ctypes.c_int, [_c_f, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, _c_f, ctypes.c_int] + [ctypes.c_int] * 5 + [ctypes.c_void_p]),
    "mpgcn_relu_backward_scatter": (ctypes.c_int, [_c_f, _c_f, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, _c_f] + [ctypes.c_int] * 5 +
                                    [ctypes.c_void_p]),
    "mpgcn_bias_act": (ctypes.c_int, [_c_f, _c_f, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]),
    "mpgcn_relu_backward": (ctypes.c_int, [_c_f, _c_f, ctypes.c_int, _c_f, _c_f, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]),
    "mpgcn_lstm_last_backward": (ctypes.c_int, [_c_f] * 12 + [ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_void_p]),
    "mpgcn_lstm_stack_supported": (ctypes.c_int, [ctypes.c_int] * 4),
    "mpgcn_lstm_stack_saved_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "mpgcn_lstm_stack_fwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                                                ctypes.c_int]),
    "mpgcn_lstm_stack_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                                                ctypes.c_int]),
    "mpgcn_lstm_stack_forward": (ctypes.c_int, [_c_f, ctypes.c_int] + [ctypes.POINTER(ctypes.c_void_p)] * 4 + [_c_f, _c_f, ctypes.c_size_t, _c_f,
                                 ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "mpgcn_lstm_stack_backward": (ctypes.c_int, [_c_f, ctypes.c_int] + [ctypes.POINTER(ctypes.c_void_p)] * 4 + [_c_f] +
                                  [ctypes.POINTER(ctypes.c_void_p)] * 4 + [_c_f, _c_f, ctypes.c_size_t, _c_f, ctypes.c_size_t, ctypes.c_int,
                                  ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, _c_f, ctypes.c_void_p]),
    "mpgcn_bdgcn_support_grad_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int] * 7),
    "mpgcn_bdgcn_backward_supports": (ctypes.c_int, [_c_f, _c_f, _c_f, _c_f, ctypes.c_int, _c_f, ctypes.c_int, _c_f, _c_f, _c_f, _c_f, _c_f,
                                                     ctypes.c_size_t] + [ctypes.c_int] * 6 + [ctypes.c_void_p, _c_f, _c_f, _c_f, ctypes.c_void_p]),
    "mpgcn_adj_backward_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int] * 4),
    "mpgcn_adj_process_backward": (ctypes.c_int, [_c_f, _c_f, _c_f, _c_f, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _c_f,
                                                  ctypes.c_size_t, ctypes.c_void_p]),
    "mpgcn_set_deterministic": (ctypes.c_int, [ctypes.c_int]),
    "mpgcn_get_deterministic": (ctypes.c_int, []),
    "mpgcn_head_backward_workspace_bytes": (ctypes.c_size_t, [ctypes.c_longlong, ctypes.c_int, ctypes.c_int]),
    "mpgcn_head_backward_ex": (ctypes.c_int, [ctypes.POINTER(ctypes.c_void_p), _c_f, _c_f, _c_f, ctypes.POINTER(ctypes.c_void_p), _c_f, _c_f,
                                              _c_f, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, _c_f, ctypes.c_size_t, ctypes.c_void_p]),
    "mpgcn_sparse_supports_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int, ctypes.c_longlong]),
    "mpgcn_sparse_supports_build": (ctypes.c_int, [_c_f, _c_f, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, _c_f, ctypes.c_size_t,
                                                   ctypes.c_void_p]),
    "mpgcn_bdgcn_forward_sparse": (ctypes.c_int, [_c_f, _c_f, ctypes.c_size_t, ctypes.c_longlong, _c_f, _c_f, ctypes.c_int, _c_f, _c_f, _c_f,
                                                  ctypes.c_size_t] + [ctypes.c_int] * 5 + [ctypes.c_void_p]),
    "mpgcn_bdgcn_backward_sparse": (ctypes.c_int, [_c_f, _c_f, _c_f, ctypes.c_size_t, ctypes.c_longlong, _c_f, ctypes.c_int, _c_f, _c_f, _c_f,
                                                   _c_f, _c_f, ctypes.c_size_t] + [ctypes.c_int] * 5 + [ctypes.c_void_p]),
    "mpgcn_lstm_recompute_bwd_workspace_bytes": (ctypes.c_size_t, [ctypes.c_int, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                                                    ctypes.c_longlong, ctypes.c_int]),
    "mpgcn_lstm_backward_recompute": (ctypes.c_int, [_c_f, ctypes.c_int] + [ctypes.POINTER(ctypes.c_void_p)] * 4 + [_c_f] +
                                      [ctypes.POINTER(ctypes.c_void_p)] * 4 + [_c_f, ctypes.c_longlong, _c_f, ctypes.c_size_t, ctypes.c_int,
                                      ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, _c_f, ctypes.c_void_p]),
}
ABI_VERSION = 4          # MPGCN_B200_ABI_VERSION of include/mpgcn_b200.h this binding was written against
EXPORTED_SYMBOLS = tuple(_SIGS)


class BdgcnExtras(ctypes.Structure):
    """mpgcn_bdgcn_extras (include/mpgcn_b200.h): optional side inputs / outputs of the tensor-core layer."""
    _fields_ = [("go_prepared", ctypes.c_void_p), ("gd_prepared", ctypes.c_void_p), ("x_f16", ctypes.c_void_p),
                ("out_f16", ctypes.c_void_p), ("d_out_absmax", ctypes.c_void_p), ("dX_absmax", ctypes.c_void_p),
                ("d_pre_f16", ctypes.c_void_p), ("d_pre_scale2", ctypes.c_void_p)]


class BdgcnPart(ctypes.Structure):
    """mpgcn_bdgcn_part (include/mpgcn_b200.h): origin rows [row0, row0 + rows), Ko origin / Kd destination supports."""
    _fields_ = [("row0", ctypes.c_int), ("rows", ctypes.c_int), ("Ko", ctypes.c_int), ("Kd", ctypes.c_int)]


def build(verbose: bool = False) -> str:
    """Compile the CUDA library for sm_90a (nvcc cross-compiles without a GPU)."""
    r = subprocess.run(["make", "-C", CSRC, "-j", str(max(1, (os.cpu_count() or 2)))], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout[-4000:])
        print(r.stderr[-4000:])
    if r.returncode != 0:
        raise RuntimeError("building libmpgcn_b200.so failed (see output above)")
    return LIB_PATH


def load() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"mpgcn_b200: CUDA library {LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            f"or `make -C {CSRC}`. There is no CPU / PyTorch fallback for the hot path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    if lib.mpgcn_abi_version() != ABI_VERSION:
        raise RuntimeError("mpgcn_b200: ABI version mismatch between the Python binding and libmpgcn_b200.so")
    _lib = lib
    return lib


# The library's deterministic mode is per host thread (mpgcn_set_deterministic); this is the value last set on each thread, so that a
# thread whose mode already matches makes no call.  A thread starts at 0 in both.
_DET = threading.local()


def set_deterministic(on: bool) -> bool:
    """Set the calling thread's library mode to `on` (one ctypes call only when it changes); -> `on`."""
    on = bool(on)
    if getattr(_DET, "on", False) != on:
        load().mpgcn_set_deterministic(int(on))
        _DET.on = on
    return on


def sync_deterministic() -> bool:
    """Give the calling thread's library mode the value of torch.are_deterministic_algorithms_enabled(); -> that value.
    Every autograd Function calls it in forward AND in backward: autograd runs CUDA backward on its own device thread, where a mode
    set during forward does not hold."""
    import torch
    return set_deterministic(torch.are_deterministic_algorithms_enabled())


class engine_buffers:
    """Context (and decorator) for the engine's own allocations: under torch.use_deterministic_algorithms(True) torch fills every
    torch.empty tensor with NaN (torch.utils.deterministic.fill_uninitialized_memory).  The engine's workspaces, stashes and outputs
    are written in full by its kernels before anything reads them (the stage tests prefill them with NaN and check), so that fill
    is pure memory traffic -- gigabytes per step at N = 1000.  Inside this context it is skipped.  The setting is process-wide:
    another thread allocating meanwhile may skip its fill too, which changes no result."""

    def __enter__(self):
        import torch
        import torch.utils.deterministic as det
        self._prev = torch.are_deterministic_algorithms_enabled() and det.fill_uninitialized_memory
        if self._prev:
            det.fill_uninitialized_memory = False
        return self

    def __exit__(self, *exc):
        if self._prev:
            import torch.utils.deterministic as det
            det.fill_uninitialized_memory = True
        return False

    def __call__(self, fn):
        import functools

        @functools.wraps(fn)
        def wrapped(*args, **kwargs):
            with engine_buffers():
                return fn(*args, **kwargs)
        return wrapped


def check(code: int, what: str) -> None:
    if code != 0:
        msg = load().mpgcn_last_error()
        raise RuntimeError(f"mpgcn_b200.{what} failed: {msg.decode() if msg else 'unknown error'}")


PROFILE_TAGS = ("FWD_A", "FWD_MIX", "FWD_B", "BWD_V", "BWD_DW", "BWD_MIX", "BWD_DX", "SIMT_GEMM", "ELEMENTWISE", "LSTM_FWD", "LSTM_BWD",
                "LAYER_FWD", "LAYER_BWD", "HEAD", "EXCHANGE", "BWD_DG")
REGION_TAGS = ("LAYER_FWD", "LAYER_BWD", "HEAD")      # whole C-ABI calls (their `launches` count calls, not kernels)


def profile_read() -> dict:
    """{tag: {launches, flops, ms}} since the last mpgcn_profile_reset(); synchronise the device first."""
    lib = load()
    out = {}
    for i, name in enumerate(PROFILE_TAGS):
        n, f, ms = ctypes.c_longlong(0), ctypes.c_double(0), ctypes.c_double(0)
        check(lib.mpgcn_profile_read(i, ctypes.byref(n), ctypes.byref(f), ctypes.byref(ms)), "profile_read")
        out[name] = dict(launches=n.value, flops=f.value, ms=ms.value)
    return out
