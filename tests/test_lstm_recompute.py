"""The recomputing LSTM backward without a device: the C ABI entry points are exported, the workspace query's shape (O(chunk),
not O(B NN T C)), and the refusals before any CUDA call (fake device addresses are never touched)."""
import ctypes

import pytest
import torch

from mpgcn_b200 import _lib, ops

NEW = ("mpgcn_lstm_recompute_bwd_workspace_bytes", "mpgcn_lstm_backward_recompute")
FAKE = ctypes.c_void_p(0x1000)     # never dereferenced: every call below fails its argument checks first
P = _lib.PREC_FP16_TC


def test_new_symbols_are_exported():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name)


@pytest.mark.parametrize("C,L", [(32, 1), (96, 1), (128, 1), (32, 2), (96, 3)])
def test_workspace_is_independent_of_b_and_grows_with_the_chunk(C, L):
    q = _lib.load().mpgcn_lstm_recompute_bwd_workspace_bytes
    T, NN, chunk = 12, 1000 * 1000, 200_000
    sizes = [q(B, T, NN, C, L, chunk, P) for B in (1, 2, 4, 8)]
    assert sizes[0] > 0 and len(set(sizes)) == 1, sizes
    assert all(s % 256 == 0 for s in sizes)
    # far below the stored state it replaces
    assert sizes[-1] < _lib.load().mpgcn_lstm_stack_saved_bytes(8, T, NN, C, L, P) / 10 if L > 1 else \
        sizes[-1] < _lib.load().mpgcn_lstm_saved_bytes(8, T, NN, C, P) / 10
    grow = [q(4, T, NN, C, L, c, P) for c in (400_000, 800_000, 1_600_000)]
    assert sizes[0] < grow[0] < grow[1] < grow[2], grow
    # a chunk is at least one wave of the backward grid: smaller requests give the same size
    assert q(4, T, NN, C, L, 1, P) == q(4, T, NN, C, L, 100, P) > 0
    # and at most every cell
    assert q(1, T, 1000, C, L, 10 ** 15, P) == q(1, T, 1000, C, L, 1000, P) > 0


def test_workspace_query_returns_zero_where_the_call_refuses():
    q = _lib.load().mpgcn_lstm_recompute_bwd_workspace_bytes
    assert q(1, 4, 100, 32, 1, 100, _lib.PREC_FP32) == 0           # precision 0 keeps no state in the first place
    assert q(1, 4, 100, 64, 1, 100, P) == 0                        # no tensor-core kernel at 64
    assert q(1, 4, 100, 128, 2, 100, P) == 0                       # no stacks at 128
    assert q(1, 257, 100, 32, 1, 100, P) == 0
    assert q(1, 4, 100, 32, 0, 100, P) == 0
    assert q(1, 4, 100, 32, 1, 0, P) == 0
    assert q(0, 4, 100, 32, 1, 100, P) == 0


def _err(rc, *needles):
    msg = _lib.load().mpgcn_last_error().decode()
    assert rc != 0 and all(n in msg for n in needles), msg


def test_backward_refuses_bad_arguments():
    lib = _lib.load()
    B, T, NN, C, L, chunk = 2, 5, 100, 32, 2, 64
    need = lib.mpgcn_lstm_recompute_bwd_workspace_bytes(B, T, NN, C, L, chunk, P)
    arr = lambda n=L, p=FAKE: (ctypes.c_void_p * n)(*([p] * n))  # noqa: E731

    def call(**kw):
        a = dict(x=FAKE, L=L, w=arr(), d_hT=FAKE, g=arr(), dx=FAKE, chunk=chunk, ws=FAKE, wsb=need, B=B, T=T, NN=NN, C=C, prec=P)
        a.update(kw)
        n = a["L"]
        w = a["w"] if "w" in kw else arr(max(n, 1))
        g = a["g"] if "g" in kw else arr(max(n, 1))
        return lib.mpgcn_lstm_backward_recompute(a["x"], n, w, w, w, w, a["d_hT"], g, g, g, g, a["dx"], a["chunk"], a["ws"], a["wsb"],
                                                 a["B"], a["T"], a["NN"], a["C"], a["prec"], None, None)

    _err(call(chunk=0), "chunk_cells=0")
    _err(call(chunk=-5), "chunk_cells=-5")
    _err(call(wsb=need - 1), "workspace too small")
    _err(call(ws=None), "workspace too small")
    _err(call(ws=ctypes.c_void_p(0x1010)), "256-byte aligned")
    _err(call(prec=_lib.PREC_FP32), "does not support")
    _err(call(C=128), "does not support")                # stacks stop at hidden 96
    _err(call(C=64, L=1), "does not support")
    _err(call(T=257), "does not support")
    _err(call(L=0), "L=0")
    _err(call(B=0), "empty input")
    _err(call(x=None), "null")
    _err(call(d_hT=None), "null")
    _err(call(w=arr(L, None)), "null")
    _err(call(g=arr(L, None)), "null")


def test_python_refuses_a_bad_recompute_value():
    x = torch.zeros(1, 2, 2, 2, 1)
    for bad in (0, -3, 1.5, "yes"):
        with pytest.raises(ValueError, match="recompute"):
            ops._check_recompute(bad)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.lstm_last(x, *[torch.zeros(s) for s in ((128, 1), (128, 32), (128,), (128,))], recompute=True)
    assert ops.lstm_recompute_chunk_cells(None, 12, 32, 1) == 0 and ops.lstm_recompute_chunk_cells(False, 12, 32, 1) == 0
    assert ops.lstm_recompute_chunk_cells(5000, 12, 32, 1) == 5000
    # True: a chunk whose workspace takes about the state budget
    for C, L in ((32, 1), (96, 1), (128, 1), (96, 2)):
        chunk = ops.lstm_recompute_chunk_cells(True, 12, C, L)
        ws = _lib.load().mpgcn_lstm_recompute_bwd_workspace_bytes(1, 12, 10 ** 8, C, L, chunk, P)
        assert 0.9 * ops.LSTM_RECOMPUTE_BUDGET_BYTES <= ws <= 1.01 * ops.LSTM_RECOMPUTE_BUDGET_BYTES, (C, L, ws)
