"""Sparse static supports without a device: the C ABI entry points are exported and refuse bad arguments before any CUDA call
(fake device addresses are never touched), and the Python refusals that need no GPU."""
import ctypes

import pytest
import torch
from torch import nn

import MPGCN as shim
from mpgcn_b200 import _lib, ops, shard

NEW = ("mpgcn_sparse_supports_bytes", "mpgcn_sparse_supports_build", "mpgcn_bdgcn_forward_sparse", "mpgcn_bdgcn_backward_sparse")
FAKE = ctypes.c_void_p(0x1000)     # never dereferenced: every call below fails its argument checks first


def test_new_symbols_are_exported():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name)


def test_supports_bytes_query():
    lib = _lib.load()
    for K, N, nnz in ((0, 4, 1), (1, 0, 1), (1, 4, -1), (1, 4, 2 ** 31), (-3, 4, 0)):
        assert lib.mpgcn_sparse_supports_bytes(K, N, nnz) == 0, (K, N, nnz)
    a, b = lib.mpgcn_sparse_supports_bytes(3, 100, 0), lib.mpgcn_sparse_supports_bytes(3, 100, 700)
    assert 0 < a < b and a % 256 == 0 and b % 256 == 0
    assert b - a >= 700 * 4 * 6            # CSR + CSC indices and values, the build's key / entry pairs
    assert lib.mpgcn_sparse_supports_bytes(1, 1, 2 ** 31 - 1) > 0


def _err(rc, *needles):
    msg = _lib.load().mpgcn_last_error().decode()
    assert rc != 0 and all(n in msg for n in needles), msg


def test_build_refuses_bad_arguments():
    lib = _lib.load()
    need = lib.mpgcn_sparse_supports_bytes(2, 10, 5)
    _err(lib.mpgcn_sparse_supports_build(FAKE, FAKE, 2 ** 31, 2, 10, FAKE, 2 ** 40, None), "nnz", "2^31")
    _err(lib.mpgcn_sparse_supports_build(FAKE, FAKE, 5, 0, 10, FAKE, need, None), "K=0")
    _err(lib.mpgcn_sparse_supports_build(FAKE, FAKE, 5, 2, 0, FAKE, need, None), "N=0")
    _err(lib.mpgcn_sparse_supports_build(FAKE, FAKE, -1, 2, 10, FAKE, need, None), "nnz=-1")
    _err(lib.mpgcn_sparse_supports_build(None, FAKE, 5, 2, 10, FAKE, need, None), "null")
    _err(lib.mpgcn_sparse_supports_build(FAKE, None, 5, 2, 10, FAKE, need, None), "null")
    _err(lib.mpgcn_sparse_supports_build(FAKE, FAKE, 5, 2, 10, None, need, None), "null")
    _err(lib.mpgcn_sparse_supports_build(FAKE, FAKE, 5, 2, 10, FAKE, need - 1, None), "too small")


def test_layer_calls_refuse_bad_arguments():
    lib = _lib.load()
    B, N, K, C, H, nnz = 2, 10, 3, 5, 7, 40
    sb = lib.mpgcn_sparse_supports_bytes(K, N, nnz)
    fw = lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, C, H, 0, 0)
    bw = lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, 0, 0)
    fwd = lambda **kw: lib.mpgcn_bdgcn_forward_sparse(*[kw.get(k, v) for k, v in (
        ("X", FAKE), ("sp", FAKE), ("sb", sb), ("nnz", nnz), ("W", FAKE), ("bias", None), ("act", 1), ("out", FAKE), ("saved", FAKE),
        ("ws", FAKE), ("wsb", fw), ("B", B), ("N", N), ("K", K), ("C", C), ("H", H), ("st", None))])
    bwd = lambda **kw: lib.mpgcn_bdgcn_backward_sparse(*[kw.get(k, v) for k, v in (
        ("d_out", FAKE), ("out", FAKE), ("sp", FAKE), ("sb", sb), ("nnz", nnz), ("W", FAKE), ("act", 1), ("saved", FAKE), ("dX", FAKE),
        ("dW", FAKE), ("db", FAKE), ("ws", FAKE), ("wsb", bw), ("B", B), ("N", N), ("K", K), ("C", C), ("H", H), ("st", None))])
    for call, ws_name in ((fwd, "wsb"), (bwd, "wsb")):
        _err(call(K=0), "bad BDGCN shape")
        _err(call(N=0), "bad BDGCN shape")
        _err(call(C=0), "bad BDGCN shape")
        _err(call(B=0), "bad BDGCN shape")
        _err(call(act=2), "activation")
        _err(call(nnz=-1), "bad support stack")
        _err(call(nnz=2 ** 31), "bad support stack")
        _err(call(sp=None), "null")
        _err(call(W=None), "null")
        _err(call(ws=None), "null")
        _err(call(sb=sb - 1), "support buffer too small")
        _err(call(**{ws_name: 100}), "workspace too small")
    _err(fwd(X=None), "null")
    _err(fwd(out=None), "null")
    _err(bwd(d_out=None), "null")
    _err(bwd(out=None), "null")
    _err(bwd(saved=None), "null")
    _err(bwd(dW=None), "null")


def test_python_refusals_need_no_device():
    N, K, C, H = 6, 2, 3, 4
    X = torch.randn(1, N, N, C)
    W = torch.randn(K * K * C, H)
    G = torch.rand(K, N, N)
    Gs = G.to_sparse()
    with pytest.raises(NotImplementedError, match="dynamic pair"):
        ops.bdgcn(X, (Gs.unsqueeze(0), G.unsqueeze(0)), W, None, True)
    with pytest.raises(NotImplementedError, match="dynamic pair"):
        ops.bdgcn(X, (G.unsqueeze(0), Gs.unsqueeze(0)), W, None, True)
    for sg in (False, True):
        with pytest.raises(NotImplementedError, match="no gradient"):
            ops.bdgcn(X, Gs.clone().requires_grad_(True), W, None, True, support_grad=sg)
    with pytest.raises(NotImplementedError, match="COO"):
        ops.bdgcn(X, G.to_sparse_csr(), W, None, True)
    with pytest.raises(NotImplementedError, match="COO"):
        ops.bdgcn(X, G.to_sparse_bsr((1, 1)), W, None, True)
    with pytest.raises(ValueError, match="dense"):
        ops.bdgcn(X, G.unsqueeze(-1).to_sparse(3), W, None, True)
    with pytest.raises(ValueError, match="floating"):
        ops.bdgcn(X, (G > 0.5).to(torch.int64).to_sparse(), W, None, True)
    with pytest.raises(RuntimeError, match="no fp16 sparse kernels"):
        ops.bdgcn(X, Gs, W, None, True, precision="fp16")
    with pytest.raises(ValueError, match="unknown precision"):
        ops.bdgcn(X, Gs, W, None, True, precision="bf16")
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.bdgcn(X, Gs, W, None, True)
    layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=H, activation=nn.ReLU)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        layer(X, Gs)                               # the module's shape assertions accept a sparse stack
    with pytest.raises(NotImplementedError, match="sharded layers take dense supports"):
        shard.sharded_bdgcn(layer, X, Gs, plan=None)


def test_fp16_default_precision_is_refused_for_sparse(monkeypatch):
    monkeypatch.setenv("MPGCN_B200_PRECISION", "fp16")
    G = torch.rand(1, 4, 4).to_sparse()
    with pytest.raises(RuntimeError, match="no fp16 sparse kernels"):
        ops.bdgcn(torch.randn(1, 4, 4, 2), G, torch.randn(2, 3), None, False)
