"""numpy emulation of the bf16x3 BDGCN layer (precision 2, DESIGN.md section 3), for the tests.

Every tensor-core operand a becomes hi = bf16_rn(a), lo = bf16_rn(a - hi) (round to nearest even, by bit manipulation of the
float32 pattern), each product is hi*hi + hi*lo + lo*hi, accumulated here in float64 (the engine accumulates in fp32 registers, an
error far below the pair's), and every intermediate the engine stores as a pair (Z, U, V, Y) is split again.  The factored order is
the engine's: Z = X x2 G_d, U = mix(Z, W), pre = G_o^T x1 U + b; V = G_o x1 dPre, dW = Z^T V, Y = mix(V, W^T), dX = Y x2 G_d^T."""
from __future__ import annotations

import numpy as np


def bf16_rn(a):
    """float32 -> the nearest bfloat16 (ties to even), returned as float32."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).reshape(np.shape(a))


def split(a):
    """(hi, lo) of the pair of a (first rounded to float32, as the engine reads fp32 tensors)."""
    a = np.asarray(a, dtype=np.float32)
    hi = bf16_rn(a)
    return hi, bf16_rn(a - hi)


def product(spec, a, b):
    """einsum(spec, a, b) as the engine forms it from the pairs of a and b."""
    (ah, al), (bh, bl) = split(a), split(b)
    f = lambda x, y: np.einsum(spec, x.astype(np.float64), y.astype(np.float64), optimize=True)
    return f(ah, bh) + f(ah, bl) + f(al, bh)


def _stacks(G, B):
    if isinstance(G, tuple):
        return G[0], G[1]
    return np.broadcast_to(G, (B,) + G.shape), np.broadcast_to(G, (B,) + G.shape)


def forward(X, G, W, b, relu=True):
    """-> (out, pre, Z); G is [K,N,N] or a pair of [B,K,N,N] (origin, destination)."""
    B, N, _, C = X.shape
    go, gd = _stacks(G, B)
    K, H = go.shape[1], W.shape[1]
    Z = product("bncl,bdce->bdnel", X, gd)                                # X x2 G_d
    U = product("bdnel,odlh->bonhe", Z, W.reshape(K, K, C, H)).transpose(0, 1, 2, 4, 3)   # [b,o,n,e,h]
    pre = product("bonm,bonhe->bmeh", go, U.transpose(0, 1, 2, 4, 3).astype(np.float32))
    if b is not None:
        pre = pre + b
    out = np.maximum(pre, 0.0) if relu else pre
    return out, pre, Z


def backward(X, G, W, b, d_out, relu=True, mask_from=None):
    """-> (out, dX, dW, db); mask_from: the forward output whose sign gives the ReLU mask (default: the emulated one)."""
    B, N, _, C = X.shape
    go, gd = _stacks(G, B)
    K, H = go.shape[1], W.shape[1]
    out, pre, Z = forward(X, G, W, b, relu)
    mask = (mask_from if mask_from is not None else out) > 0 if relu else np.ones_like(out, dtype=bool)
    dP = np.where(mask, d_out, 0.0)
    db = dP.sum(axis=(0, 1, 2))
    V = product("bonm,bmeh->bonhe", go, dP.astype(np.float32))            # [b,o,n,h,e]
    dW = product("bdnel,bonhe->odlh", Z.astype(np.float32), V.astype(np.float32)).reshape(K * K * C, H)
    Y = product("bonhe,odlh->bdnel", V.astype(np.float32), W.reshape(K, K, C, H))
    dX = product("bdce,bdnel->bncl", gd, Y.astype(np.float32))
    return out, dX, dW, db
