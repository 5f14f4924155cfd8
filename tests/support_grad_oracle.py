"""Float64 gradient of a BDGCN layer with respect to its supports, in the factored order of the engine's dG stages.

    pre[b,m,e,h] = sum_{o,d} sum_{n,c,l} G_o[n,m] X[b,n,c,l] G_d[c,e] W[o,d,l,h]      dPre = d_out * act'(pre)
    dG_o[n,m] = sum_{b,e,h} U_o[b,n,e,h] dPre[b,m,e,h]     U_o = sum_d Z_d W[o,d],   Z_d[b,n,e,l] = sum_c X[b,n,c,l] G_d[c,e]
    dG_d[c,e] = sum_{b,n,l} X[b,n,c,l] Y_d[b,n,e,l]        Y_d = sum_o V_o W[o,d]^T, V_o[b,n,e,h] = sum_m G_o[n,m] dPre[b,m,e,h]

Static supports (one [K,N,N] stack in both roles) get dG_o + dG_d summed over the batch; dynamic ones ([B,K,N,N] pairs) get
(dG_o, dG_d) per sample.  Written with torch so that it runs on the CPU for the fixture checks and on the GPU (still float64) at
the sizes the GPU tests use.
"""
from __future__ import annotations

import numpy as np
import torch


def _t(a, dev):
    return a.to(device=dev, dtype=torch.float64) if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a, dtype=np.float64)).to(dev)


def support_grads(X, G, W, b, act, d_out, mask_from=None, device="cpu"):
    """X [B,N,N,C], G [K,N,N] or (G_o, G_d) [B,K,N,N], W [K*K*C, H], b [H] or None, act "relu" / "none", d_out [B,N,N,H].
    mask_from: the ReLU mask from this output instead of the float64 pre-activation (the gradient of the function a kernel
    computed).  -> dG [K,N,N] (static) or (dG_o, dG_d) [B,K,N,N], float64 numpy."""
    dynamic = not (isinstance(G, (np.ndarray, torch.Tensor)))
    X, d_out = _t(X, device), _t(d_out, device)
    B, N, _, C = X.shape
    H = d_out.shape[-1]
    if dynamic:
        go, gd = _t(G[0], device), _t(G[1], device)
        K = go.shape[1]
    else:
        go = gd = _t(G, device)
        K = go.shape[0]
    Wk = _t(W, device).reshape(K, K, C, H)
    zs = "bdce" if dynamic else "dce"
    Z = torch.einsum(f"bncl,{zs}->bdnel", X, gd)                         # [B,Kd,N,N,C]
    U = torch.einsum("bdnel,odlh->boneh", Z, Wk)                         # [B,Ko,N,N,H]
    if act == "relu":
        if mask_from is None:
            gs = "bonm" if dynamic else "onm"
            pre = torch.einsum(f"{gs},boneh->bmeh", go, U)
            if b is not None:
                pre = pre + _t(b, device)
            mask = pre > 0
        else:
            mask = _t(mask_from, device) > 0
        dpre = d_out * mask
    else:
        dpre = d_out
    gs = "bonm" if dynamic else "onm"
    V = torch.einsum(f"{gs},bmeh->boneh", go, dpre)                      # [B,Ko,N,N,H]
    Y = torch.einsum("boneh,odlh->bdnel", V, Wk)                         # [B,Kd,N,N,C]
    if dynamic:
        dgo = torch.einsum("boneh,bmeh->bonm", U, dpre)
        dgd = torch.einsum("bncl,bdnel->bdce", X, Y)
        return dgo.cpu().numpy(), dgd.cpu().numpy()
    dg = torch.einsum("boneh,bmeh->onm", U, dpre) + torch.einsum("bncl,bdnel->dce", X, Y)
    return dg.cpu().numpy()
