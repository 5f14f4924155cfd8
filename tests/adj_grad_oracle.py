"""Float64 adjoint of the support-matrix builder: dL/dflow of `Adj_Processor(kernel_type, K).process(flow)` from dL/dsupports.

Per batch element A = flow[b], G_k = dL/dT_k (oracle.mpgcn_oracle.adj_process gives the forward):

    series adjoint (T_0 = I, T_1 = x, T_k = 2 x T_{k-1} - T_{k-2}), k = K .. 2:
        gx += 2 G_k T_{k-1}^T,   G_{k-1} += 2 x^T G_k,   G_{k-2} -= G_k;     then gx += G_1 (G_0 belongs to the identity)
    random walk    x_ij = A_ji dinv_j:  dA_ji += gx_ij dinv_j,  dA_j. += -dinv_j^2 sum_i gx_ij A_ji
    dual, backward series x_ij = A_ij cinv_j:  dA_ij += gx_ij cinv_j,  dA_.j += -cinv_j^2 sum_i gx_ij A_ij
    chebyshev / localpool  An = D A D, d = r^-1/2, gAn = -gx / d_supports[0]:
        dA_ij = d_i d_j gAn_ij + gr_i,  gr_i = -1/2 r_i^-3/2 (sum_j gAn_ij A_ij d_j + sum_j gAn_ji d_j A_ji)

dinv / cinv are 0 where 1/sum is inf, so a masked row (column) contributes exactly 0; the reference's autograd gives NaN there.
`series` restricts the gradient to one series' contribution ("forward" / "backward"; the symmetric kernels have one).
"""
from __future__ import annotations

import numpy as np

from oracle.mpgcn_oracle import _cheb_series, _rw_normalize, _sym_normalize, adj_process  # noqa: F401  (adj_process re-exported)


def _masked_inv(s):
    with np.errstate(divide="ignore"):
        v = 1.0 / s
    return np.where(np.isinf(v), 0.0, v)


def _series_adjoint(x, G):
    """x [N,N], G: list of K+1 upstream gradients of T_0..T_K -> dL/dx."""
    K = len(G) - 1
    if K == 0:
        return np.zeros_like(x)
    T = _cheb_series(x, K)
    G = [g.copy() for g in G]
    gx = np.zeros_like(x)
    for k in range(K, 1, -1):
        gx += 2 * G[k] @ T[k - 1].T
        G[k - 1] += 2 * x.T @ G[k]
        G[k - 2] -= G[k]
    return gx + G[1]


def _rw_rows(A, gx):
    dinv = _masked_inv(A.sum(axis=1))
    return gx.T * dinv[:, None] - (dinv ** 2 * (gx.T * A).sum(axis=1))[:, None]


def _rw_cols(A, gx):
    cinv = _masked_inv(A.sum(axis=0))
    return gx * cinv[None, :] - (cinv ** 2 * (gx * A).sum(axis=0))[None, :]


def _sym(A, gAn):
    r = A.sum(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.power(r, -0.5)
        gr = -0.5 * np.power(r, -1.5) * ((gAn * A * d[None, :]).sum(axis=1) + (gAn * A * d[:, None]).sum(axis=0))
        return d[:, None] * d[None, :] * gAn + gr[:, None]


def adj_process_grad(flow, d_supports, kernel_type, K, series=None):
    """flow [B,N,N], d_supports [B,Ks,N,N] -> dL/dflow [B,N,N], float64."""
    flow = np.asarray(flow, dtype=np.float64)
    d_supports = np.asarray(d_supports, dtype=np.float64)
    if kernel_type == "localpool":
        K = 1
    out = []
    for A, dS in zip(flow, d_supports):
        if kernel_type == "localpool":
            out.append(_sym(A, dS[0]))
        elif kernel_type == "chebyshev":
            x = (2 / 2) * (np.eye(A.shape[0]) - _sym_normalize(A)) - np.eye(A.shape[0])
            out.append(_sym(A, -_series_adjoint(x, list(dS[:K + 1]))))
        elif kernel_type in ("random_walk_diffusion", "dual_random_walk_diffusion"):
            g = np.zeros_like(A)
            if series in (None, "forward"):
                g += _rw_rows(A, _series_adjoint(_rw_normalize(A).T, list(dS[:K + 1])))
            if kernel_type == "dual_random_walk_diffusion" and series in (None, "backward"):
                g += _rw_cols(A, _series_adjoint(_rw_normalize(A.T).T, [dS[0]] + list(dS[K + 1:2 * K + 1])))
            out.append(g)
        else:
            raise ValueError("Invalid kernel_type. Must be one of [chebyshev, localpool, random_walk_diffusion, dual_random_walk_diffusion].")
    return np.stack(out, axis=0)
