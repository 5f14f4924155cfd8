"""Float64 oracle and rounding emulation of the stacked per-cell LSTM (nn.LSTM(1, C, L), last hidden state of the top layer),
built on oracle/mpgcn_oracle.py (the float64 single-layer LSTM and the model) and oracle/lstm_tc_oracle.py (the kernels'
roundings), which it extends without changing.

Float64:
    lstm_stack_forward(x, layers)          -> h_T of the top layer [S, C]
    lstm_stack_backward(x, layers, d_hT)   -> (dx, [(dw_ih, dw_hh, db_ih, db_hh) per layer])
    mpgcn_forward_backward(params, ...)    -> mpgcn_oracle.mpgcn_forward_backward with temporal.*_l{l} of every layer

Emulation of the stack kernels (mpgcn_b200/csrc/lstm_tc.cu; every layer on the width-generic kernels, hidden 32 included):
    forward_up(h_in, ...)                  a layer above the first, driven by the kernel's saved fp16 h of the layer below
    walk(...)                              one layer's reverse walk, teacher-forced by the kernel's saved state and da records
    decode_dseq(buf, cells, T, H)          the fp32 gradient sequence d(h^{l-1}_t) between the walks (dseq_off)

layers: [(w_ih, w_hh, b_ih, b_hh)] from the bottom layer up; x [S, T, I].
"""
from __future__ import annotations

from unittest import mock

import numpy as np

from oracle import lstm_tc_oracle as emu
from oracle import mpgcn_oracle as orc


_lstm_last_forward = orc.lstm_last_forward       # (mpgcn_forward_backward substitutes the module's name while the model runs)


def _layer_forward(seq, w):
    """one layer over seq [S,T,I] -> (its h sequence [S,T,C], the single-layer oracle's cache)"""
    h, cache = _lstm_last_forward(seq, *w, return_cache=True)
    T = seq.shape[1]
    return np.stack([cache[t][0] for t in range(1, T)] + [h], axis=1), cache


def lstm_stack_forward(x, layers, return_seqs=False):
    seqs = [x]
    for w in layers:
        seqs.append(_layer_forward(seqs[-1], w)[0])
    return (seqs[-1][:, -1], seqs) if return_seqs else seqs[-1][:, -1]


def _layer_backward(seq, w, cache, d_hseq):
    """BPTT of one layer given dL/dh_t of every step (d_hseq [S,T,C]) -> (d_seq [S,T,I], dw_ih, dw_hh, db)"""
    w_ih, w_hh = w[0], w[1]
    S, T, _ = seq.shape
    C = w_hh.shape[1]
    dh = np.zeros((S, C))
    dc = np.zeros((S, C))
    d_in = np.zeros_like(seq)
    dw_ih, dw_hh, db = np.zeros_like(w_ih), np.zeros_like(w_hh), np.zeros_like(w[2])
    for t in reversed(range(T)):
        h_prev, c_prev, i, f, g, o, tc = cache[t]
        dh = dh + d_hseq[:, t]
        do = dh * tc
        dc = dc + dh * o * (1 - tc * tc)
        da = np.concatenate([dc * g * i * (1 - i), dc * c_prev * f * (1 - f), dc * i * (1 - g * g), do * o * (1 - o)], axis=1)
        dw_ih += da.T @ seq[:, t, :]
        dw_hh += da.T @ h_prev
        db += da.sum(axis=0)
        d_in[:, t, :] = da @ w_ih
        dh = da @ w_hh
        dc = dc * f
    return d_in, dw_ih, dw_hh, db


def lstm_stack_backward(x, layers, d_hT):
    seqs, caches = [x], []
    for w in layers:
        s, c = _layer_forward(seqs[-1], w)
        seqs.append(s)
        caches.append(c)
    d_hseq = np.zeros_like(seqs[-1])
    d_hseq[:, -1] = d_hT
    grads = [None] * len(layers)
    for l in reversed(range(len(layers))):
        d_hseq, dwi, dwh, db = _layer_backward(seqs[l], layers[l], caches[l], d_hseq)
        grads[l] = (dwi, dwh, db, db.copy())
    return d_hseq, grads


def temporal_layers(params, prefix, L):
    return [tuple(np.asarray(params[f"{prefix}temporal.{k}_l{l}"], dtype=np.float64) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
            for l in range(L)]


def mpgcn_forward_backward(params, x_seq, G_list, M, gcn_num_layers, L, d_y, act="relu", masks=None):
    """mpgcn_oracle.mpgcn_forward_backward (reference MPGCN.py:89-112) with an L-layer LSTM in every branch: the model oracle
    runs as it is, with its single-layer LSTM calls answered by the stack of the branch whose weight_ih_l0 they pass; the
    gradients of the layers above the first are added under their temporal.*_l{l} keys."""
    p64 = {k: np.asarray(v, np.float64) for k, v in params.items()}
    stacks = {id(p64[f"branch_models.{m}.temporal.weight_ih_l0"]): (m, temporal_layers(p64, f"branch_models.{m}.", L)) for m in range(M)}
    upper = {}

    def forward(x, w_ih, *_):
        return lstm_stack_forward(x, stacks[id(w_ih)][1])

    def backward(x, w_ih, w_hh, b_ih, b_hh, d_hT):
        m, layers = stacks[id(w_ih)]
        dx, grads = lstm_stack_backward(x, layers, d_hT)
        upper[m] = grads[1:]
        return (dx, *grads[0])

    with mock.patch.object(orc, "lstm_last_forward", forward), mock.patch.object(orc, "lstm_last_backward", backward):
        y, grads = orc.mpgcn_forward_backward(p64, np.asarray(x_seq, np.float64), G_list, M, gcn_num_layers, np.asarray(d_y, np.float64),
                                              act=act, masks=masks)
    for m, rest in upper.items():
        for l, g in enumerate(rest, start=1):
            for k, v in zip(("weight_ih", "weight_hh", "bias_ih", "bias_hh"), g):
                grads[f"branch_models.{m}.temporal.{k}_l{l}"] = v
    return y, grads


# ------------------------------------------------------------------------------------------------------------------------------
# emulation of the stack kernels' roundings
# ------------------------------------------------------------------------------------------------------------------------------
def build_wx_up(w_ih, w_hh, b_ih, b_hh):
    """Wx of a layer above the first as load_wx<CH, UP> builds it, natural gate-row order: whh = fp16(s_j W_hh), wih =
    fp16(s_j W_ih) (a single fp16, like W_hh), b = s_j (b_ih + b_hh) formed in fp32 and split into b_hi = fp16(b) and
    b_lo = fp16(b - b_hi) (the difference in fp32) against the operand columns 1, 1 -> dict of float64 arrays, s float32."""
    w_hh = np.asarray(w_hh, np.float32)
    C = w_hh.shape[1]
    s = emu.row_scale(C)
    b = s * (np.asarray(b_ih, np.float32).reshape(4 * C) + np.asarray(b_hh, np.float32).reshape(4 * C))
    b_hi = emu.f16(b)
    return dict(whh=emu.f16(s[:, None] * w_hh), wih=emu.f16(s[:, None] * np.asarray(w_ih, np.float32)), b_hi=b_hi,
                b_lo=emu.f16(b - b_hi.astype(np.float32)), s=s)


def gate_args_up(h_op, hin_op, wx):
    """hx_t . Wx^T of an upper layer and the sum of the |terms| -> ([S,4C], [S,4C])"""
    acc = h_op @ wx["whh"].T + hin_op @ wx["wih"].T + wx["b_hi"] + wx["b_lo"]
    mag = np.abs(h_op) @ np.abs(wx["whh"]).T + np.abs(hin_op) @ np.abs(wx["wih"]).T + np.abs(wx["b_hi"]) + np.abs(wx["b_lo"])
    return acc, mag


def forward_up(h_in, w_ih, w_hh, b_ih, b_hh, h_saved=None):
    """A layer above the first: h_in [S,T,C] the kernel's saved fp16 h_t of the layer below (the operand its gate GEMM reads);
    h_saved: this layer's saved h, whose h_{t-1} then is the operand (teacher forcing) -> dict c, h, f, A as
    lstm_tc_oracle.forward (so forward_error_scale applies)."""
    S, T, C = h_in.shape
    wx = build_wx_up(w_ih, w_hh, b_ih, b_hh)
    c, h = np.zeros((S, C)), np.zeros((S, C))
    out = {k: np.zeros((S, T, C)) for k in ("c", "h", "f", "A")}
    for t in range(T):
        h_op = np.zeros((S, C)) if t == 0 else (h_saved[:, t - 1] if h_saved is not None else emu.f16(h))
        acc, mag = gate_args_up(h_op, h_in[:, t], wx)
        i, f, g, o = emu.activations(acc, C)
        c = f * c + i * g
        h = o * emu.tanh_c(c)
        out["c"][:, t], out["h"][:, t], out["f"][:, t] = c, h, f
        out["A"][:, t] = mag.reshape(S, 4, C).max(axis=1)
    return out


def walk(w_ih, w_hh, b_ih, b_hh, c_saved, h_saved, S, da_kernel, x=None, h_in=None, d_hT=None, dh_in=None):
    """One layer's reverse walk in a stack (the width-generic walk at every width), teacher-forced: gates recomputed from the
    kernel's saved h_{t-1} and input (x [S_,T] for the first layer, h_in [S_,T,C] the lower layer's saved h above it); each
    step's dh, dh_{t-1} and d(h^{l-1}_t) formed from the kernel's own da' records da_kernel [S_,T,4C] (natural gate order).
    dh seeds: S d_hT (top layer) and, below the top, dh_in [S_,T,C] (the fp32 d(h_t) the layer above handed down, in units of S)
    added at each step.
    -> dict da (S da_t / s_j, unrounded) and da_mag [S_,T,4C] (as lstm_tc_oracle.backward); d_in [S_,T,C] (= da' . fp16(s W_ih),
       units of S) and d_in_mag (sum of |terms|) above the first layer; dx [S_,T] for the first; dw_ih, dw_hh, db un-scaled by
       1/S with their *_mag and *_sub (terms with an fp16-subnormal operand)."""
    Sc, T, C = c_saved.shape
    up = h_in is not None
    if up:
        wx = build_wx_up(w_ih, w_hh, b_ih, b_hh)
    else:
        wx = emu.build_wx(w_ih, w_hh, b_ih, b_hh)
        x_hi, x_lo = emu.x_split(np.asarray(x, np.float32))
        w_ih32 = np.asarray(w_ih, np.float32).reshape(4 * C).astype(np.float64)
    inv_s, back = emu.inv_row_scale(C).astype(np.float64), wx["s"].astype(np.float64)
    dh = np.zeros((Sc, C)) if d_hT is None else np.asarray(d_hT, np.float64) * S
    dc, run = np.zeros((Sc, C)), np.zeros((Sc, C))
    out = dict(da=np.zeros((Sc, T, 4 * C)), da_mag=np.zeros((Sc, T, 4 * C)))
    if up:
        out.update(d_in=np.zeros((Sc, T, C)), d_in_mag=np.zeros((Sc, T, C)))
    else:
        out["dx"] = np.zeros((Sc, T))
    wi_shape = (4 * C, C) if up else (4 * C,)
    acc_ = {k: np.zeros(wi_shape if k.startswith("dw_ih") else (4 * C, C) if k.startswith("dw_hh") else 4 * C)
            for k in ("dw_hh", "dw_hh_mag", "dw_hh_sub", "dw_ih", "dw_ih_mag", "dw_ih_sub", "db", "db_mag", "db_sub")}
    sub_ = lambda v: np.where(v < 2.0 ** -14, v, 0.0)  # noqa: E731   fp16 subnormal operands
    for t in reversed(range(T)):
        if dh_in is not None:
            dh = dh + dh_in[:, t]
        h_op = h_saved[:, t - 1] if t > 0 else np.zeros((Sc, C))
        c_t, c_prev = c_saved[:, t], (c_saved[:, t - 1] if t > 0 else np.zeros((Sc, C)))
        acc, mag = gate_args_up(h_op, h_in[:, t], wx) if up else emu.gate_args(h_op, x_hi[:, t], x_lo[:, t], wx)
        gi, gf, gg, go = emu.activations(acc, C)
        tc = emu.tanh_c(c_t)
        dcv = dh * go * (1.0 - tc * tc) + dc
        da = np.concatenate([dcv * gg * gi * (1.0 - gi), dcv * c_prev * gf * (1.0 - gf), dcv * gi * (1.0 - gg * gg),
                             dh * tc * go * (1.0 - go)], axis=1)
        dc = dcv * gf
        run = gf * run + np.abs(dh) + np.abs(dcv)
        m = (np.abs(dh) + run) * (1.0 + np.abs(c_prev)) * (1.0 + mag.reshape(Sc, 4, C).max(axis=1))
        out["da"][:, t], out["da_mag"][:, t] = da * inv_s, np.tile(m, 4) * np.abs(inv_s)
        da16 = da_kernel[:, t]
        a16 = np.abs(da16)
        if up:
            out["d_in"][:, t], out["d_in_mag"][:, t] = da16 @ wx["wih"], a16 @ np.abs(wx["wih"])
            op_i, a_i = h_in[:, t], np.abs(h_in[:, t])
            acc_["dw_ih"] += back[:, None] * (da16.T @ op_i)
            acc_["dw_ih_mag"] += np.abs(back)[:, None] * (a16.T @ a_i)
            acc_["dw_ih_sub"] += np.abs(back)[:, None] * (sub_(a16).T @ a_i + (a16 - sub_(a16)).T @ sub_(a_i))
        else:
            out["dx"][:, t] = (da @ w_ih32) / S
            hx_x, ax = x_hi[:, t] + x_lo[:, t], np.abs(x_hi[:, t]) + np.abs(x_lo[:, t])
            acc_["dw_ih"] += back * (da16.T @ hx_x)
            acc_["dw_ih_mag"] += np.abs(back) * (a16.T @ ax)
            acc_["dw_ih_sub"] += np.abs(back) * (sub_(a16).T @ ax + (a16 - sub_(a16)).T @ sub_(ax))
        ah = np.abs(h_op)
        acc_["dw_hh"] += back[:, None] * (da16.T @ h_op)
        acc_["dw_hh_mag"] += np.abs(back)[:, None] * (a16.T @ ah)
        acc_["dw_hh_sub"] += np.abs(back)[:, None] * (sub_(a16).T @ ah + (a16 - sub_(a16)).T @ sub_(ah))
        acc_["db"] += back * da16.sum(axis=0)
        acc_["db_mag"] += np.abs(back) * a16.sum(axis=0)
        acc_["db_sub"] += np.abs(back) * sub_(a16).sum(axis=0)
        dh = da16 @ wx["whh"]
    out.update({k: v / S for k, v in acc_.items()})
    return out


def decode_dseq(buf, cells, T, H):
    """The fp32 gradient sequence of the stack backward (dseq_off: per (tile, step) and warp w = cg CH + js, [lane][16 floats],
    slot h2 * 8 + s of lane l = 4 g + q being cell 16 cg + g + 8 h2 and unit 32 js + 8 (s >> 1) + 2 q + (s & 1))
    -> [cells, T, H] float64.  buf: numpy float32 from workspace byte 1024."""
    CH, CG, CELLS = emu.dims(H)
    nt = emu.tiles(cells, H)
    a = np.asarray(buf)[:nt * T * CELLS * H].reshape(nt, T, CG, CH, 8, 4, 2, 4, 2)
    #                                                 tile t  cg  js g  q  h2 jn e
    return a.transpose(0, 2, 6, 4, 1, 3, 7, 5, 8).reshape(nt * CELLS, T, H)[:cells].astype(np.float64)


def encode_dseq(d, H):
    """Inverse of decode_dseq (padded cells zero) -> float32 buffer."""
    CH, CG, CELLS = emu.dims(H)
    cells, T = d.shape[:2]
    nt = emu.tiles(cells, H)
    a = np.zeros((nt * CELLS, T, H), np.float32)
    a[:cells] = d
    a = a.reshape(nt, CG, 2, 8, T, CH, 4, 4, 2)              # tile cg h2 g t js jn q e
    return np.ascontiguousarray(a.transpose(0, 4, 1, 5, 3, 7, 2, 6, 8)).reshape(-1)
