"""Float64 emulation of the tensor-core LSTM (mpgcn_b200/csrc/lstm_tc.cu, precision 1) with the kernels' own roundings.

Test infrastructure, numpy only.  It reproduces what the kernels round and nothing else:

  * the gate weights `Wx` exactly as `load_wx` builds them: `s_j*W_hh` rounded to fp16, `s_j*w_ih` and `s_j*b`
    (b = b_ih + b_hh, formed in fp32) each split into an fp16 hi part and a separately fp16-rounded lo part, with
    `s_j = -log2 e` for the i, f, o gates and `-2 log2 e` for g;
  * the operand row of a cell as `x_cols` builds it, `[h_{t-1} | x_hi 1 x_lo x_hi 1]`, x saturated at +-65504;
  * `h_{t-1}` rounded to fp16 as the MMA operand.

Everything else (accumulation, the activations, the cell state) is float64, so a kernel differs from this emulation only by its
fp32 arithmetic and the SFU approximations.  Switches drop each lo half (`keep_xlo`, `keep_wlo`, `keep_blo`) so that a test can
measure the part of a kernel's result that each of them contributes, and `exact=True` turns every rounding off (then the
emulation is the plain LSTM of `mpgcn_oracle.lstm_last_forward`).

The backward is "teacher-forced": it takes the saved fp16 `c_t` / `h_t` the training forward wrote (the very bits the forward's
GEMM read, since `pack2` / `pack8` round the same fp32 value) and emulates one reverse-walk step from them: the gates recomputed
from the saved `h_{t-1}`, the power-of-two gradient scale S applied before the fp16 rounding of `da_t` (and at hidden 96 / 128
the division by `s_j`), `dh_{t-1}` from the operands the kernel's dh GEMM reads, and `dWext = sum da_t^T hx_t`.

Decoders map the kernels' buffers to [cell, t, unit] arrays: the saved state (`save_off`, DESIGN.md section 5) and the
gate-gradient records of the wide backward (`[tile][t][cell][4H]`, columns `128 js + 32 gate + u`).
"""
import numpy as np

HALF_MAX = 65504.0
S_IFO = np.float32(-1.4426950408889634)     # s_j of the i, f, o gate rows
S_G = np.float32(-2.8853900817779268)       # s_j of the g gate rows
LN2 = np.float32(0.69314718055994531)
GRAD_SCALE_BYTES = 1024                     # the [S, 1/S] block at the start of the backward workspace


# ------------------------------------------------------------------------------------------------------------------------------
# roundings
# ------------------------------------------------------------------------------------------------------------------------------
def f16(x):
    """fp32 -> fp16 round to nearest even (as __float2half_rn: overflow gives inf), returned as float64 values."""
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float64)


def row_scale(C):
    """s_j of every gate row j (natural order i, f, g, o), float32."""
    s = np.full(4 * C, S_IFO, np.float32)
    s[2 * C:3 * C] = S_G
    return s


def inv_row_scale(C):
    """The 1/s_j the wide walk multiplies da_t by before its fp16 rounding: -ln 2 (i, f, o) and -ln 2 / 2 (g), float32."""
    r = np.full(4 * C, -LN2, np.float32)
    r[2 * C:3 * C] = np.float32(-0.5) * LN2
    return r


def x_split(x, exact=False, keep_xlo=True):
    """x_cols: x_hi = fp16(sat(x)), x_lo = fp16(sat(x - x_hi)) (the difference in fp32).  -> (x_hi, x_lo) float64."""
    x = np.asarray(x, np.float32)
    if exact:
        return x.astype(np.float64), np.zeros(x.shape)
    hi32 = np.clip(x, -HALF_MAX, HALF_MAX).astype(np.float16).astype(np.float32)
    lo = f16(np.clip(x - hi32, -HALF_MAX, HALF_MAX)) if keep_xlo else np.zeros(x.shape)
    return hi32.astype(np.float64), lo


def build_wx(w_ih, w_hh, b_ih, b_hh, exact=False, keep_wlo=True, keep_blo=True):
    """Wx as load_wx builds it, in natural gate-row order -> dict of float64 arrays: whh [4C,C] = fp16(s_j W_hh), wi_hi, wi_lo,
    b_hi, b_lo [4C], and s [4C] (float32 s_j)."""
    w_hh = np.asarray(w_hh, np.float32)
    C = w_hh.shape[1]
    s = row_scale(C)
    w_ih = np.asarray(w_ih, np.float32).reshape(4 * C)
    b = np.asarray(b_ih, np.float32).reshape(4 * C) + np.asarray(b_hh, np.float32).reshape(4 * C)
    if exact:                                                 # s_j in float64 too: the float32 constants are off by ~1e-8
        s64 = np.where(np.arange(4 * C) // C == 2, -2.0, -1.0) * np.log2(np.e)
        z = np.zeros(4 * C)
        b64 = np.asarray(b_ih, np.float64).reshape(4 * C) + np.asarray(b_hh, np.float64).reshape(4 * C)
        return dict(whh=s64[:, None] * w_hh, wi_hi=s64 * w_ih, wi_lo=z, b_hi=s64 * b64, b_lo=z, s=s64)
    wi, bb = s * w_ih, s * b                                  # fp32 products, as the kernel forms them
    wi_hi, b_hi = f16(wi), f16(bb)
    return dict(whh=f16(s[:, None] * w_hh), wi_hi=wi_hi, b_hi=b_hi, s=s,
                wi_lo=f16(wi - wi_hi.astype(np.float32)) if keep_wlo else np.zeros(4 * C),
                b_lo=f16(bb - b_hi.astype(np.float32)) if keep_blo else np.zeros(4 * C))


# ------------------------------------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------------------------------------
def gate_args(h_op, x_hi, x_lo, wx):
    """The accumulator of the gate GEMM, hx_t . Wx^T (the ex2 arguments), and the sum of the absolute values of its terms.
    h_op [S,C] (already the MMA operand), x_hi / x_lo [S] -> ([S,4C], [S,4C])."""
    xh, xl = x_hi[:, None], x_lo[:, None]
    acc = h_op @ wx["whh"].T + xh * wx["wi_hi"] + wx["b_hi"] + xl * wx["wi_hi"] + xh * wx["wi_lo"] + wx["b_lo"]
    mag = (np.abs(h_op) @ np.abs(wx["whh"]).T + np.abs(xh) * (2 * np.abs(wx["wi_hi"]) + np.abs(wx["wi_lo"]))
           + np.abs(xl) * np.abs(wx["wi_hi"]) + np.abs(wx["b_hi"]) + np.abs(wx["b_lo"]))
    return acc, mag


def activations(acc, C):
    """(i, f, g, o) from the ex2 arguments: sigmoid = 1 / (1 + 2^a), tanh = 2 / (1 + 2^a) - 1, a clamped from above at 40."""
    r = 1.0 / (1.0 + np.exp2(np.minimum(acc, 40.0)))
    return r[:, :C], r[:, C:2 * C], 2.0 * r[:, 2 * C:3 * C] - 1.0, r[:, 3 * C:]


def tanh_c(c):
    return 2.0 / (1.0 + np.exp2(np.minimum(-2.0 * np.log2(np.e) * c, 40.0))) - 1.0


def step(c_prev, h_op, x_hi, x_lo, wx):
    """One cell update from the MMA operand h_op = h_{t-1} -> (c_t, h_t, gates (i, f, g, o), |terms| of the gate arguments)."""
    C = c_prev.shape[1]
    acc, mag = gate_args(h_op, x_hi, x_lo, wx)
    i, f, g, o = activations(acc, C)
    c = f * c_prev + i * g
    return c, o * tanh_c(c), (i, f, g, o), mag


def forward(x, w_ih, w_hh, b_ih, b_hh, h_saved=None, exact=False, keep_xlo=True, keep_wlo=True, keep_blo=True):
    """x [S,T] -> dict c, h [S,T,C] (float64, unrounded), f [S,T,C] (forget gate), A [S,T,C] (largest |terms| sum of the four
    gate arguments of a unit).  h_saved [S,T,C]: the kernel's saved fp16 h_t; step t then reads h_saved[:, t-1] as its operand
    (teacher forcing), else the emulation's own h_{t-1} rounded to fp16 (or not rounded when exact)."""
    x = np.asarray(x, np.float32)
    S, T = x.shape
    C = np.asarray(w_hh).shape[1]
    wx = build_wx(w_ih, w_hh, b_ih, b_hh, exact, keep_wlo, keep_blo)
    x_hi, x_lo = x_split(x, exact, keep_xlo)
    c, h = np.zeros((S, C)), np.zeros((S, C))
    out = {k: np.zeros((S, T, C)) for k in ("c", "h", "f", "A")}
    for t in range(T):
        if t == 0:
            h_op = np.zeros((S, C))
        elif h_saved is not None:
            h_op = h_saved[:, t - 1]
        else:
            h_op = h if exact else f16(h)
        c, h, gates, mag = step(c, h_op, x_hi[:, t], x_lo[:, t], wx)
        out["c"][:, t], out["h"][:, t], out["f"][:, t] = c, h, gates[1]
        out["A"][:, t] = mag.reshape(S, 4, C).max(axis=1)
    return out


def forward_error_scale(fwd):
    """Per element of c_t / h_t, the magnitude that the kernel's fp32 arithmetic and SFU approximations are measured in (units of
    2^-22): e_c(t) = f_t e_c(t-1) + 1 + |c_{t-1}| + A_t (an error of c is carried on by the forget gate), e_h = 1 + A_t + e_c."""
    c, f, A = fwd["c"], fwd["f"], fwd["A"]
    e_c, e_h = np.zeros_like(c), np.zeros_like(c)
    prev, c_prev = np.zeros(c.shape[::2]), np.zeros(c.shape[::2])
    for t in range(c.shape[1]):
        prev = f[:, t] * prev + 1.0 + np.abs(c_prev) + A[:, t]
        e_c[:, t], e_h[:, t] = prev, 1.0 + A[:, t] + prev
        c_prev = c[:, t]
    return e_c, e_h


# ------------------------------------------------------------------------------------------------------------------------------
# backward (teacher-forced)
# ------------------------------------------------------------------------------------------------------------------------------
def backward(x, w_ih, w_hh, b_ih, b_hh, d_hT, c_saved, h_saved, S, da_kernel=None, exact=False):
    """One emulated reverse walk from the kernel's saved state.

    x [S_,T]; d_hT [S_,C]; c_saved, h_saved [S_,T,C] the decoded fp16 state; S the power-of-two gradient scale.  At hidden 32
    `da` is fp16(S da_t) and dh_{t-1} = da . fp16(W_hh); at 96 / 128 the kernel keeps da' = fp16(S da_t / s_j) and forms
    dh_{t-1} = da' . fp16(s_j W_hh).  da_kernel [S_,T,4C] (wide widths, natural gate order): the kernel's own da' records; dh and
    dWext are then formed from them, so that every step starts from the kernel's own dh.
    -> dict da (unrounded S da_t, or S da_t / s_j at the wide widths) [S_,T,4C], da_mag (error scale of da, units of 2^-22)
       [S_,T,4C], dx [S_,T], dw_ih, db [4C], dw_hh [4C,C] (un-scaled by 1/S), dw_*_mag (sum of |da16| |hx|)
       and dw_*_sub (the same over the terms with an fp16-subnormal operand)."""
    x = np.asarray(x, np.float32)
    Sc, T = x.shape
    C = np.asarray(w_hh).shape[1]
    wide = C != 32
    wx = build_wx(w_ih, w_hh, b_ih, b_hh, exact)
    x_hi, x_lo = x_split(x, exact)
    w_ih32 = np.asarray(w_ih, np.float32).reshape(4 * C).astype(np.float64)
    inv_s = (1.0 / wx["s"] if exact else inv_row_scale(C).astype(np.float64)) if wide else np.ones(4 * C)
    back = wx["s"].astype(np.float64) if wide else np.ones(4 * C)               # what the weight-gradient pass multiplies back
    w_dh = wx["whh"] if wide else (np.asarray(w_hh, np.float64) if exact else f16(w_hh))
    dh = np.asarray(d_hT, np.float64) * S
    dc = np.zeros((Sc, C))
    run = np.zeros((Sc, C))                  # propagated error scale of dc
    out = dict(da=np.zeros((Sc, T, 4 * C)), da_mag=np.zeros((Sc, T, 4 * C)), dx=np.zeros((Sc, T)))
    dw_hh, dw_hh_mag, dw_hh_sub = np.zeros((4 * C, C)), np.zeros((4 * C, C)), np.zeros((4 * C, C))
    dwi, dwi_mag, dwi_sub, db, db_mag, db_sub = (np.zeros(4 * C) for _ in range(6))
    for t in reversed(range(T)):
        h_op = h_saved[:, t - 1] if t > 0 else np.zeros((Sc, C))
        c_t, c_prev = c_saved[:, t], (c_saved[:, t - 1] if t > 0 else np.zeros((Sc, C)))
        acc, mag = gate_args(h_op, x_hi[:, t], x_lo[:, t], wx)
        gi, gf, gg, go = activations(acc, C)
        tc = tanh_c(c_t)
        dcv = dh * go * (1.0 - tc * tc) + dc
        d_o = dh * tc * go * (1.0 - go)
        di = dcv * gg * gi * (1.0 - gi)
        df = dcv * c_prev * gf * (1.0 - gf)
        dg = dcv * gi * (1.0 - gg * gg)
        dc = dcv * gf
        da = np.concatenate([di, df, dg, d_o], axis=1)
        out["dx"][:, t] = (da @ w_ih32) / S
        run = gf * run + np.abs(dh) + np.abs(dcv)
        A = mag.reshape(Sc, 4, C).max(axis=1)
        m = (np.abs(dh) + run) * (1.0 + np.abs(c_prev)) * (1.0 + A)
        out["da"][:, t] = da * inv_s
        out["da_mag"][:, t] = np.tile(m, 4) * np.abs(inv_s)
        da16 = (da_kernel[:, t] if da_kernel is not None else (da * inv_s if exact else f16(da * inv_s)))
        dh = da16 @ w_dh
        hx_x = x_hi[:, t] + x_lo[:, t]
        a16, ah = np.abs(da16), np.abs(h_op)
        ax = np.abs(x_hi[:, t]) + np.abs(x_lo[:, t])
        sub, sh, sx = (np.where(v < 2.0 ** -14, v, 0.0) for v in (a16, ah, ax))      # fp16 subnormal operands
        dw_hh += back[:, None] * (da16.T @ h_op)
        dw_hh_mag += np.abs(back)[:, None] * (a16.T @ ah)
        dw_hh_sub += np.abs(back)[:, None] * (sub.T @ ah + (a16 - sub).T @ sh)         # terms with a subnormal operand
        dwi += back * (da16.T @ hx_x)
        dwi_mag += np.abs(back) * (a16.T @ ax)
        dwi_sub += np.abs(back) * (sub.T @ ax + (a16 - sub).T @ sx)
        db += back * da16.sum(axis=0)
        db_mag += np.abs(back) * a16.sum(axis=0)
        db_sub += np.abs(back) * sub.sum(axis=0)
    out.update(dw_hh=dw_hh / S, dw_ih=dwi / S, db=db / S, dw_hh_mag=dw_hh_mag / S, dw_ih_mag=dwi_mag / S, db_mag=db_mag / S,
               dw_hh_sub=dw_hh_sub / S, dw_ih_sub=dwi_sub / S, db_sub=db_sub / S)
    return out


def expected_scale(amax):
    """[S, 1/S] of make_scale_kernel: S = 2^k with S * amax in [16, 32), k clamped to [-100, 100]; S = 1 for amax = 0 / inf."""
    if not (0.0 < amax < 3.0e38):
        return 1.0, 1.0
    k = max(-100, min(100, 5 - int(np.frexp(amax)[1])))
    return 2.0 ** k, 2.0 ** -k


# ------------------------------------------------------------------------------------------------------------------------------
# buffer layouts
# ------------------------------------------------------------------------------------------------------------------------------
def dims(H):
    """(CH 32-unit slices, CG 16-cell groups per tile, cells per tile) of the kernel that runs hidden H."""
    CH = H // 32
    CG = {1: 8, 3: 4, 4: 3}[CH]
    return CH, CG, 16 * CG


def tiles(cells, H):
    return -(-cells // dims(H)[2])


def decode_saved(buf, cells, T, H):
    """The training forward's saved state -> (c, h) [cells, T, H] float64.  buf: the fp16 buffer (numpy float16, at least
    tiles * T * CELLS * 2H halves).  Per (tile, step) the warps w = cg CH + js hold [c | h][lane][16 halves]; slot h2 * 8 + s of
    lane l = 4 g + q is cell tile * CELLS + 16 cg + g + 8 h2 and unit 32 js + 8 (s >> 1) + 2 q + (s & 1) (save_off)."""
    CH, CG, CELLS = dims(H)
    nt = tiles(cells, H)
    a = np.asarray(buf)[:nt * T * CELLS * 2 * H].reshape(nt, T, CG, CH, 2, 8, 4, 2, 4, 2)
    #                                                     tile t  cg  js kind g  q  h2 jn e
    a = a.transpose(0, 2, 7, 5, 1, 4, 3, 8, 6, 9).reshape(nt * CELLS, T, 2, H)[:cells].astype(np.float64)
    return a[:, :, 0], a[:, :, 1]


def encode_saved(c, h, H):
    """Inverse of decode_saved (padded cells zero) -> fp16 buffer."""
    CH, CG, CELLS = dims(H)
    cells, T = c.shape[:2]
    nt = tiles(cells, H)
    a = np.zeros((nt * CELLS, T, 2, H), np.float16)
    a[:cells, :, 0], a[:cells, :, 1] = c, h
    a = a.reshape(nt, CG, 2, 8, T, 2, CH, 4, 4, 2)          # tile cg h2 g t kind js jn q e
    return np.ascontiguousarray(a.transpose(0, 4, 1, 6, 5, 3, 8, 2, 7, 9)).reshape(-1)


def decode_da_records(buf, cells, T, H):
    """The wide backward's gate-gradient records [tile][t][cell][4H] (columns 128 js + 32 gate + u, gate row
    gate * H + 32 js + u) -> [tiles * CELLS, T, 4H] float64 in natural gate order, the padded cells of the last tile included.
    buf starts at the records (workspace byte 1024)."""
    CH, _, CELLS = dims(H)
    nt = tiles(cells, H)
    a = np.asarray(buf)[:nt * T * CELLS * 4 * H].reshape(nt, T, CELLS, CH, 4, 32)
    return a.transpose(0, 2, 1, 4, 3, 5).reshape(nt * CELLS, T, 4 * H).astype(np.float64)


def encode_da_records(da, H):
    """Inverse of decode_da_records -> fp16 buffer (padded cells zero)."""
    CH, _, CELLS = dims(H)
    cells, T = da.shape[:2]
    nt = tiles(cells, H)
    a = np.zeros((nt * CELLS, T, 4 * H), np.float16)
    a[:cells] = da
    a = a.reshape(nt, CELLS, T, 4, CH, 32).transpose(0, 2, 1, 4, 3, 5)
    return np.ascontiguousarray(a).reshape(-1)
