"""Both LSTM kernel families checked below the end-to-end bars of 1e-3 (h_T) and 2e-3 (gradients).

fp32 CUDA-core kernels (precision 0, lstm_kernels.cu)
  Forward and backward through the C ABI against the float64 oracle at every hidden width class the kernels distinguish (forward
  tiles of 256 / C cells capped at 32, thread counts that are not multiples of 32, the backward's cell count) and every sequence
  length the backward accepts, up to T_max(C): the backward keeps the recomputed sequence of its cells in shared memory, so T is
  bounded per width (8041 steps at hidden 1, 15 at 64).  `mpgcn_lstm_precision_supported(T, C, 0)` must say 1 exactly where both
  kernels run.

Tensor-core kernels (precision 1, lstm_tc.cu; hidden 32, 96, 128)
  One training forward and one backward run through the C ABI into NaN-prefilled buffers; the saved state (fp16 c_t, h_t of
  every step) and, at 96 / 128, the fp16 gate-gradient records are read back and decoded (oracle/lstm_tc_oracle.py), and every
  stage is compared with a float64 emulation of the kernels' own roundings driven by the kernel's own saved h_{t-1}:

    saved c_t, h_t (fp16):  |y - r| <= 2^-11 |r| + 2^-25 + EPS_LSTM * 2^-22 * e      (fp16 store, subnormal floor)
    h_T (fp32):             |y - r| <=                     EPS_LSTM * 2^-22 * e
    da records (fp16):      the same as c_t with the backward's error scale
    dW from the records:    |y - r| <= EPS_LSTM * 2^-24 * sqrt(L) * sum |da||hx|      (L = cells * T terms)
                                       + 2^-12 * (the part of that sum with an fp16-subnormal operand, SUBNORMAL_REL)

  e is the error scale of emulate.forward_error_scale / backward: the SFU approximations (2 ulp each) and fp32 accumulation,
  carried along the cell state.  The largest coefficient measured on an H100 is written to parity_report.json ("lstm stages ...
  coef"); EPS_LSTM = 8 leaves room above it (DESIGN.md section 4).  At hidden 32 the gate gradients never leave registers, so
  the weight gradients and dx are held in rel_L2 to the emulation's own backward from the saved state.
  The fp16 lo halves of x, s_j w_ih and s_j b change h_T by less than 1e-3, so each is checked as the regression slope of the
  kernel's deviation from the emulation without that half on the term the half contributes: 1 within SLOPE_BAND.

The CPU tests show that the emulation is the plain LSTM when its roundings are off, that the decoders invert the kernels'
layouts, and that the helpers accept a simulated faithful kernel and reject each defect they are meant to find.
"""
import math

import numpy as np
import pytest
import torch
from torch import nn

from conftest import record_parity
from oracle import lstm_tc_oracle as emu
from oracle import mpgcn_oracle as orc

import MPGCN as shim
from mpgcn_b200 import _lib, ops

# fp32 CUDA-core kernels against float64 (the tolerances of tests/golden/lstm_* fixtures)
FP32_H_TOL, FP32_G_TOL = 1e-4, 2e-4
FP32_WIDTHS = (1, 3, 8, 16, 17, 31, 33, 48, 63, 64)
SMEM_BUDGET = 220 * 1024          # lstm_kernels.cu kBwdSmemBudget

# tensor-core kernels
EPS_LSTM = 8.0
SLOPE_BAND = (0.9, 1.1)
SLOPE_MIN_TERMS = 100000
# the tensor cores do not keep full precision in products with a subnormal fp16 operand: on an H100 a weight-gradient element
# made of such terms (tiny h_{t-1} of saturated output gates) came out 2^-15.6 (relative) off its float64 value; such an operand
# carries at most 10 significant bits into the MMA anyway, so those terms are allowed 2^-12 of their magnitude
SUBNORMAL_REL = 2.0 ** -12
GRAD32_L2_TOL = 1e-4              # hidden 32 weight gradients and every dx: rel_L2 against the emulated walk
TC_TILE = {32: 128, 96: 64, 128: 48}
TC_WIDTHS = (32, 96, 128)


def fp32_t_max(C):
    """Longest sequence the fp32 backward holds for hidden C: weights + gradient accumulators (12 C^2 + 16 C floats) and per cell
    T (6C + 1) + 5C floats must fit in 220 KB."""
    if not 1 <= C <= 64:
        return 0
    free = (SMEM_BUDGET - (12 * C * C + 16 * C) * 4) // 4
    return max(0, (free - 5 * C) // (6 * C + 1))


def _rel_check(a, ref, tol, what, l2_only=False):
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol), f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"


# ------------------------------------------------------------------------------------------------------------------------------
# checking helpers (numpy; also fed simulated kernels by the CPU tests)
# ------------------------------------------------------------------------------------------------------------------------------
def store_coef(y, r, scale, fp16_store):
    """Largest excess of |y - r| over the fp16 store allowance, in units of 2^-22 * scale (NaN -> inf)."""
    y, r = np.asarray(y, np.float64), np.asarray(r, np.float64)
    ex = np.abs(y - r)
    if fp16_store:
        ex = ex - (2.0 ** -11 * np.abs(r) + 2.0 ** -25)
    ex = np.nan_to_num(ex, nan=math.inf)
    c = np.where(ex <= 0, 0.0, ex / (2.0 ** -22 * np.maximum(scale, 1e-300)))
    return float(c.max()) if c.size else 0.0


def forward_coefs(c_k, h_k, hT_k, fwd):
    """Saved c_t, h_t (fp16) and h_T (fp32) of a kernel against the emulation it drove -> {stage: coef}."""
    e_c, e_h = emu.forward_error_scale(fwd)
    return {"c_t": store_coef(c_k, fwd["c"], e_c, True), "h_t": store_coef(h_k, fwd["h"], e_h, True),
            "h_T": store_coef(hT_k, fwd["h"][:, -1], e_h[:, -1], False)}


def dw_coef(y, r, mag, sub, L):
    """fp32-accumulated sum of L terms: |y - r| in units of 2^-24 sqrt(L) sum|terms|, after SUBNORMAL_REL of the terms with an
    fp16-subnormal operand (sub: the sum of those |terms|)."""
    ex = np.nan_to_num(np.abs(np.asarray(y, np.float64) - r), nan=math.inf) - SUBNORMAL_REL * sub
    return float(np.where(ex <= 0, 0.0, ex / (2.0 ** -24 * math.sqrt(max(L, 1)) * np.maximum(mag, 1e-300))).max())


def slope(dev, term):
    """Least-squares slope through the origin of a deviation on the term it should contain -> (slope, nonzero terms)."""
    dev, term = np.ravel(dev), np.ravel(term)
    sxx = float(term @ term)
    return (float(dev @ term) / sxx if sxx > 0 else math.nan), int(np.count_nonzero(term))


def lo_slopes(hT_k, x, ws, h_saved):
    """Slope of (kernel - emulation without a lo half) on (emulation - emulation without it), h_T, for each of the three."""
    full = emu.forward(x, *ws, h_saved=h_saved)["h"][:, -1]
    out = {}
    for name, kw in (("x_lo", dict(keep_xlo=False)), ("w_ih lo", dict(keep_wlo=False)), ("b lo", dict(keep_blo=False))):
        without = emu.forward(x, *ws, h_saved=h_saved, **kw)["h"][:, -1]
        out[name] = slope(np.asarray(hT_k, np.float64) - without, full - without)
    return out


def slope_ok(v):
    s, n = v
    return n >= SLOPE_MIN_TERMS and SLOPE_BAND[0] <= s <= SLOPE_BAND[1]


def backward_coefs(C, bw, grads_k, da_k, cells, T):
    """Gradients of a kernel against the emulated walk -> ({stage: coef} element-wise, {stage: rel_L2})."""
    coefs, l2 = {}, {}
    if da_k is not None:
        coefs["da records"] = store_coef(da_k, bw["da"], bw["da_mag"], True)
        L = cells * T
        coefs["dW_hh"] = dw_coef(grads_k["dw_hh"], bw["dw_hh"], bw["dw_hh_mag"], bw["dw_hh_sub"], L)
        coefs["dW_ih"] = dw_coef(grads_k["dw_ih"], bw["dw_ih"], bw["dw_ih_mag"], bw["dw_ih_sub"], L)
        coefs["db"] = dw_coef(grads_k["db"], bw["db"], bw["db_mag"], bw["db_sub"], L)
    else:
        for k in ("dw_hh", "dw_ih", "db"):
            l2[k] = orc.rel_errors(grads_k[k], bw[k])[1]
    l2["dx"] = orc.rel_errors(grads_k["dx"], bw["dx"])[1]
    return coefs, l2


# ------------------------------------------------------------------------------------------------------------------------------
# CPU: the emulation, the decoders and the helpers
# ------------------------------------------------------------------------------------------------------------------------------
def _params(C, seed, xmag=8.0, wih_scale=None, bias_mag=None, S=50, T=5):
    rng = np.random.default_rng(seed)
    k = 1.0 / math.sqrt(C)
    w_ih = (rng.standard_normal((4 * C, 1)) * wih_scale if wih_scale else rng.uniform(-k, k, (4 * C, 1))).astype(np.float32)
    w_hh = rng.uniform(-k, k, (4 * C, C)).astype(np.float32)
    bm = bias_mag or k
    b_ih, b_hh = (rng.uniform(-bm, bm, 4 * C).astype(np.float32) for _ in range(2))
    x = (rng.uniform(0.5, 1.5, (S, T)) * xmag * rng.choice([-1.0, 1.0], (S, T))).astype(np.float32)
    return x, (w_ih, w_hh, b_ih, b_hh)


@pytest.mark.parametrize("C", [8, 32, 96, 128])
def test_emulation_without_roundings_is_the_float64_lstm(C):
    x, ws = _params(C, C, xmag=2.0, S=40, T=6)
    w64 = [w.astype(np.float64) for w in ws]
    x3 = x.astype(np.float64)[:, :, None]
    fwd = emu.forward(x, *ws, exact=True)
    ref = orc.lstm_last_forward(x3, *w64)
    assert np.abs(fwd["h"][:, -1] - ref).max() <= 1e-12
    d_hT = np.random.default_rng(1).standard_normal((40, C))
    bw = emu.backward(x, *ws, d_hT, fwd["c"], fwd["h"], 1.0, exact=True)
    dx, dw_ih, dw_hh, db, _ = orc.lstm_last_backward(x3, *w64, d_hT)
    for a, r in ((bw["dx"], dx[:, :, 0]), (bw["dw_ih"], dw_ih[:, 0]), (bw["dw_hh"], dw_hh), (bw["db"], db)):
        assert np.abs(a - r).max() <= 1e-12 * max(1.0, np.abs(r).max())


@pytest.mark.parametrize("H", TC_WIDTHS)
def test_decoders_invert_the_kernel_layouts(H):
    rng = np.random.default_rng(H)
    CH, CG, CELLS = emu.dims(H)
    cells, T = 2 * CELLS + 5, 3
    c, h = (rng.standard_normal((cells, T, H)).astype(np.float16) for _ in range(2))
    c2, h2 = emu.decode_saved(emu.encode_saved(c, h, H), cells, T, H)
    assert np.array_equal(c2, c.astype(np.float64)) and np.array_equal(h2, h.astype(np.float64))
    da = rng.standard_normal((cells, T, 4 * H)).astype(np.float16)
    rec = emu.decode_da_records(emu.encode_da_records(da, H), cells, T, H)
    assert np.array_equal(rec[:cells], da.astype(np.float64)) and not rec[cells:].any()

    # the formulas of save_off and of the fragment: every half of the buffer lands on its (cell, t, unit)
    nt = emu.tiles(cells, H)
    buf = np.arange(nt * T * CELLS * 2 * H, dtype=np.int64)
    tile, t, w, kind, lane, slot = np.unravel_index(buf, (nt, T, CG * CH, 2, 32, 16))
    off = ((tile * T + t) * (CELLS * 2 * H) + w * 1024 + kind * 512 + lane * 16 + slot)
    assert np.array_equal(off, buf)
    cg, js, g, q, hh, s = w // CH, w % CH, lane >> 2, lane & 3, slot >> 3, slot & 7
    cell = tile * CELLS + 16 * cg + g + 8 * hh
    unit = 32 * js + 8 * (s >> 1) + 2 * q + (s & 1)
    dec_c, dec_h = emu.decode_saved(buf.astype(np.float64), nt * CELLS, T, H)
    got = np.where(kind == 0, dec_c[cell, t, unit], dec_h[cell, t, unit])
    assert np.array_equal(got, buf.astype(np.float64))
    # records: column 128 js + 32 gate + u is gate row gate H + 32 js + u
    rb = np.arange(nt * T * CELLS * 4 * H, dtype=np.int64)
    tile, t, cl, col = np.unravel_index(rb, (nt, T, CELLS, 4 * H))
    j = (col % 128) // 32 * H + 32 * (col // 128) + col % 32
    dec = emu.decode_da_records(rb.astype(np.float64), nt * CELLS, T, H)
    assert np.array_equal(dec[tile * CELLS + cl, t, j], rb.astype(np.float64))


def _simulated_forward(x, ws, gen, kappa=1.0, lag=1, **kw):
    """A kernel that rounds as the emulation does, plus SFU / fp32-sized noise: saved fp16 c_t, h_t and fp32 h_T.  lag = 2 feeds
    step t with h_{t-2} (a wrong operand); kw drop lo halves."""
    S, T = x.shape
    C = ws[1].shape[1]
    wx = emu.build_wx(*ws, **{k: v for k, v in kw.items() if k != "keep_xlo"})
    x_hi, x_lo = emu.x_split(x, keep_xlo=kw.get("keep_xlo", True))
    c = np.zeros((S, C))
    hs, cs = [], []
    for t in range(T):
        h_op = emu.f16(hs[t - lag]) if t - lag >= 0 else np.zeros((S, C))
        c, h, _, mag = emu.step(c, h_op, x_hi[:, t], x_lo[:, t], wx)
        noise = lambda: (gen.random((S, C)) * 2 - 1) * kappa * 2.0 ** -22 * (1 + mag.reshape(S, 4, C).max(axis=1))
        c = c + noise()
        h = h + noise()
        cs.append(c)
        hs.append(h)
    c, h = np.stack(cs, 1), np.stack(hs, 1)
    return emu.f16(c), emu.f16(h), h[:, -1].astype(np.float32).astype(np.float64)


def test_helpers_accept_a_faithful_kernel_and_reject_each_defect():
    gen = np.random.default_rng(0)
    C = 32
    # the lo halves: x not representable in fp16 at |x| ~ 8, w_ih scaled so that x w_ih ~ 1, biases of order 1
    x, ws = _params(C, 3, xmag=8.0, wih_scale=0.125, bias_mag=1.0, S=3800, T=2)
    c_k, h_k, hT_k = _simulated_forward(x, ws, gen)
    fwd = emu.forward(x, *ws, h_saved=h_k)
    coefs = forward_coefs(c_k, h_k, hT_k, fwd)
    assert all(v <= EPS_LSTM for v in coefs.values()), coefs
    sl = lo_slopes(hT_k, x, ws, h_k)
    assert all(slope_ok(v) for v in sl.values()), sl
    for drop, name in (("keep_xlo", "x_lo"), ("keep_blo", "b lo"), ("keep_wlo", "w_ih lo")):
        _, h_d, hT_d = _simulated_forward(x, ws, gen, **{drop: False})
        v = lo_slopes(hT_d, x, ws, h_d)[name]
        assert not slope_ok(v) and abs(v[0]) < 0.2, (name, v)
    # h_{t-1} taken from step t-2
    x5, ws5 = _params(C, 4, S=200, T=5)
    c_l, h_l, hT_l = _simulated_forward(x5, ws5, gen, lag=2)
    bad = forward_coefs(c_l, h_l, hT_l, emu.forward(x5, *ws5, h_saved=h_l))
    assert bad["c_t"] > 100 * EPS_LSTM, bad

    # backward at a wide width: faithful records pass; S off by 2, a zeroed record and a record the dW pass skips fail
    H = 96
    x, ws = _params(H, 5, S=150, T=4)
    c_k, h_k, _ = _simulated_forward(x, ws, gen)
    d_hT = gen.standard_normal((150, H))
    S, _ = emu.expected_scale(float(np.abs(d_hT.astype(np.float32)).max()))
    da_k = emu.f16(emu.backward(x, *ws, d_hT, c_k, h_k, S)["da"])       # a walk that rounds its own da' (dh from those bits)
    bwk = emu.backward(x, *ws, d_hT, c_k, h_k, S, da_kernel=da_k)
    L = 150 * 4

    def kernel_grads(b):                                                   # + fp32-accumulation-sized noise
        out = {k: b[k] + (gen.random(b[k].shape) * 2 - 1) * 2.0 ** -24 * math.sqrt(L) * b[k + "_mag"] for k in ("dw_hh", "dw_ih", "db")}
        return dict(out, dx=b["dx"])

    coefs, l2 = backward_coefs(H, bwk, kernel_grads(bwk), da_k, 150, 4)
    assert all(v <= EPS_LSTM for v in coefs.values()) and all(v <= GRAD32_L2_TOL for v in l2.values()), (coefs, l2)
    coefs, _ = backward_coefs(H, bwk, kernel_grads(bwk), 2 * da_k, 150, 4)                  # S doubled in the walk
    assert coefs["da records"] > 1000 * EPS_LSTM
    zeroed = da_k.copy()
    zeroed[:emu.dims(H)[2], 2] = 0.0                                       # the record of (tile 0, step 2)
    coefs, _ = backward_coefs(H, emu.backward(x, *ws, d_hT, c_k, h_k, S, da_kernel=zeroed), kernel_grads(bwk), zeroed, 150, 4)
    assert coefs["da records"] > 1000 * EPS_LSTM
    step0 = emu.backward(x, *ws, d_hT, c_k, h_k, S, da_kernel=np.where(np.arange(4)[None, :, None] == 0, da_k, 0.0))
    partial = kernel_grads(bwk)                                            # a weight-gradient pass that never adds step 0
    for k in ("dw_hh", "dw_ih", "db"):
        partial[k] = partial[k] - step0[k]
    coefs, _ = backward_coefs(H, bwk, partial, da_k, 150, 4)
    assert max(coefs["dW_hh"], coefs["dW_ih"], coefs["db"]) > 1000 * EPS_LSTM, coefs
    # the gradient scale rule: S off by a factor of 2 is not it
    for amax in (3.1e-7, 1.0, 4096.0, 1e-36, 2.0 ** 121):
        S, invS = emu.expected_scale(amax)
        k = 5 - math.frexp(amax)[1]
        if -100 < k < 100:
            assert 16 <= S * amax < 32 and not 16 <= 2 * S * amax < 32
    assert emu.expected_scale(0.0) == (1.0, 1.0) and emu.expected_scale(1e-36)[0] == 2.0 ** 100


# ------------------------------------------------------------------------------------------------------------------------------
# CPU: the fp32 kernels' length limit
# ------------------------------------------------------------------------------------------------------------------------------
def test_fp32_lstm_supports_exactly_the_lengths_its_backward_holds():
    lib = _lib.load()
    assert {C: fp32_t_max(C) for C in (1, 8, 16, 32, 48, 64)} == {1: 8041, 8: 1130, 16: 545, 32: 224, 48: 95, 64: 15}
    for C in (1, 2, 3, 8, 16, 17, 31, 32, 33, 48, 63, 64):
        tm = fp32_t_max(C)
        for T in (1, 2, tm - 1, tm, tm + 1, 2 * tm):
            if T >= 1:
                assert lib.mpgcn_lstm_precision_supported(T, C, 0) == (T <= tm), (T, C)
    for C in (0, 65, 96, 128):
        assert lib.mpgcn_lstm_precision_supported(1, C, 0) == 0
    assert lib.mpgcn_lstm_precision_supported(0, 8, 0) == 0


def test_auto_precision_keeps_nn_lstm_past_the_fp32_limit():
    for C in (16, 48, 64):
        tm = fp32_t_max(C)
        assert ops.lstm_engine_supports("auto", tm, C) and not ops.lstm_engine_supports("auto", tm + 1, C)
        assert not ops.lstm_engine_supports("fp32", tm + 1, C)
        with pytest.raises(RuntimeError, match="does not support"):
            ops.resolve_lstm_precision("fp32", tm + 1, C)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: fp32 CUDA-core kernels
# ------------------------------------------------------------------------------------------------------------------------------
def _fp32_cases():
    rows = []
    for C in FP32_WIDTHS:
        tm = fp32_t_max(C)
        rows += [(C, T) for T in sorted({1, 2, 15, 16, tm}) if T <= tm]
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("C,T", _fp32_cases())
def test_fp32_lstm_matches_float64_at_every_width_and_length(C, T, cuda_device):
    """B = 2, NN = 37: 74 cells, ragged against the forward tile (256 / C cells, at most 32) and the backward's block, with a
    tile that straddles the batch boundary."""
    B, NN = 2, 37
    rng = np.random.default_rng(1000 * C + T)
    k = 1.0 / math.sqrt(C)
    ws0 = [rng.uniform(-k, k, s).astype(np.float32) for s in ((4 * C, 1), (4 * C, C), (4 * C,), (4 * C,))]
    x0 = (rng.random((B, T, NN)) * 2).astype(np.float32)
    d_h = rng.standard_normal((B * NN, C)).astype(np.float32)
    t = lambda a, g=False: torch.from_numpy(a).to(cuda_device).requires_grad_(g)
    ws = [t(w, True) for w in ws0]
    x = t(x0, True)
    h = ops.lstm_last(x.view(B, T, NN, 1, 1), *ws, precision="fp32")
    h.backward(t(d_h))
    torch.cuda.synchronize()
    xs = x0.transpose(0, 2, 1).reshape(B * NN, T, 1).astype(np.float64)
    w64 = [w.astype(np.float64) for w in ws0]
    tag = f"fp32 lstm C={C} T={T}"
    _rel_check(h.detach().cpu().numpy(), orc.lstm_last_forward(xs, *w64), FP32_H_TOL, f"{tag} hT")
    dx, dw_ih, dw_hh, db_ih, db_hh = orc.lstm_last_backward(xs, *w64, d_h.astype(np.float64))
    for w, r, n in zip(ws, (dw_ih, dw_hh, db_ih, db_hh), ("dw_ih", "dw_hh", "db_ih", "db_hh")):
        _rel_check(w.grad.cpu().numpy(), r, FP32_G_TOL, f"{tag} {n}")
    _rel_check(x.grad.cpu().numpy().transpose(0, 2, 1).reshape(B * NN, T, 1), dx, FP32_G_TOL, f"{tag} dx")


@pytest.mark.gpu
def test_fp32_lstm_predicate_matches_what_both_kernels_run(cuda_device):
    """mpgcn_lstm_precision_supported(T, C, 0) == 1 exactly where forward and backward both return 0 (return codes only)."""
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    B, NN = 1, 3
    p = lambda a: a.data_ptr()
    for C in (1, 8, 16, 31, 32, 48, 63, 64, 65):
        tm = fp32_t_max(C)
        for T in sorted({1, 16, tm, tm + 1}):
            if T < 1:
                continue
            x = torch.rand(B, T, NN, device=cuda_device)
            ws = [torch.rand(s, device=cuda_device) * 0.1 for s in ((4 * C,), (4 * C, C), (4 * C,), (4 * C,))]
            g = [torch.empty_like(w) for w in ws]
            hT = torch.empty(B * NN, C, device=cuda_device)
            d_h = torch.randn(B * NN, C, device=cuda_device)
            dx = torch.empty_like(x)
            wsb = torch.empty(256, dtype=torch.uint8, device=cuda_device)
            rf = lib.mpgcn_lstm_last_forward(p(x), *[p(w) for w in ws], p(hT), B, T, NN, C, 0, st)
            rb = lib.mpgcn_lstm_last_backward(p(x), *[p(w) for w in ws], p(d_h), *[p(a) for a in g], p(dx), p(wsb), 256, B, T, NN, C,
                                              0, st)
            torch.cuda.synchronize()
            sup = lib.mpgcn_lstm_precision_supported(T, C, 0)
            assert sup == int(rf == 0 and rb == 0), (T, C, sup, rf, rb, lib.mpgcn_last_error())


@pytest.mark.gpu
def test_hidden_64_model_trains_past_the_fp32_limit_under_auto(cuda_device, monkeypatch):
    """obs_len 16 at hidden 64: under "auto" (and the default) the model's LSTM is nn.LSTM and a training step completes; an
    explicit "fp32" is refused at forward time."""
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    torch.manual_seed(0)
    N, T = 6, 16
    model = shim.MPGCN(M=2, K=2, input_dim=1, lstm_hidden_dim=64, lstm_num_layers=1, gcn_hidden_dim=32, gcn_num_layers=2,
                       num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    x = torch.rand(2, T, N, N, 1, device=cuda_device)
    G = torch.rand(2, N, N, device=cuda_device) / N
    Gs = [G, (G[None].expand(2, -1, -1, -1).contiguous(),) * 2]
    for prec in ("auto", None):
        model.lstm_precision = prec
        model.zero_grad()
        model(x_seq=x, G_list=Gs).square().mean().backward()
        torch.cuda.synchronize()
        for name, p in model.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), name
    model.lstm_precision = "fp32"
    with pytest.raises(RuntimeError, match="does not support T=16, hidden=64"):
        model(x_seq=x, G_list=Gs)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: tensor-core kernels, stage by stage
# ------------------------------------------------------------------------------------------------------------------------------
def _garbage(nbytes, dev):
    return torch.full((max(nbytes, 1),), 0xFF, dtype=torch.uint8, device=dev)      # fp16 / fp32 NaN: unwritten bytes show


def _align(n):
    return -(-n // 256) * 256


def run_tc(x, ws, d_hT, C, flavour, dev, hint=None):
    """Training forward + one backward flavour ("saved": backward_saved on the forward's state; "rebuild": backward_ex, which
    rebuilds that state in its workspace) through the C ABI into NaN-prefilled buffers -> dict of numpy results and the
    decoded saved state / gate-gradient records."""
    lib = _lib.load()
    B, T, NN = x.shape
    cells = B * NN
    st = torch.cuda.current_stream().cuda_stream
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    p = lambda a: None if a is None else a.data_ptr()
    xt, wt, dh = t(x), [t(w) for w in ws], t(d_hT)
    hT = torch.full((cells, C), math.nan, device=dev)
    nsave = lib.mpgcn_lstm_saved_bytes(B, T, NN, C, 1)
    saved = _garbage(nsave, dev)
    _lib.check(lib.mpgcn_lstm_last_forward_train(p(xt), *[p(w) for w in wt], p(hT), p(saved), nsave, B, T, NN, C, 1, st), "fwd_train")
    g = [torch.full_like(w, math.nan) for w in wt]
    dx = torch.full_like(xt, math.nan)
    nws = lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, 1)
    hint_t = None if hint is None else torch.tensor([hint], dtype=torch.float32, device=dev)
    if flavour == "saved":
        wsb = _garbage(nws - nsave, dev)
        _lib.check(lib.mpgcn_lstm_last_backward_saved(p(xt), *[p(w) for w in wt], p(dh), *[p(a) for a in g], p(dx), p(saved), nsave,
                                                      p(wsb), wsb.numel(), B, T, NN, C, 1, p(hint_t), st), "bwd_saved")
    else:
        wsb = _garbage(nws, dev)
        _lib.check(lib.mpgcn_lstm_last_backward_ex(p(xt), *[p(w) for w in wt], p(dh), *[p(a) for a in g], p(dx), p(wsb), wsb.numel(),
                                                   B, T, NN, C, 1, p(hint_t), st), "bwd_rebuild")
    torch.cuda.synchronize()
    nt = emu.tiles(cells, C)
    da_bytes = 0 if C == 32 else nt * emu.dims(C)[2] * T * 4 * C * 2
    r = dict(hT=hT.cpu().numpy().astype(np.float64), scale2=wsb[:8].view(torch.float32).cpu().numpy().astype(np.float64),
             dw_ih=g[0].cpu().numpy()[:, 0].astype(np.float64), dw_hh=g[1].cpu().numpy().astype(np.float64),
             db=g[2].cpu().numpy().astype(np.float64), db_hh=g[3].cpu().numpy().astype(np.float64),
             dx=dx.cpu().numpy().transpose(0, 2, 1).reshape(cells, T).astype(np.float64))
    state = saved.view(torch.float16).cpu().numpy()
    if flavour == "rebuild":
        o = emu.GRAD_SCALE_BYTES + _align(da_bytes)
        rebuilt = wsb[o:o + nsave]
        assert torch.equal(rebuilt, saved), "the rebuilt state differs from the training forward's"
        state = rebuilt.view(torch.float16).cpu().numpy()
    r["c"], r["h"] = emu.decode_saved(state, cells, T, C)
    if C != 32:
        rec = wsb[emu.GRAD_SCALE_BYTES:emu.GRAD_SCALE_BYTES + da_bytes].view(torch.float16).cpu().numpy()
        r["da"] = emu.decode_da_records(rec, cells, T, C)
    return r


def tc_inputs(C, B, NN, T, xmag, gmag, seed, wih_scale=None, bias_mag=None):
    x_cells, ws = _params(C, seed, xmag=xmag, wih_scale=wih_scale, bias_mag=bias_mag, S=B * NN, T=T)
    x = np.ascontiguousarray(x_cells.reshape(B, NN, T).transpose(0, 2, 1))                      # [B, T, NN]
    d_hT = (np.random.default_rng(seed + 1).standard_normal((B * NN, C)) * gmag).astype(np.float32)
    return x, x_cells, ws, d_hT


def check_tc(r, x_cells, ws, d_hT, C, tag, hint=None):
    """Every stage of one run_tc result -> {stage: coef} (asserts the exact parts on the way)."""
    cells, T = x_cells.shape
    # decoder pin: the saved h of the last step are the fp16 bits of the returned h_T
    assert not np.isnan(r["h"]).any() and not np.isnan(r["c"]).any(), f"{tag}: saved state has unwritten halves"
    assert np.array_equal(r["h"][:, -1], emu.f16(r["hT"])), f"{tag}: decoded saved h_(T-1) != fp16(h_T)"
    res = {}
    fwd = emu.forward(x_cells, *ws, h_saved=r["h"])
    res.update({f"fwd {k}": v for k, v in forward_coefs(r["c"], r["h"], r["hT"], fwd).items()})
    amax = float(np.abs(d_hT).max()) if hint is None else hint
    S, invS = emu.expected_scale(amax)
    assert tuple(r["scale2"]) == (S, invS), f"{tag}: gradient scale {tuple(r['scale2'])}, want {(S, invS)} for max|d_hT| {amax:.6e}"
    assert np.array_equal(r["db"], r["db_hh"]), f"{tag}: d_b_hh != d_b_ih"
    da_k = None
    if C != 32:
        assert not r["da"][cells:].any(), f"{tag}: gate-gradient records of the padded cells are not zero"
        da_k = r["da"][:cells]
    bw = emu.backward(x_cells, *ws, d_hT, r["c"], r["h"], S, da_kernel=da_k)
    coefs, l2 = backward_coefs(C, bw, r, da_k, cells, T)
    res.update({f"bwd {k}": v for k, v in coefs.items()})
    return res, l2


def _assert_and_record(res, l2, tag):
    bad = []
    for stage, v in res.items():
        record_parity(f"lstm stages {tag} {stage}: coef", v, v, EPS_LSTM)
        if not v <= EPS_LSTM:
            bad.append(f"{stage}: coef {v:.3g} > {EPS_LSTM}")
    for stage, v in l2.items():
        record_parity(f"lstm stages {tag} {stage}: rel_L2 vs emulated walk", v, v, GRAD32_L2_TOL)
        if not v <= GRAD32_L2_TOL:
            bad.append(f"{stage}: rel_L2 {v:.3g} > {GRAD32_L2_TOL}")
    assert not bad, f"{tag}: " + "; ".join(bad)


def _tc_cases():
    rows = []
    for C in TC_WIDTHS:
        tile = TC_TILE[C]
        rows += [(C, 1, 1, 17, 8.0, 1.0), (C, 1, tile - 1, 256, 8.0, 1.0), (C, 2, tile // 2, 2, 3000.0, 1e3),
                 (C, 1, tile + 1, 17, 0.01, 1e-7), (C, 2, tile // 2 + 3, 1, 8.0, 1.0), (C, 2, "grid", 2, 8.0, 1.0)]
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("C,B,NN,T,xmag,gmag", _tc_cases())
def test_tc_lstm_every_stage_matches_the_emulation(C, B, NN, T, xmag, gmag, cuda_device):
    if NN == "grid":          # one cell past a full grid of tiles (two tiles per CTA at hidden 32's forward grid of 2 per SM)
        sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
        NN = (sms * (2 if C == 32 else 1) * TC_TILE[C]) // 2 + 1
    x, x_cells, ws, d_hT = tc_inputs(C, B, NN, T, xmag, gmag, seed=C * 7 + B * NN + T)
    for flavour in ("saved", "rebuild"):
        r = run_tc(x, ws, d_hT, C, flavour, cuda_device)
        tag = f"C={C} B={B} NN={NN} T={T} |x|~{xmag:g} |dh|~{gmag:g} {flavour}"
        res, l2 = check_tc(r, x_cells, ws, d_hT, C, tag)
        _assert_and_record(res, l2, tag)


@pytest.mark.gpu
@pytest.mark.parametrize("C", TC_WIDTHS)
@pytest.mark.parametrize("xmag", [8.0, 3000.0])
def test_tc_lstm_keeps_every_lo_half(C, xmag, cuda_device):
    """x not representable in fp16 at |x| ~ 8 and ~ 3000, w_ih scaled so that x w_ih ~ 1, biases of order 1: h_T must contain
    the contribution of x_lo, of the lo half of s_j w_ih and of the lo half of s_j b (slope 1), and meet the forward bounds."""
    B, T = 2, 2
    NN = -(-6 * SLOPE_MIN_TERMS // (10 * C)) + 7          # 1.2 x the terms a slope needs
    x, x_cells, ws, d_hT = tc_inputs(C, B, NN, T, xmag, 1.0, seed=C + int(xmag), wih_scale=1.0 / xmag, bias_mag=1.0)
    r = run_tc(x, ws, d_hT, C, "saved", cuda_device)
    tag = f"C={C} |x|~{xmag:g} lo halves"
    res, l2 = check_tc(r, x_cells, ws, d_hT, C, tag)
    _assert_and_record(res, l2, tag)
    bad = []
    for name, (s, n) in lo_slopes(r["hT"], x_cells, ws, r["h"]).items():
        record_parity(f"lstm stages {tag} {name} (n={n}): |slope - 1|", abs(s - 1), abs(s - 1), SLOPE_BAND[1] - 1)
        if not slope_ok((s, n)):
            bad.append(f"{name}: slope {s:.3f} over {n} terms (want 1)")
    assert not bad, f"{tag}: " + "; ".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("C", TC_WIDTHS)
@pytest.mark.parametrize("case", ["zero", "tiny", "huge", "hint"])
def test_tc_lstm_gradient_scale(C, case, cuda_device):
    """S = 2^k with S max|d_hT| in [16, 32): S = 1 for a zero d_hT, the +-100 exponent clamp at max|d_hT| ~ 1e-36 and 2^105.5
    (S max|d_hT| ~ 45, still inside fp16 once scaled), and a d_hT_absmax hint of twice the true maximum is followed (S halves)
    with every stage bound still met."""
    B, NN, T = 2, TC_TILE[C] // 2 + 5, 3
    x, x_cells, ws, d_hT = tc_inputs(C, B, NN, T, 8.0, 1.0, seed=C + 3)
    hint = None
    if case == "zero":
        d_hT = np.zeros_like(d_hT)
    elif case == "tiny":
        d_hT = (d_hT * 1e-36).astype(np.float32)
    elif case == "huge":
        d_hT = (d_hT / np.abs(d_hT).max() * 2.0 ** 105.5).astype(np.float32)
    else:
        hint = 2.0 * float(np.abs(d_hT).max())
    r = run_tc(x, ws, d_hT, C, "saved", cuda_device, hint=hint)
    amax = float(np.abs(d_hT).max()) if hint is None else hint
    S = emu.expected_scale(amax)[0]
    assert S == {"zero": 1.0, "tiny": 2.0 ** 100, "huge": 2.0 ** -100}.get(case, S)
    if case == "hint":
        assert S == emu.expected_scale(float(np.abs(d_hT).max()))[0] / 2
    tag = f"C={C} scale {case}"
    res, l2 = check_tc(r, x_cells, ws, d_hT, C, tag, hint=hint)
    for k in ("dw_ih", "dw_hh", "db", "dx"):
        assert np.isfinite(r[k]).all(), f"{tag}: {k} not finite"
    if case == "zero":
        assert not any(r[k].any() for k in ("dw_ih", "dw_hh", "db", "dx")), f"{tag}: gradients of a zero d_hT are not zero"
        return
    if case == "tiny":            # S d_hT ~ 1e-6: the fp16 gate gradients are subnormal, so only the forward stages are bounded
        res = {k: v for k, v in res.items() if k.startswith("fwd")}
        l2 = {}
    _assert_and_record(res, l2, tag)
