"""The tensor-core BDGCN layer (precision 1) at channel widths other than 32.

Any C and H that are multiples of 32 run on the tensor cores, C != H included (the first layer of a branch has C =
lstm_hidden_dim).  A "chunk" is 32 consecutive channels, cC = C / 32 and cH = H / 32: the N^3 contractions run once per chunk
(they act on each channel on its own), the channel mixes see Kd*cC input and Ko*cH output planes, and BWD_DW tiles Kd*cC by
Ko*cH chunks (DESIGN.md section 5).

  * CPU: the oracle against fixtures of the unmodified reference (`tests/golden/wide_*`, tools/gen_golden_wide.py); which
    shapes the tensor path accepts.
  * GPU: every stage against float64 with the helpers and bounds of test_gpu_engine_stages.py, reading the chunk layouts back
    from the workspaces; the layer against the fixtures and the factored oracle at size; the whole model at hidden 64; a row
    shard.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
from torch import nn

import abi
import test_gpu_at_size as at_size
from conftest import golden_names, load_golden, record_parity
from oracle import mpgcn_oracle as orc
from oracle.gen_golden import layer_fixture
from test_gpu_engine_stages import (Bound, Slope, _assert_and_record, _chunks, _garbage, bits, contract, dense_supports, diag_rule,
                                    diag_supports, expected_scale, f16_sat, fwd_a_ref, fwd_b_ref, hilo, mix_ref)

import MPGCN as shim
from mpgcn_b200 import _lib, ops, shard
from tools.gen_golden_wide import params_checksum, wide_model_params

FIXTURE_TOL = 2e-5
FWD_TOL = {"fp32": 5e-5, "fp16": 1e-3}
BWD_TOL = {"fp32": 2e-4, "fp16": 2e-3}
LOOSE_FP16_GRAD = 8e-2


def _rel_check(a, ref, tol, what, l2_only=False):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    ref = ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol), f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"
    return linf, l2


def _graph(g):
    return (g["G_o"], g["G_d"]) if int(g["dynamic"]) else g["G"]


def _model_params(g):
    """The parameters of a wide model fixture, regenerated from its seed (tools/gen_golden_wide.py) and checked against the
    stored checksum -> {state_dict key: float32 array}."""
    hid, K, N = int(g["hidden"]), int(g["K"]), g["x_seq"].shape[2]
    shapes = {k: v.shape for k, v in _model(N, K, hid, 0, "cpu").state_dict().items()}
    params = wide_model_params(int(g["seed"]), shapes)
    assert abs(float(params_checksum(params)) - float(g["params_checksum"])) < 1e-6, "numpy RNG stream changed: regenerate the fixture"
    return params


def _check_model_grads(grads, g, tol, what):
    """Gradients against a wide model fixture: every BDGCN W gradient on the stored rows (`W_rows`) and in norm, every other
    gradient in full."""
    assert set(grads) == {k.split(":", 1)[1] for k in g if k.startswith(("grad:", "grad_rows:"))}
    rows = g["W_rows"]
    for k, v in grads.items():
        v = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        if "grad_rows:" + k in g:
            _rel_check(v[rows], g["grad_rows:" + k], tol, f"{what}/grad:{k} rows")
            ref = float(g["grad_norm:" + k])
            assert abs(float(np.linalg.norm(v.astype(np.float64))) - ref) <= tol * ref, f"{what}/grad:{k}: norm of the whole tensor"
        else:
            _rel_check(v, g["grad:" + k], tol, f"{what}/grad:{k}")


# ------------------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------------------
def test_wide_fixtures_exist_and_stay_out_of_the_other_sets():
    layers, models = golden_names("wide_bdgcn_"), golden_names("wide_mpgcn_")
    assert len(layers) == 4 and len(models) == 1
    widths = {(int(load_golden(n)["C"]), int(load_golden(n)["H"])) for n in layers}
    assert widths == {(64, 64), (64, 96), (32, 64), (128, 128)}
    assert int(load_golden(models[0])["hidden"]) == 64
    for prefix in ("bdgcn_", "big_bdgcn_", "many_bdgcn_", "mpgcn_"):
        assert not set(layers + models) & set(golden_names(prefix))


@pytest.mark.parametrize("name", golden_names("wide_bdgcn_"))
def test_oracle_matches_reference_at_wide_channels(name):
    g = layer_fixture(load_golden(name))
    K, C, H = int(g["K"]), int(g["C"]), int(g["H"])
    assert g["W"].shape == (K * K * C, H) and g["X"].shape[-1] == C
    out = orc.bdgcn_forward(g["X"], _graph(g), g["W"], g["b"], "relu")
    _rel_check(out, g["out"], FIXTURE_TOL, f"{name}: out")
    dX, dW, db = orc.bdgcn_backward(g["X"], _graph(g), g["W"], g["b"], "relu", g["d_out"])
    for a, k in ((dX, "dX"), (dW, "dW"), (db, "db")):
        _rel_check(a, g[k], FIXTURE_TOL, f"{name}: {k}")
    fac = orc.bdgcn_backward_factored(g["X"], _graph(g), g["W"], g["b"], "relu", g["d_out"])
    for a, k in zip(fac, ("out", "dX", "dW", "db")):
        _rel_check(a, g[k], FIXTURE_TOL, f"{name}: factored {k}")


@pytest.mark.parametrize("name", golden_names("wide_mpgcn_"))
def test_oracle_matches_reference_model_at_hidden_64(name):
    g = load_golden(name)
    y, grads = orc.mpgcn_forward_backward(_model_params(g), g["x_seq"], [g["G_static"], (g["G_o"], g["G_d"])], M=2, gcn_num_layers=3,
                                          d_y=g["d_y"])
    _rel_check(y, g["y"], FIXTURE_TOL, f"{name}: y")
    _check_model_grads(grads, g, FIXTURE_TOL, name)


@pytest.mark.parametrize("C,H,want", [(32, 32, 1), (64, 64, 1), (32, 64, 1), (64, 32, 1), (96, 128, 1), (256, 256, 1),
                                      (16, 32, 0), (48, 48, 0), (64, 16, 0)])
def test_tensor_path_accepts_multiples_of_32(C, H, want):
    lib = _lib.load()
    assert lib.mpgcn_bdgcn_precision_supported(2, 50, 3, C, H, 1) == want
    assert ops.resolve_precision("auto", 2, 50, 3, C, H) == (_lib.PREC_FP16_TC if want else _lib.PREC_FP32)
    if not want:
        with pytest.raises(RuntimeError, match="multiples of 32"):
            ops.resolve_precision("fp16", 2, 50, 3, C, H)


def test_lstm_keeps_its_fp32_kernels_at_hidden_64():
    lib = _lib.load()
    assert lib.mpgcn_lstm_precision_supported(5, 64, 1) == 0 and lib.mpgcn_lstm_precision_supported(5, 64, 0) == 1


# ------------------------------------------------------------------------------------------------------------------------------
# one layer through the C ABI at any width, the chunk layouts read back from the workspaces
# ------------------------------------------------------------------------------------------------------------------------------
class Layout(dict):
    """name -> byte offset of consecutive regions, each starting at a multiple of `align` (bdgcn_tc.cu layouts: 1024; bdgcn_simt.cu
    layouts: 256); .size[name] = its bytes, .total = the workspace size the library asks for (`slack` bytes added)."""

    def __init__(self, parts, align=1024, slack=0):
        super().__init__()
        self.size, off = {}, 0
        for name, nbytes in parts:
            off = -(-off // align) * align
            self[name], self.size[name] = off, nbytes
            off += nbytes
        self.total = -(-off // align) * align + slack


def dw_slices(B, R, N, rows, cols, sms):
    """Split-K slices of BWD_DW (bdgcn_tc.cu dw_slices): rows = Kd*cC, cols = Ko*cH chunks, 64-row k-blocks per sample slab"""
    total = B * -(-R * N // 64)
    tiles = -(-rows // 4) * -(-cols // 8)
    per = max(1, -(-total // max(1, sms // tiles)))
    return -(-total // per)


def part_ws_layout(B, N, C, H, dyn, R, row0, Ko, Kd, sms):
    """The forward / backward workspace layouts of a layer part (bdgcn_tc.cu fwd_layout / bwd_layout): origin rows [row0, row0 + R)
    (the layout does not depend on row0), Ko origin and Kd destination supports.  The whole layer is R = N, Ko = Kd = K."""
    nz, Np, RN = (B if dyn else 1), (N + 7) // 8 * 8, R * N
    g16, rem = (lambda K: nz * K * N * Np * 2), (lambda K: nz * K * N * 4)
    fwd = Layout([("x16", B * RN * C * 2), ("gd16", g16(Kd)), ("go16", g16(Ko)), ("w16", 2 * Ko * Kd * C * H * 2), ("u16", B * Ko * RN * H * 2),
                  ("dd", rem(Kd)), ("dgo", rem(Ko)), ("dgo_masked", rem(Ko)), ("z16", B * Kd * RN * C * 2)])
    rows, cols = Kd * C // 32, Ko * H // 32
    slices = dw_slices(B, R, N, rows, cols, sms)
    bwd = Layout([("dp16", B * N * N * H * 2), ("gd16", g16(Kd)), ("go16", g16(Ko)), ("v16", B * Ko * RN * H * 2), ("y16", B * Kd * RN * C * 2),
                  ("wq16", Ko * Kd * C * H * 2), ("partials", slices * -(-rows // 4) * 128 * Ko * H * 4), ("scale", 64)])
    return fwd, bwd


def ws_layout(B, N, K, C, H, dyn, sms):
    """The forward / backward workspace layouts of a whole layer."""
    return part_ws_layout(B, N, C, H, dyn, N, 0, K, K, sms)


def simt_ws_layout(B, N, C, H, R, Ko, Kd):
    """The fp32 family's workspaces (bdgcn_simt.cu simt_fwd_layout / simt_bwd_layout): forward U (Z lives in `saved`; its region serves only a call without
    one); backward dPre (whole layer: a part reads the caller's), V, Y, Wq [d][o][h][l].  The size functions add 256 / 1024 bytes."""
    RN = R * N
    fwd = Layout([("u", B * Ko * RN * H * 4), ("z", B * Kd * RN * C * 4)], 256, 256)
    bwd = Layout([("dpre", B * N * N * H * 4), ("v", B * Ko * RN * H * 4), ("y", B * Kd * RN * C * 4), ("wq", Ko * Kd * C * H * 4)], 256, 1024)
    return fwd, bwd


def _nan_alloc(nbytes, dev, what):
    return _garbage(nbytes, dev)


def run_layer_wide(X, Go, Gd, W, bias, d_out, dyn, row0=None, prec=1, alloc=_nan_alloc, d_pre16=None):
    """Forward + backward of one layer (ReLU) or, with row0 set, of one PART of a layer (mpgcn_bdgcn_forward_part / _backward_part):
    X is then the slab [B,R,N,C] of origin rows [row0, row0 + R), Go / Gd hold the part's Ko / Kd supports, W its [Ko*Kd*C, H]
    slice, `out` receives the raw partial pre-activation and d_out is dPre -- or d_pre16 = (fp16 dPre, [S, 1/S]) as
    mpgcn_relu_backward_scatter_f16 leaves them, passed in the extras.  prec 1: the tensor-core family, 0: the fp32 one.
    Every buffer the library writes comes from alloc(nbytes, device, what) (uint8, prefilled).
    -> outputs and the intermediates in their logical layouts (n < R): Z / Y [B][d][n][e][C], U / V [B][o][n][e][H], dP [B][m][e][H];
    tensor cores: W16 [2][o][d][C][H], Wq16 [o][d][C][H] and the fp16 operand copies; fp32: Wq [d][o][H][C] as stored."""
    lib = _lib.load()
    dev = X.device
    B, R, N, C = X.shape
    Ko, Kd, H = Go.shape[-3], Gd.shape[-3], W.shape[1]
    part, backward = row0 is not None, d_out is not None or d_pre16 is not None
    nz, Np = (B if dyn else 1), (N + 7) // 8 * 8
    st = torch.cuda.current_stream().cuda_stream
    if part:
        pdesc = _lib.BdgcnPart(row0, R, Ko, Kd)
        pp = ctypes.addressof(pdesc)
        n_saved = lib.mpgcn_bdgcn_part_saved_bytes(B, N, C, H, prec, pp)
        n_ws = lib.mpgcn_bdgcn_part_fwd_workspace_bytes(B, N, C, H, int(dyn), prec, pp)
        n_wsb = lib.mpgcn_bdgcn_part_bwd_workspace_bytes(B, N, C, H, int(dyn), prec, pp)
    else:
        assert R == N and Ko == Kd
        n_saved = lib.mpgcn_bdgcn_saved_bytes(B, N, Ko, C, H, prec)
        n_ws = lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, Ko, C, H, int(dyn), prec)
        n_wsb = lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, Ko, C, H, int(dyn), prec)
    if prec == 1:
        fo, bo = part_ws_layout(B, N, C, H, dyn, R, row0 or 0, Ko, Kd, torch.cuda.get_device_properties(dev).multi_processor_count)
    else:
        fo, bo = simt_ws_layout(B, N, C, H, R, Ko, Kd)
    assert (fo.total, bo.total) == (n_ws, n_wsb), f"workspace layouts {(fo.total, bo.total)} != library sizes {(n_ws, n_wsb)}"
    assert n_saved == B * Kd * R * N * C * (2 if prec == 1 else 4)
    out_b = alloc(4 * B * N * N * H, dev, "out")
    out = out_b.view(torch.float32).view(B, N, N, H)
    saved = alloc(n_saved, dev, "saved")
    ws = alloc(n_ws, dev, "forward workspace")
    if part:
        _lib.check(lib.mpgcn_bdgcn_forward_part(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn), W.data_ptr(), out.data_ptr(),
                                                saved.data_ptr(), ws.data_ptr(), n_ws, B, N, C, H, prec, pp, None, st), "forward_part")
    else:
        _lib.check(lib.mpgcn_bdgcn_forward(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn), W.data_ptr(), bias.data_ptr(), 1, out.data_ptr(),
                                           saved.data_ptr(), ws.data_ptr(), n_ws, B, N, Ko, C, H, prec, st), "forward")
    r = dict(out=out, layouts=(fo, bo), bufs=dict(out=out_b, saved=saved, ws=ws))
    if backward:
        dX_b = alloc(4 * B * R * N * C, dev, "dX")
        dX = dX_b.view(torch.float32).view(B, R, N, C)
        dW = torch.full_like(W, math.nan)
        wsb = alloc(n_wsb, dev, "backward workspace")
        if part:
            ex = _lib.BdgcnExtras()
            if d_pre16 is not None:
                ex.d_pre_f16, ex.d_pre_scale2 = d_pre16[0].data_ptr(), d_pre16[1].data_ptr()
            _lib.check(lib.mpgcn_bdgcn_backward_part(None if d_pre16 is not None else d_out.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn),
                                                     W.data_ptr(), saved.data_ptr(), dX.data_ptr(), dW.data_ptr(), wsb.data_ptr(), n_wsb, B, N, C,
                                                     H, prec, pp, ctypes.addressof(ex), st), "backward_part")
        else:
            db = torch.full((H,), math.nan, device=dev)
            dx_amax = torch.full((1,), math.nan, device=dev)
            _lib.check(lib.mpgcn_bdgcn_backward_ex(d_out.data_ptr(), out.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn), W.data_ptr(), 1,
                                                   saved.data_ptr(), dX.data_ptr(), dW.data_ptr(), db.data_ptr(), wsb.data_ptr(), n_wsb,
                                                   B, N, Ko, C, H, prec, None, dx_amax.data_ptr(), st), "backward_ex")
            r.update(db=db, dx_amax=dx_amax)
        r.update(dX=dX, dW=dW)
        r["bufs"].update(dX=dX_b, wsb=wsb)
    torch.cuda.synchronize()

    if prec != 1:
        r.update(z=saved.view(torch.float32).view(B, Kd, R, N, C), u=f32(ws, fo["u"], B, Ko, R, N, H))
        if backward:
            r.update(simt_backward_views(wsb, bo, B, R, N, C, H, Ko, Kd, part))
        return r
    cC = C // 32
    r.update(x16=h16(ws, fo["x16"], B, R, N, C), gd16=h16(ws, fo["gd16"], nz, Kd, N, Np), dd=f32(ws, fo["dd"], nz, Kd, N),
             w16=w16_view(ws, fo["w16"], Ko, Kd, C, H), u=u16_view(ws, fo["u16"], B, Ko, R, N, H),
             z=in_planes(saved.view(torch.float16).view(B, Kd, cC, R, N, 32)))
    # G_o gets its own fp16 copy (and remainders) unless it is the G_d buffer with as many planes: nothing writes go16 / dgo then
    r["own_go"] = own_go = Go.data_ptr() != Gd.data_ptr() or Ko != Kd
    r["go16"], r["dgo"] = (h16(ws, fo["go16"], nz, Ko, N, Np), f32(ws, fo["dgo"], nz, Ko, N)) if own_go else (r["gd16"], r["dd"])
    if R < N:
        r["dgo_masked"] = f32(ws, fo["dgo_masked"], nz, Ko, N)
    if backward:
        r.update(tc_backward_views(wsb, bo, B, R, N, C, H, Ko, Kd, nz, own_go))
        if d_pre16 is not None:
            r.update(dp=d_pre16[0], scale=d_pre16[1])
    return r


def h16(buf, o, *shape):
    return buf[o:o + 2 * math.prod(shape)].view(torch.float16).view(*shape)


def f32(buf, o, *shape):
    return buf[o:o + 4 * math.prod(shape)].view(torch.float32).view(*shape)


def in_planes(t):
    """[B][d][lc][n][e][32] -> [B][d][n][e][C]"""
    B, Kd, cC, R, N = t.shape[:5]
    return t.permute(0, 1, 3, 4, 2, 5).reshape(B, Kd, R, N, 32 * cC)


def out_planes(t):
    """[B][o][hc][n][e][32] -> [B][o][n][e][H]"""
    B, Ko, cH, R, N = t.shape[:5]
    return t.permute(0, 1, 3, 4, 2, 5).reshape(B, Ko, R, N, 32 * cH)


def w16_view(buf, o, Ko, Kd, C, H):
    """The mix's fp16 W split [2][hc][o][d][lc][32][32] -> [2][o][d][C][H]"""
    return h16(buf, o, 2, H // 32, Ko, Kd, C // 32, 32, 32).permute(0, 2, 3, 4, 5, 1, 6).reshape(2, Ko, Kd, C, H)


def u16_view(buf, o, B, Ko, R, N, H):
    """U16 [B][hc][o][n][e][32] -> [B][o][n][e][H]"""
    return h16(buf, o, B, H // 32, Ko, R, N, 32).permute(0, 2, 3, 4, 1, 5).reshape(B, Ko, R, N, H)


def tc_backward_views(wsb, bo, B, R, N, C, H, Ko, Kd, nz, own_go):
    """The tensor-core backward workspace in logical layouts: dP16, [S, 1/S], the fp16 supports, V16 / Y16 and Wq16 [o][d][C][H]."""
    Np, cC, cH = (N + 7) // 8 * 8, C // 32, H // 32
    r = dict(dp=h16(wsb, bo["dp16"], B, N, N, H), scale=f32(wsb, bo["scale"], 2), bgd16=h16(wsb, bo["gd16"], nz, Kd, N, Np),
             v=out_planes(h16(wsb, bo["v16"], B, Ko, cH, R, N, 32)), y=in_planes(h16(wsb, bo["y16"], B, Kd, cC, R, N, 32)),
             wq16=h16(wsb, bo["wq16"], Kd, cC, Ko, cH, 32, 32).permute(2, 0, 1, 5, 3, 4).reshape(Ko, Kd, C, H))
    r["bgo16"] = h16(wsb, bo["go16"], nz, Ko, N, Np) if own_go else r["bgd16"]
    return r


def simt_backward_views(wsb, bo, B, R, N, C, H, Ko, Kd, part):
    """The fp32 backward workspace: V, Y, Wq [d][o][H][C] as stored and (whole layer) dPre."""
    r = dict(v=f32(wsb, bo["v"], B, Ko, R, N, H), y=f32(wsb, bo["y"], B, Kd, R, N, C), wq=f32(wsb, bo["wq"], Kd, Ko, H, C))
    if not part:
        r["dpre"] = f32(wsb, bo["dpre"], B, N, N, H)
    return r


def _dims(X, Go, Gd, W, dyn):
    B, R, N, C = X.shape
    Ko, Kd, H = Go.shape[-3], Gd.shape[-3], W.shape[1]
    nz = B if dyn else 1
    wf = max(1, -(-(C + H) // 32))        # memory budget of the float64 recomputation, in 32-channel units
    return B, R, N, C, H, Ko, Kd, nz, Go.reshape(nz, Ko, N, N), Gd.reshape(nz, Kd, N, N), W.view(Ko, Kd, C, H), wf


def forward_stages(r, X, Go, Gd, W, bias, dyn, kind, row0=None, prec=1):
    """The forward stages of run_layer_wide's result against float64 -> {stage: Bound or Slope}.  The fp32 family is the same algebra
    with no operand conversions, no remainders, no `lo` half of W and fp32 intermediates."""
    B, R, N, C, H, Ko, Kd, nz, Go4, Gd4, W4, wf = _dims(X, Go, Gd, W, dyn)
    part, row0, fp16 = row0 is not None, row0 or 0, prec == 1
    zb = (lambda b: b) if dyn else (lambda b: 0)
    res = {}
    if fp16:
        assert torch.equal(bits(r["x16"]), bits(f16_sat(X))), "x16"
        for g16, G, what in ((r["gd16"], Gd4, "gd16"), (r["go16"], Go4, "go16")):
            assert torch.equal(bits(g16[..., :N]), bits(f16_sat(G))) and not bits(g16[..., N:]).any(), what
        hi, lo = hilo(W4)
        assert torch.equal(bits(r["w16"][0]), bits(hi)) and torch.equal(bits(r["w16"][1]), bits(lo)), "w16 hi / lo in the mix's chunk order"
        fired = 0.0
        for name, G in (("dd", Gd4), ("dgo", Go4)):
            P = G.shape[1]
            want, near = diag_rule(G.reshape(nz * P, N, N).cpu().numpy())
            got = r[name].reshape(nz * P, N).double().cpu().numpy()
            assert not ((got != want) & ~near).any(), f"{name}: remainders differ from the tau = 1/16 rule"
            fired = max(fired, np.count_nonzero(got) / (nz * P * N))
        if kind == "diag":
            assert fired >= 0.5, "the inputs were meant to make the remainder correction fire"
        dgo = r["dgo"]
        if "dgo_masked" in r:                 # a row slab: the origin remainders act on the slab's own rows m only
            m = r["dgo_masked"]
            assert torch.equal(bits(m[..., row0:row0 + R]), bits(dgo[..., row0:row0 + R])), "dgo_masked != dgo on the slab rows"
            assert not bits(m[..., :row0]).any() and not bits(m[..., row0 + R:]).any(), "dgo_masked != 0 outside the slab rows"
            dgo = m
        x, gd, go, dd = r["x16"], r["gd16"][..., :N], r["go16"][..., :N], r["dd"]
    else:
        x, gd, go, hi, lo = X, Gd4, Go4, W4, torch.zeros_like(W4)
        dd, dgo = torch.zeros(nz, Kd, N, device=X.device), torch.zeros(nz, Ko, N, device=X.device)
    z, u, out = r["z"], r["u"], r["out"]

    bA, sA = Bound(N, fp16), Slope()
    for b in range(B):
        for d in range(Kd):
            for ns in _chunks(R, N * 32 * wf):
                base, corr, ab = fwd_a_ref(x[b, ns], gd[zb(b), d], dd[zb(b), d])
                y = z[b, d, ns]
                bA.add(y, base + corr, ab)
                sA.add(y.double() - base, corr)
    res["FWD_A"] = bA

    bM, sM = Bound((2 if fp16 else 1) * Kd * C, fp16), Slope()
    for b in range(B):
        for ns in _chunks(R, (Ko + Kd) * N * 32 * 2 * wf):
            base, lpart, ab = mix_ref(z[b, :, ns], hi, lo)
            y = u[b, :, ns]
            bM.add(y, base + lpart, ab)
            sM.add(y.double() - base, lpart)
    res["FWD_MIX"] = bM

    # FWD_B: a part's output is the raw partial sum over (o, n in the slab) for every m (no bias, no ReLU)
    bB, sB = Bound(Ko * R + Ko + 1, False), Slope()
    for b in range(B):
        for es in _chunks(N, Ko * R * 32 * 4 * wf):
            base, corr, ab = fwd_b_ref(go[zb(b), :, row0:row0 + R], u[b, :, :, es], dgo[zb(b)], None if part else bias, row0)
            y = out[b, :, es]
            bB.add(y, base + corr if part else torch.relu(base + corr), ab)
            sB.add(y.double() - base, corr if part else corr * (y > 0))
    res["FWD_B"] = bB
    if fp16:
        res.update({"FWD_A remainder slope": sA, "FWD_MIX lo slope": sM, "FWD_B remainder slope": sB})
    return res


def backward_stages(r, X, Go, Gd, W, d_out, dyn, row0=None, prec=1, amax=None):
    """The backward stages of run_layer_wide's result against float64 -> {stage: Bound}.  d_out: dOut of a whole layer (ReLU), dPre
    of a part; amax: the max|dPre| the gradient scale comes from (default max|d_out|; a prepared dPre takes a global one)."""
    B, R, N, C, H, Ko, Kd, nz, Go4, Gd4, W4, wf = _dims(X, Go, Gd, W, dyn)
    part, row0, fp16 = row0 is not None, row0 or 0, prec == 1
    zb = (lambda b: b) if dyn else (lambda b: 0)
    res = {}
    d_pre = d_out if part else torch.where(r["out"] > 0, d_out, torch.zeros_like(d_out))
    if fp16:
        S, invS = expected_scale(float(d_out.abs().max()) if amax is None else amax)
        assert (float(r["scale"][0]), float(r["scale"][1])) == (S, invS), "gradient scale"
        assert torch.equal(bits(r["dp"]), bits(f16_sat(d_pre * S))), "dP16 != fp16_sat(S dPre)"
        for g16, G, what in ((r["bgd16"], Gd4, "backward gd16"), (r["bgo16"], Go4, "backward go16")):
            assert torch.equal(bits(g16[..., :N]), bits(f16_sat(G))) and not bits(g16[..., N:]).any(), what
        assert torch.equal(bits(r["wq16"]), bits(f16_sat(W4))), "wq16 != fp16(W) in the backward mix's chunk order"
        dp, bgd, bgo, wq = r["dp"], r["bgd16"][..., :N], r["bgo16"][..., :N], r["wq16"].permute(1, 0, 3, 2)      # wq: [d][o][h][c]
    else:
        S = invS = 1.0
        if not part:
            assert torch.equal(r["dpre"], d_pre), "dPre != dOut * [out > 0]"
        assert torch.equal(bits(r["wq"]), bits(W4.permute(1, 0, 3, 2).contiguous())), "Wq != W as [d][o][h][c]"
        dp, bgd, bgo, wq = d_pre, Gd4, Go4, r["wq"]
    if not part:
        res["db"] = Bound(B * N * N, False).add(r["db"], d_pre.double().sum(dim=(0, 1, 2)), d_pre.double().abs().sum(dim=(0, 1, 2)))
    v, y = r["v"], r["y"]

    bV = Bound(N, fp16)
    for b in range(B):
        for o in range(Ko):
            for es in _chunks(N, (N + R) * 32 * 2 * wf):
                ref, ab = contract("nm,meh->neh", bgo[zb(b), o, row0:row0 + R], dp[b, :, es])
                bV.add(v[b, o, :, es], ref, ab)
    res["BWD_V"] = bV

    acc = torch.zeros(Ko, Kd, C, H, dtype=torch.float64, device=X.device)
    aab = torch.zeros_like(acc)
    for b in range(B):
        for ns in _chunks(R, 2 * (Ko + Kd) * N * 32 * wf):
            ref, ab = contract("dnel,oneh->odlh", r["z"][b, :, ns], v[b, :, ns])
            acc += ref
            aab += ab
    res["BWD_DW"] = Bound(B * R * N, False).add(r["dW"].view(Ko, Kd, C, H), acc * invS, aab * invS)

    bY = Bound(H * Ko, fp16)
    for b in range(B):
        for ns in _chunks(R, 2 * (Ko + Kd) * N * 32 * wf):
            ref, ab = contract("oneh,dohl->dnel", v[b, :, ns], wq)
            bY.add(y[b, :, ns], ref, ab)
    res["BWD_MIX"] = bY

    bX = Bound(Kd * N, False)
    for b in range(B):
        for ns in _chunks(R, 2 * Kd * N * 32 * wf):
            ref, ab = contract("dnel,dce->ncl", y[b, :, ns], bgd[zb(b)])
            bX.add(r["dX"][b, ns], ref * invS, ab * invS)
    res["BWD_DX"] = bX
    if not part:      # the max|dX| hint: exact on the tensor cores, 0 ("unknown") from the fp32 kernels
        assert float(r["dx_amax"][0]) == (float(r["dX"].abs().max()) if fp16 else 0.0), "dX_absmax hint"
    return res


def check_stages_wide(r, X, Go, Gd, W, bias, d_out, dyn, kind, row0=None, prec=1):
    """test_gpu_engine_stages.check_stages at any width, for a whole layer or a part (row0 set), for either kernel family: every
    stage of run_layer_wide's result against float64."""
    res = forward_stages(r, X, Go, Gd, W, bias, dyn, kind, row0, prec)
    if d_out is not None:
        res.update(backward_stages(r, X, Go, Gd, W, d_out, dyn, row0, prec))
    return res


def _make_cases():
    rows = []          # (C, H, N, K, B, dyn, kind, grad)
    shapes = ([(C, H, 130, 3, 2, None) for C, H in ((64, 64), (32, 64), (64, 32), (96, 128), (128, 128))]
              + [(64, 64, 130, K, 2, None) for K in (1, 9)]             # K = 9: 18 mix output planes in three groups
              + [(64, 64, N, 3, 2, None) for N in (1, 65, 257)]         # tile edges
              + [(32, 64, 65, 1, 2, None),                              # backward mix: 2 input planes in one k-block
                 (64, 32, 65, 1, 2, None),                              # forward mix: the same
                 (96, 128, 257, 1, 1, None),                            # 3 input planes in one k-block
                 (128, 128, 1, 3, 2, None)]
              + [(96, 128, 65, 9, 2, False),                            # 27 -> 36 planes: five mix groups, 7 x 5 dW tiles, W streamed
                 (128, 128, 130, 9, 1, True),
                 (64, 64, 257, 9, 3, True)])                            # odd batch
    for i, (C, H, N, K, B, only) in enumerate(shapes):
        for dyn in ((False, True) if only is None else (only,)):
            kind = "diag" if (i + dyn) % 2 == 0 else "dense"
            grad = 1e4 if (i + 2 * dyn) % 3 == 1 else 1e-5
            rows.append((C, H, N, K, B, dyn, kind, grad))
    return rows


CASES = _make_cases()


def test_stage_cases_cover_every_width_k_n_kind_and_scale():
    assert {(c[0], c[1]) for c in CASES} == {(64, 64), (32, 64), (64, 32), (96, 128), (128, 128)}
    assert {c[3] for c in CASES} == {1, 3, 9} and {c[2] for c in CASES} >= {1, 65, 130, 257}
    assert {c[5] for c in CASES} == {False, True} and {c[6] for c in CASES} == {"diag", "dense"} and {c[7] for c in CASES} == {1e-5, 1e4}
    for C, H in {(c[0], c[1]) for c in CASES}:
        rows = [c for c in CASES if (c[0], c[1]) == (C, H)]
        assert {c[5] for c in rows} == {False, True}, (C, H)


def _inputs(C, H, N, K, B, dyn, kind, seed, dev):
    rng = np.random.default_rng(seed)
    nz = B if dyn else 1
    mk = (lambda: diag_supports(rng, nz * K, N)) if kind == "diag" else (lambda: dense_supports(rng, nz * K, N))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    X = t(np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32))
    Gd = t(mk().reshape((B, K, N, N) if dyn else (K, N, N)))
    Go = t(mk().reshape((B, K, N, N))) if dyn else Gd
    W = t((rng.standard_normal((K * K * C, H)) * (2.0 / (K * K * C + H)) ** 0.5).astype(np.float32))
    bias = t((rng.standard_normal(H) * 0.1).astype(np.float32))
    return X, Go, Gd, W, bias


@pytest.mark.gpu
@pytest.mark.parametrize("C,H,N,K,B,dyn,kind,grad", CASES)
def test_every_stage_matches_float64_at_wide_channels(C, H, N, K, B, dyn, kind, grad, cuda_device):
    X, Go, Gd, W, bias = _inputs(C, H, N, K, B, dyn, kind, 7919 * N + 31 * K + 2 * B + dyn + 3 * C + 5 * H, cuda_device)
    d_out = torch.randn(B, N, N, H, device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(N + K + C + H)) * grad
    r = run_layer_wide(X, Go, Gd, W, bias, d_out, dyn)
    tag = f"C={C} H={H} N={N} K={K} B={B} {'dyn' if dyn else 'static'}/{kind} |dOut|~{grad:g}"
    _assert_and_record(check_stages_wide(r, X, Go, Gd, W, bias, d_out, dyn, kind), tag)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: end to end
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("wide_bdgcn_"))
def test_layer_matches_reference_fixture_at_wide_channels(name, cuda_device):
    g = layer_fixture(load_golden(name))
    X, G, W, b, d_out = g["X"], _graph(g), g["W"], g["b"], g["d_out"]
    for prec in ("fp32", "fp16"):
        out, dX, dW, db = at_size._run_layer(X, G, W, b, d_out, prec, cuda_device)
        _rel_check(out, g["out"], FWD_TOL[prec], f"{name}/{prec}/out vs reference")
        if prec == "fp32":
            for a, k in ((dX, "dX"), (dW, "dW"), (db, "db")):
                _rel_check(a, g[k], BWD_TOL[prec], f"{name}/{prec}/{k} vs reference")
        else:
            f64 = lambda a: a.astype(np.float64)
            refs = orc.bdgcn_backward_factored(f64(X), tuple(f64(a) for a in G) if isinstance(G, tuple) else f64(G), f64(W), f64(b), "relu",
                                               f64(d_out), mask_from=out)[1:]
            for a, ref, k in zip((dX, dW, db), refs, ("dX", "dW", "db")):
                _rel_check(a, ref, BWD_TOL[prec], f"{name}/{prec}/{k} (engine mask)")
                _rel_check(a, g[k], LOOSE_FP16_GRAD, f"{name}/{prec}/{k} vs reference", l2_only=True)


@pytest.mark.gpu
@pytest.mark.parametrize("N,dyn,kind", [(500, False, "rw"), (1000, True, "dense")])
def test_layer_matches_oracle_at_size_at_64_channels(N, dyn, kind, cuda_device):
    """test_gpu_at_size.test_layer_matches_oracle_at_size at C = H = 64, K = 3, B = 1: forward <= 1e-3 and every gradient <= 2e-3
    against the factored oracle on the engine's ReLU mask, both kernel families."""
    K, B, C = 3, 1, 64
    rng = np.random.default_rng(1000 * N + 64 + dyn)
    X = np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32)
    G = (at_size._supports(rng, kind, K, N, B), at_size._supports(rng, kind, K, N, B)) if dyn else at_size._supports(rng, kind, K, N, 0)
    W = (rng.standard_normal((K * K * C, C)) * (2.0 / (K * K * C + C)) ** 0.5).astype(np.float32)
    b = (rng.standard_normal(C) * 0.1).astype(np.float32)
    d_out = (rng.standard_normal((B, N, N, C)) * 1e-5).astype(np.float32)
    out_o = orc.bdgcn_backward_factored(X, G, W, b, "relu", d_out)[0]
    tag = f"layer C=H=64 N={N} K={K} {'dyn' if dyn else 'static'}/{kind}"
    for prec in ("fp32", "fp16"):
        out, dX, dW, db = at_size._run_layer(X, G, W, b, d_out, prec, cuda_device)
        _rel_check(out, out_o, FWD_TOL[prec], f"{tag}/{prec}/out vs oracle")
        refs = orc.bdgcn_backward_factored(X, G, W, b, "relu", d_out, mask_from=out)[1:]
        for a, r, what in zip((dX, dW, db), refs, ("dX", "dW", "db")):
            _rel_check(a, r, BWD_TOL[prec], f"{tag}/{prec}/{what} (engine mask)")


def _model(N, K, hid, seed, dev):
    torch.manual_seed(seed)
    return shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3, num_nodes=N,
                      user_bias=True, activation=nn.ReLU).to(dev)


def _set_layer_precision(model, prec):
    """BDGCN layers on `prec`; the LSTM on its fp32 kernels (the tensor-core LSTM is hidden-32 only)."""
    model.lstm_precision = "fp32"
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = prec


def _run_model(model, x_seq, G_list, d_y, prec):
    _set_layer_precision(model, prec)
    model.zero_grad(set_to_none=True)
    y = model(x_seq=x_seq, G_list=G_list)
    y.backward(d_y)
    torch.cuda.synchronize()
    return y.detach().clone(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("wide_mpgcn_"))
def test_model_at_hidden_64_matches_reference_fixture(name, cuda_device):
    """The whole model at hidden 64 (every BDGCN layer is 64 -> 64) against the reference: fp32 layers to 5e-5 / 2e-4 (as
    test_gpu_parity.py; BDGCN W gradients on the fixture's rows and in norm); fp16 layers to 1e-3 in rel_L2 forward (its
    rel_Linf recorded) and to 5e-3 in rel_L2 against the oracle's gradients on the engine's ReLU masks."""
    g = load_golden(name)
    K, hid = int(g["K"]), int(g["hidden"])
    N = g["x_seq"].shape[2]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    G_list = [t(g["G_static"]), (t(g["G_o"]), t(g["G_d"]))]
    params = _model_params(g)
    for prec in ("fp32", "fp16"):
        model = _model(N, K, hid, 0, "cpu")
        model.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
        model = model.to(cuda_device)
        caps = {m: {"layers": [], "fc": None} for m in range(2)}
        hooks = [layer.register_forward_hook(lambda mod, inp, out, m=m: caps[m]["layers"].append(out.detach().cpu().numpy()))
                 for m in range(2) for layer in model.branch_models[m]['spatial']]
        y, grads = _run_model(model, t(g["x_seq"]), G_list, t(g["d_y"]), prec)
        for h in hooks:
            h.remove()
        if prec == "fp32":
            _rel_check(y, g["y"], 5e-5, f"{name}/{prec}/y")
            _check_model_grads(grads, g, 2e-4, f"{name}/{prec}")
        else:
            _rel_check(y, g["y"], FWD_TOL[prec], f"{name}/{prec}/y", l2_only=True)
            for m in range(2):
                fc = model.branch_models[m]['fc'][0]
                caps[m]["fc"] = orc.fc_relu_forward(caps[m]["layers"][-1], fc.weight.detach().cpu().numpy(), fc.bias.detach().cpu().numpy())
            _, grads_m = orc.mpgcn_forward_backward(params, g["x_seq"], [g["G_static"], (g["G_o"], g["G_d"])], M=2, gcn_num_layers=3,
                                                    d_y=g["d_y"], masks=caps)
            for k, v in grads.items():
                _rel_check(v, grads_m[k], 5e-3, f"{name}/{prec}/grad:{k} (engine masks)", l2_only=True)


@pytest.mark.gpu
def test_model_at_hidden_64_fp16_matches_fp32(cuda_device):
    """The whole model at hidden 64, N = 60, K = 3, static and dynamic graphs: the tensor-core layers against the fp32 layers.
    The forward is bounded in rel_L2 (1e-3) and its rel_Linf recorded, as in test_gpu_many_supports.py; gradients to 8e-2 in
    rel_L2 (another forward's ReLU mask).  The first seed whose fp32 run gives every parameter a gradient is used."""
    dev = cuda_device
    N, T, B, K = 60, 4, 2, 3
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    for seed in range(64, 2000, 100):
        rng = np.random.default_rng(seed)
        G_list = [t(at_size._supports(rng, "rw", K, N, 0)), (t(at_size._supports(rng, "rw", K, N, B)), t(at_size._supports(rng, "rw", K, N, B)))]
        model = _model(N, K, 64, seed, dev)
        x_seq = t((rng.random((B, T, N, N, 1)) * 8).astype(np.float32))
        d_y = t(rng.standard_normal((B, 1, N, N, 1)).astype(np.float32))
        y32, g32 = _run_model(model, x_seq, G_list, d_y, "fp32")
        if all(float(g.abs().max()) > 0 for g in g32.values()):
            break
    else:
        pytest.fail("no seed gives both branches a gradient")
    y16, g16 = _run_model(model, x_seq, G_list, d_y, "fp16")
    _rel_check(y16, y32, FWD_TOL["fp16"], f"model hidden 64 (seed {seed}): fp16 y vs fp32", l2_only=True)
    for k, g in g32.items():
        _rel_check(g16[k], g, LOOSE_FP16_GRAD, f"model hidden 64: fp16 grad:{k} vs fp32", l2_only=True)


@pytest.mark.gpu
def test_model_at_hidden_64_no_grad_allocates_no_stash_and_graph_rollout_equals_eager(cuda_device):
    """Under torch.no_grad() the hidden-64 model keeps no Z stash (nor any other training state); the CUDA-graph rollout of
    Model_Trainer.test's loop equals the eager loop bitwise."""
    from mpgcn_b200 import rollout
    dev = cuda_device
    N, K, B, T, P = 47, 3, 2, 5, 3
    model = _model(N, K, 64, 3, dev)
    _set_layer_precision(model, "auto")
    assert ops.resolve_precision("auto", B, N, K, 64, 64) == _lib.PREC_FP16_TC
    G = torch.rand(K, N, N, device=dev) / N
    dyn = (torch.rand(B, K, N, N, device=dev) / N, torch.rand(B, K, N, N, device=dev) / N)
    x = torch.rand(B, T, N, N, 1, device=dev) * 8
    ops.STASH_BYTES.clear()
    with torch.no_grad():
        y0 = model(x_seq=x, G_list=[G, dyn])
    assert sum(ops.STASH_BYTES.values()) == 0, dict(ops.STASH_BYTES)
    y1 = model(x_seq=x, G_list=[G, dyn])
    assert ops.STASH_BYTES["bdgcn"] > 0 and torch.equal(y0, y1.detach())
    eager = rollout.forecast(model, x, [G, dyn], P, use_cuda_graph=False)
    graphed = rollout.forecast(model, x, [G, dyn], P, use_cuda_graph=True)
    assert tuple(graphed.shape) == (B, P, N, N, 1)
    assert torch.equal(eager, graphed)


@pytest.mark.gpu
@pytest.mark.parametrize("N,dyn", [(130, False), (258, True)])
def test_row_shard_at_64_channels_sums_to_the_whole_layer(N, dyn, cuda_device):
    """Row shard over 2 ranks at C = H = 64 on supports whose diagonal remainders fire: the fp16 partial pre-activations summed
    equal the fp16 whole layer to 1e-5 (as test_gpu_shard.py at 32 channels)."""
    dev = cuda_device
    rng = np.random.default_rng(N + 64)
    B, K, C, world = 2, 3, 64, 2
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    X = t(np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32))
    shape = (B, K, N, N) if dyn else (K, N, N)
    Gd = t(diag_supports(rng, (B if dyn else 1) * K, N).reshape(shape))
    Go = t(diag_supports(rng, B * K, N).reshape(shape)) if dyn else Gd
    W = t((rng.standard_normal((K * K * C, C)) * (2.0 / (K * K * C + C)) ** 0.5).astype(np.float32))
    assert ops.resolve_precision("auto", B, N, K, C, C) == _lib.PREC_FP16_TC
    cuda = shard.CudaEngine()
    total = torch.zeros(B, N, N, C, dtype=torch.float64, device=dev)
    for r in range(world):
        plan = shard.ShardPlan("row", r, world, N, K)
        pre, _ = cuda.forward_part(X[:, plan.row_lo:plan.row_hi].contiguous(), Go, Gd, dyn, W, N, plan.row_lo, K, K, 1, False)
        total += pre.double()
    whole, _ = abi.forward(X, Go, Gd, W, torch.zeros(C, device=dev), False, "fp16", want_saved=False)
    _rel_check(total, whole.double(), 1e-5, f"row shard C=H=64 N={N} x{world} {'dyn' if dyn else 'static'}/diag fp16: sum of partials == whole")
