"""The support-gradient stages of one BDGCN layer (`mpgcn_bdgcn_backward_supports`), checked in isolation against float64 in both
kernel families.

One whole layer runs through the C ABI (forward, then the backward with dG_o / dG_d, ReLU) into buffers prefilled with NaN
bytes; every intermediate is read back from the workspaces and each stage is recomputed in float64 from the operands THAT stage
read, with the bounds of test_gpu_engine_stages.py (EPS_C * 2^-24 sqrt(L) |A|.|B| per element):

    BWD_DGO  dG_o[n,m] = (1/S) sum_{e,h} U16[o,n,e,h] dP16[m,e,h]        L = N H      (static: summed over b, L = B N H)
    BWD_DGD  dG_d[c,e] = (1/S) sum_{n,l} X16[n,c,l] Y16[d,n,e,l]         L = N C
    static   dG = dG_o + dG_d, one gradient                             L = B N (H + C)

The fp32 family is the same algebra on the fp32 operands (dPre, U, Y, X) with S = 1.  U16 and X16 are formed again by the
backward (from the Z stash and from X): on the tensor cores they must be bitwise the forward's, or dG_o would be the gradient of
another function.  A call with one side of a dynamic pair gives that side bitwise as the call with both.  Shapes are chosen for
the tile edges of BWD_DGO / BWD_DGD: a dG row is tiled in 32-column chunks, at most 8 per tile, so N = 257 and 300 end in a
column tile with 1 and 2 valid chunks, N = 129 in an m-tile with one row, N = 31 / 33 around one chunk.

`test_support_grad_detectors_*` (no GPU) feeds the bound simulated outputs to show that it accepts an fp32-accumulated result and
rejects each defect it is meant to find.
"""
import ctypes

import numpy as np
import pytest
import torch

from test_gpu_channel_widths import (Layout, backward_stages, f32, h16, run_layer_wide, simt_backward_views, simt_ws_layout,
                                     tc_backward_views, u16_view, w16_view, ws_layout)
from test_gpu_engine_stages import (Bound, _assert_and_record, _chunks, _garbage, _simulated, bits, contract, dense_supports,
                                    diag_supports, expected_scale, f16_sat)

from mpgcn_b200 import _lib

KINDS = ("diag", "dense", "rw", "cheb", "drw")       # rw / cheb / drw: Adj_Processor random walk, Chebyshev, dual random walk
ADJ = {"rw": "random_walk_diffusion", "cheb": "chebyshev", "drw": "dual_random_walk_diffusion"}
GRADS = (1e-5, 1e4, 0.0)


def bits32(t):
    return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------------------------------------
# float64 references (device-agnostic)
# ------------------------------------------------------------------------------------------------------------------------------
def dgo_ref(u, dp):
    """dG_o[n,m] = sum_{e,h} u[n,e,h] dp[m,e,h] of one sample and support -> (float64 product, |A|.|B|)"""
    N, M = u.shape[0], dp.shape[0]
    dp = dp.double()
    ref = torch.zeros(N, M, dtype=torch.float64, device=u.device)
    ab = torch.zeros_like(ref)
    for ns in _chunks(N, u[0].numel() + M):
        ref[ns], ab[ns] = contract("neh,meh->nm", u[ns], dp)
    return ref, ab


def dgd_ref(x, y):
    """dG_d[c,e] = sum_{n,l} x[n,c,l] y[n,e,l] of one sample and support -> (float64 product, |A|.|B|)"""
    ref = torch.zeros(x.shape[1], y.shape[1], dtype=torch.float64, device=x.device)
    ab = torch.zeros_like(ref)
    for ns in _chunks(x.shape[0], x[0].numel() + y[0].numel()):
        r, a = contract("ncl,nel->ce", x[ns], y[ns])
        ref += r
        ab += a
    return ref, ab


def dg_max_slices(N, sms):
    """Split-K slices of the dG partials (bdgcn_tc.cu dg_max_slices): ceil(N/128) m-tiles x column tiles of up to 8 chunks"""
    chunks = -(-N // 32)
    return max(1, sms // (-(-N // 128) * -(-chunks // min(chunks, 8))))


def sgrad_ws_layout(B, N, K, C, H, dyn, prec, sms):
    """The support-gradient workspace (tensor cores: bdgcn_tc.cu bwd_layout(s, true); fp32: bdgcn_simt.cu simt_bwd_layout(s, true))
    -> (its Layout, the backward's Layout it begins with).  Tensor cores: the backward's regions, X16, U16, the fp16 W split and the fp32 partials
    [slice][N][32 ceil(N/32)], 1024-aligned; fp32: the backward's regions, then U, 256-aligned (the size adds 1024 + 256)."""
    if prec == 1:
        _, bo = ws_layout(B, N, K, C, H, dyn, sms)
        chunks = -(-N // 32)
        extra = [("x16", B * N * N * C * 2), ("u16", B * K * N * N * H * 2), ("w16", 2 * K * K * C * H * 2),
                 ("partials", dg_max_slices(N, sms) * N * 32 * chunks * 4)]
        return Layout([(n, bo.size[n]) for n in bo] + extra), bo
    _, bo = simt_ws_layout(B, N, C, H, N, K, K)
    return Layout([(n, bo.size[n]) for n in bo] + [("u", B * K * N * N * H * 4)], 256, 1024 + 256), bo


# ------------------------------------------------------------------------------------------------------------------------------
# one layer through the C ABI
# ------------------------------------------------------------------------------------------------------------------------------
def run_support_grads(r, X, Go, Gd, W, d_out, dyn, prec, want_o=True, want_d=True):
    """mpgcn_bdgcn_backward_supports after run_layer_wide's forward `r` (ReLU), every output prefilled with NaN bytes.  want_o /
    want_d: which side of a dynamic pair gets its gradient (a static stack has one, in dG_o).  -> r's forward views plus the
    backward's (tc_backward_views / simt_backward_views), dX, dW, db, dG_o / dG_d (None if not asked for), and the support-grad
    region: sx16, su [B][o][n][e][H], sw16 [2][o][d][C][H] (tensor cores) / su (fp32)."""
    lib = _lib.load()
    dev = X.device
    B, N, _, C = X.shape
    K, H = Go.shape[-3], W.shape[1]
    nz = B if dyn else 1
    n_ws = lib.mpgcn_bdgcn_support_grad_workspace_bytes(B, N, K, C, H, int(dyn), prec)
    lay, bo = sgrad_ws_layout(B, N, K, C, H, dyn, prec, torch.cuda.get_device_properties(dev).multi_processor_count)
    assert lay.total == n_ws, f"support-grad workspace layout {lay.total} != library size {n_ws}"
    f32buf = lambda n: _garbage(4 * n, dev).view(torch.float32)
    wsb = _garbage(n_ws, dev)
    dX, dW, db, dx_amax = f32buf(B * N * N * C).view(B, N, N, C), f32buf(W.numel()).view_as(W), f32buf(H), f32buf(1)
    send_o, send_d = want_o or not dyn, want_d and dyn
    dgo_b, dgd_b = (_garbage(4 * nz * K * N * N, dev) if send else None for send in (send_o, send_d))
    ex = _lib.BdgcnExtras()
    ex.dX_absmax = dx_amax.data_ptr()
    _lib.check(lib.mpgcn_bdgcn_backward_supports(d_out.data_ptr(), r["out"].data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn), W.data_ptr(),
                                                 1, r["bufs"]["saved"].data_ptr(), dX.data_ptr(), dW.data_ptr(), db.data_ptr(), wsb.data_ptr(),
                                                 n_ws, B, N, K, C, H, prec, ctypes.addressof(ex), X.data_ptr(),
                                                 dgo_b.data_ptr() if send_o else None, dgd_b.data_ptr() if send_d else None,
                                                 torch.cuda.current_stream().cuda_stream), "backward_supports")
    torch.cuda.synchronize()
    s = dict(r)
    shape = (B, K, N, N) if dyn else (K, N, N)
    s.update(dX=dX, dW=dW, db=db, dx_amax=dx_amax, dGo=dgo_b.view(torch.float32).view(shape) if send_o else None,
             dGd=dgd_b.view(torch.float32).view(shape) if send_d else None)
    if prec == 1:
        s.update(tc_backward_views(wsb, bo, B, N, N, C, H, K, K, nz, r["own_go"]))
        s.update(sx16=h16(wsb, lay["x16"], B, N, N, C), su=u16_view(wsb, lay["u16"], B, K, N, N, H), sw16=w16_view(wsb, lay["w16"], K, K, C, H))
    else:
        s.update(simt_backward_views(wsb, bo, B, N, N, C, H, K, K, False))
        s["su"] = f32(wsb, lay["u"], B, K, N, N, H)
    return s


def check_recomputed_operands(s, X, dyn, prec, want_o=True, want_d=True):
    """The operands the support-grad call formed again are the forward's: X16 (dG_d) and the W16 split and U16 (dG_o) bitwise on the
    tensor cores; U bitwise on the fp32 kernels (the same SGEMM as the forward's)."""
    if prec == 1:
        if want_d or not dyn:
            assert torch.equal(bits(s["sx16"]), bits(f16_sat(X))), "support-grad X16 != fp16_sat(X)"
            assert torch.equal(bits(s["sx16"]), bits(s["x16"])), "support-grad X16 != the forward's X16"
        if want_o or not dyn:
            assert torch.equal(bits(s["sw16"]), bits(s["w16"])), "support-grad W16 hi / lo != the forward's"
            assert torch.equal(bits(s["su"]), bits(s["u"])), "support-grad U16 != the forward's U16 (FWD_MIX of the Z stash)"
    elif want_o or not dyn:
        assert torch.equal(bits32(s["su"]), bits32(s["u"])), "support-grad U != the forward's U"


def support_grad_stages(s, X, W, dyn, prec):
    """The support-gradient stages of run_support_grads' result (both sides) against float64 -> {stage: Bound}; the recomputed
    operands are checked on the way."""
    B, N, _, C = X.shape
    K, H = s["su"].shape[1], W.shape[1]
    check_recomputed_operands(s, X, dyn, prec)
    res = {}
    if prec == 1:
        invS, dp, x = float(s["scale"][1]), s["dp"], s["sx16"]
    else:
        invS, dp, x = 1.0, s["dpre"], X
        bU = Bound(K * C, False)
        W4 = W.view(K, K, C, H)
        for b in range(B):
            for ns in _chunks(N, 2 * K * N * (C + H)):
                ref, ab = contract("dnel,odlh->oneh", s["z"][b, :, ns], W4)
                bU.add(s["su"][b, :, ns], ref, ab)
        res["BWD_DG U = sum_d Z_d W[o,d]"] = bU
    u, y = s["su"], s["y"]
    if not dyn:
        bS = Bound(B * N * (H + C), False)
        for k in range(K):
            ref = torch.zeros(N, N, dtype=torch.float64, device=X.device)
            ab = torch.zeros_like(ref)
            for b in range(B):
                for r_, a_ in (dgo_ref(u[b, k], dp[b]), dgd_ref(x[b], y[b, k])):
                    ref += r_
                    ab += a_
            bS.add(s["dGo"][k], ref * invS, ab * invS)
        res["BWD_DGO + BWD_DGD (static)"] = bS
        return res
    bO, bD = Bound(N * H, False), Bound(N * C, False)
    for b in range(B):
        for k in range(K):
            ref, ab = dgo_ref(u[b, k], dp[b])
            bO.add(s["dGo"][b, k], ref * invS, ab * invS)
            ref, ab = dgd_ref(x[b], y[b, k])
            bD.add(s["dGd"][b, k], ref * invS, ab * invS)
    res["BWD_DGO"], res["BWD_DGD"] = bO, bD
    return res


# ------------------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------------------
def _make_cases():
    rows = []          # (C, H, N, K, B, dyn, kind, grad, prec)
    shapes = [(32, 32, N, 3, 2, None) for N in (1, 31, 33, 129, 257)]
    shapes += [(32, 32, 300, 3, 1, None),
               (64, 32, 33, 3, 2, None),
               (32, 96, 129, 1, 3, None),
               (96, 128, 257, 3, 1, None),
               (32, 96, 31, 9, 3, None),
               (128, 128, 300, 9, 1, False),                  # the largest: 2 valid chunks in the last column tile, 9 supports
               (128, 128, 129, 9, 2, True),
               (64, 32, 300, 1, 3, True),
               (32, 32, 257, 9, 2, True)]
    for C, H, N, K, B, only in shapes:
        for dyn in ((False, True) if only is None else (only,)):
            for prec in (1, 0):
                i = len(rows)
                rows.append((C, H, N, K, B, dyn, KINDS[i % len(KINDS)], GRADS[i % len(GRADS)], prec))
    return rows


CASES = _make_cases()


def test_support_grad_stage_cases_cover_every_width_n_k_kind_and_scale():
    widths = {(32, 32), (64, 32), (32, 96), (96, 128), (128, 128)}
    for prec in (1, 0):
        rows = [c for c in CASES if c[8] == prec]
        assert {(c[0], c[1]) for c in rows} == widths
        assert {c[2] for c in rows} == {1, 31, 33, 129, 257, 300} and {c[3] for c in rows} == {1, 3, 9} and {c[4] for c in rows} == {1, 2, 3}
        for dyn in (False, True):
            sub = [c for c in rows if c[5] == dyn]
            assert {c[6] for c in sub} == set(KINDS), (prec, dyn)
            assert {c[7] for c in sub} == set(GRADS), (prec, dyn)
            assert {c[2] for c in sub} >= {129, 257, 300}, (prec, dyn)
        assert {c[3] for c in rows if c[2] >= 257} >= {3, 9}
        for N in (129, 257, 300):          # every tile edge sees a nonzero gradient, static and dynamic
            assert {c[5] for c in rows if c[2] == N and c[7]} == {False, True}, (prec, N)


def _adj_supports(rng, kind, nb, K, N, dev):
    """[nb, K, N, N] supports built on the GPU by Adj_Processor from a random flow (K odd for the dual random walk)."""
    from mpgcn_b200.GCN import Adj_Processor
    order = (K - 1) // 2 if kind == "drw" else K - 1
    flow = torch.from_numpy((rng.random((nb, N, N)) + 0.05).astype(np.float32)).to(dev)
    G = Adj_Processor(ADJ[kind], order, device=dev).process(flow)
    assert G.shape == (nb, K, N, N)
    return G.contiguous()


def _inputs(C, H, N, K, B, dyn, kind, seed, dev):
    rng = np.random.default_rng(seed)
    nz = B if dyn else 1
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    if kind in ADJ:
        mk = lambda: _adj_supports(rng, kind, nz, K, N, dev)
    else:
        mk = lambda: t(diag_supports(rng, nz * K, N) if kind == "diag" else dense_supports(rng, nz * K, N))
    X = t(np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32))
    Gd = mk().reshape((B, K, N, N) if dyn else (K, N, N)).contiguous()
    Go = mk().reshape((B, K, N, N)).contiguous() if dyn else Gd
    W = t((rng.standard_normal((K * K * C, H)) * (2.0 / (K * K * C + H)) ** 0.5).astype(np.float32))
    bias = t((rng.standard_normal(H) * 0.1).astype(np.float32))
    return X, Go, Gd, W, bias


@pytest.mark.gpu
@pytest.mark.parametrize("C,H,N,K,B,dyn,kind,grad,prec", CASES)
def test_support_grad_stages_match_float64(C, H, N, K, B, dyn, kind, grad, prec, cuda_device):
    X, Go, Gd, W, bias = _inputs(C, H, N, K, B, dyn, kind, 7919 * N + 31 * K + 2 * B + dyn + 3 * C + 5 * H + KINDS.index(kind), cuda_device)
    gen = torch.Generator(cuda_device).manual_seed(N + K + C + H)
    d_out = torch.randn(B, N, N, H, device=cuda_device, generator=gen) * grad if grad else torch.zeros(B, N, N, H, device=cuda_device)
    r = run_layer_wide(X, Go, Gd, W, bias, None, dyn, prec=prec)
    s = run_support_grads(r, X, Go, Gd, W, d_out, dyn, prec)
    tag = f"sgrad {'fp16' if prec == 1 else 'fp32'} C={C} H={H} N={N} K={K} B={B} {'dyn' if dyn else 'static'}/{kind} |dOut|~{grad:g}"
    res = backward_stages(s, X, Go, Gd, W, d_out, dyn, prec=prec)
    res.update(support_grad_stages(s, X, W, dyn, prec))
    if grad == 0:
        assert prec == 0 or (float(s["scale"][0]), float(s["scale"][1])) == (1.0, 1.0)
        for g in (s["dGo"], s["dGd"]):
            assert g is None or not bits32(g).any(), "dG must be exactly +0 for a zero dOut"
    if dyn:       # one side of the pair at a time: that side, dX (and on the tensor cores dW) bitwise as with both
        for want_o, want_d, side in ((True, False, "dGo"), (False, True, "dGd")):
            one = run_support_grads(r, X, Go, Gd, W, d_out, dyn, prec, want_o, want_d)
            assert torch.equal(bits32(one[side]), bits32(s[side])), f"{side} alone != {side} with both sides"
            assert torch.equal(bits32(one["dX"]), bits32(s["dX"])), f"dX of the {side}-only call"
            # dW only on the tensor cores: its split-K partials are reduced in a fixed order there, while the fp32 BWD_DW adds its
            # ksplit = RN / 2048 slices with atomics, in an order that changes from run to run (bdgcn_simt.cu)
            if prec == 1:
                assert torch.equal(bits32(one["dW"]), bits32(s["dW"])), f"dW of the {side}-only call"
            check_recomputed_operands(one, X, dyn, prec, want_o, want_d)
    _assert_and_record(res, tag)


# ------------------------------------------------------------------------------------------------------------------------------
# the detector detects (CPU)
# ------------------------------------------------------------------------------------------------------------------------------
def test_support_grad_detectors_accept_a_faithful_kernel_and_reject_each_defect():
    gen = torch.Generator().manual_seed(1)
    B, K, N, C, H = 2, 2, 40, 32, 64           # N = 40: a second 32-column chunk with 8 valid columns; H = 64: two hc segments
    S, invS = expected_scale(1e-5 * 4.5)
    assert S > 1
    u = f16_sat(torch.randn(B, K, N, N, H, generator=gen) * 0.3)
    dp = f16_sat(torch.randn(B, N, N, H, generator=gen).clamp(-4.5, 4.5) * 1e-5 * S)
    x = f16_sat(torch.tanh(torch.randn(B, N, N, C, generator=gen)))
    y = f16_sat(torch.randn(B, K, N, N, C, generator=gen))
    sim = lambda ref, ab: _simulated(ref * invS, ab * invS, gen, fp16=False)
    bound = lambda L, got, ref, ab: Bound(L, False).add(got, ref * invS, ab * invS)

    # dynamic BWD_DGO / BWD_DGD: faithful passes; a dropped hc segment, a missing or doubled 1/S, a transposed result and a last
    # partial column chunk left at zero fail
    ro, ao = dgo_ref(u[0, 1], dp[0])
    rd, ad = dgd_ref(x[0], y[0, 1])
    for L, ref, ab in ((N * H, ro, ao), (N * C, rd, ad)):
        assert bound(L, sim(ref, ab), ref, ab).ok
        assert not bound(L, sim(ref, ab) * S, ref, ab).ok, "missing 1/S"
        assert not bound(L, sim(ref, ab) * 2, ref, ab).ok, "1/S off by 2x"
        assert not bound(L, sim(ref, ab).T.contiguous(), ref, ab).ok, "transposed"
        cut = sim(ref, ab).clone()
        cut[:, 32:] = 0
        assert not bound(L, cut, ref, ab).ok, "last partial column chunk left at zero"
    u_seg = u[0, 1].clone()
    u_seg[..., 32:] = 0
    r_seg, a_seg = dgo_ref(u_seg, dp[0])
    assert not bound(N * H, sim(r_seg, a_seg), ro, ao).ok, "one hc segment's k-blocks dropped"

    # static: one gradient, sum over the batch of both terms; a dropped sample and dG_d written over dG_o fail
    def static_terms(bs):
        ref = torch.zeros(N, N, dtype=torch.float64)
        ab, rds = torch.zeros_like(ref), torch.zeros_like(ref)
        for b in bs:
            r1, a1 = dgo_ref(u[b, 0], dp[b])
            r2, a2 = dgd_ref(x[b], y[b, 0])
            ref, ab, rds = ref + r1 + r2, ab + a1 + a2, rds + r2
        return ref, ab, rds
    ref, ab, rds = static_terms(range(B))
    L = B * N * (H + C)
    assert bound(L, sim(ref, ab), ref, ab).ok
    r0, a0, _ = static_terms([0])
    assert not bound(L, sim(r0, a0), ref, ab).ok, "one sample's k-blocks dropped"
    assert not bound(L, sim(rds, ab), ref, ab).ok, "static dG_d written instead of accumulated"
