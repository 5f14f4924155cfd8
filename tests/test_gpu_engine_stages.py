"""Every tensor-core contraction of one BDGCN layer (precision 1), checked in isolation against float64.

One whole-layer forward and backward runs through the C ABI; every intermediate is then read back from the workspaces
(`mpgcn_debug_tc_workspace_offset`) and each stage is recomputed in float64 on the GPU with torch from the fp16 operands THAT
stage read, so an error is pinned to the stage that made it.  Conversions must be bit-exact; contractions must satisfy, element
by element, with |A|.|B| the same contraction on absolute values (L terms):

    fp16 output:  |y - r| <= 2^-11 |r| + 2^-25 + EPS_C * 2^-24 * sqrt(L) * (|A|.|B|)      (rounding of the store, subnormal floor)
    fp32 output:  |y - r| <=                     EPS_C * 2^-24 * sqrt(L) * (|A|.|B|)

The last term is the fp32 accumulation of the tensor cores and the epilogues.  EPS_C = 8: on an H100 the largest measured
coefficient over every case below is reported in `parity_report.json` ("stages ... coef") and stays below 1 (a correctly
rounded sequential fp32 sum of random-sign terms has a coefficient of about 1); 8 leaves room for other data while a dropped
k-block, a wrong operand map or a gradient scale off by a power of two is larger by orders of magnitude.
The fp16 rounding of Z16 / U16 is larger than the support-diagonal remainder correction and the fp16 `lo` half of W, so those
two are checked statistically: the regression slope of the kernel's deviation from the product without them on the term
they contribute must be 1 (0 when the term is missing).

The helpers are plain torch / numpy; `test_detectors_*` (no GPU) feeds them simulated kernel outputs to show that they
accept an fp32-accumulated result and reject each of the defects they are meant to find.
"""
import math

import numpy as np
import pytest
import torch

from conftest import record_parity

HALF_MAX = 65504.0
TAU = 1.0 / 16           # kDiagTau of diag_delta_kernel (simt_kernels.cu)
EPS_C = 8.0
SLOPE_MIN_TERMS = 100000 # below this many correction terms the slope is too noisy to judge (fp16 rounding is the noise)


# ------------------------------------------------------------------------------------------------------------------------------
# checking helpers (device-agnostic)
# ------------------------------------------------------------------------------------------------------------------------------
def f16_sat(x):
    """fp32 -> fp16 as the engine converts: round to nearest even, |x| > 65504 -> +-65504, NaN stays NaN."""
    x = x.float()
    return torch.where(x.abs() > HALF_MAX, torch.copysign(torch.full_like(x, HALF_MAX), x), x).half()


def bits(h):
    return h.contiguous().view(torch.int16)


def hilo(W):
    """fp16 hi / lo split of W: hi = fp16(W), lo = fp16(W - hi) (the difference is exact in fp32)."""
    hi = f16_sat(W)
    return hi, f16_sat(W.float() - hi.float())


def diag_rule(G):
    """Support-diagonal remainders in float64.  G [P,N,N] fp32 (numpy) -> (delta [P,N] float64, near [P,N] bool):
    delta = G_ii - fp16(G_ii) where G_ii^2 > TAU * sum_{c != i} G_ci^2, else 0; `near` marks diagonals within 1e-3 (relative)
    of the threshold, where the kernel's fp32 column sum may decide either way."""
    G = np.asarray(G, np.float32)
    g = np.diagonal(G, axis1=1, axis2=2).astype(np.float64)
    col = (G.astype(np.float64) ** 2).sum(axis=1)
    lhs, rhs = g * g, TAU * (col - g * g)
    fires = lhs > rhs
    g32 = np.array(np.diagonal(G, axis1=1, axis2=2))
    rem = g32.astype(np.float64) - f16_sat(torch.from_numpy(g32)).double().numpy()
    near = np.abs(lhs - rhs) <= 1e-3 * (lhs + np.abs(rhs))
    return np.where(fires, rem, 0.0), near


def diag_supports(rng, planes, N, nnz=6, weak=0.1):
    """[planes,N,N] float32: alpha_i on the diagonal (alpha ~ U[0.6, 1.4], not representable in fp16) plus `nnz` N(0, 0.25^2)
    off-diagonal entries per column.  The diagonal dominates its column (the remainder correction fires) except in a `weak`
    fraction of columns whose alpha ~ U[0.01, 0.05] keeps it below the threshold."""
    G = np.zeros((planes, N, N), np.float32)
    idx = np.arange(N)
    for p in range(planes):
        alpha = rng.uniform(0.6, 1.4, N)
        w = rng.random(N) < weak
        alpha[w] = rng.uniform(0.01, 0.05, int(w.sum()))
        k = min(nnz, N - 1)
        if k:
            rows = (idx[:, None] + rng.integers(1, N, size=(N, k))) % N          # never the diagonal
            G[p][rows, np.repeat(idx[:, None], k, axis=1)] = rng.normal(0.0, 0.25, (N, k))
        G[p][idx, idx] = alpha
    return G


def dense_supports(rng, planes, N):
    return (rng.standard_normal((planes, N, N)) / np.sqrt(N)).astype(np.float32)


def expected_scale(amax):
    """[S, 1/S] of make_scale_kernel: S = 2^k with S * amax in [16, 32), k clamped to [-100, 100]; S = 1 for amax = 0 / inf."""
    if not (0.0 < amax < 3.0e38):
        return 1.0, 1.0
    k = max(-100, min(100, 5 - math.frexp(amax)[1]))
    return 2.0 ** k, 2.0 ** -k


class Bound:
    """Worst element of one stage in units of 2^-24 sqrt(L) (|A|.|B|) (after the fp16 store allowance); passes if <= EPS_C."""

    def __init__(self, L, fp16):
        self.unit = 2.0 ** -24 * math.sqrt(max(L, 1))
        self.fp16 = fp16
        self.coef = 0.0

    def add(self, y, r, ab):
        y, r, ab = y.double(), r.double(), ab.double()
        if self.fp16:
            r = r.clamp(-HALF_MAX, HALF_MAX)
        ex = (y - r).abs()
        if self.fp16:
            ex = ex - (2.0 ** -11 * r.abs() + 2.0 ** -25)
        ex = torch.nan_to_num(ex, nan=math.inf)
        c = torch.where(ex <= 0, torch.zeros_like(ex), ex / (self.unit * ab))
        self.coef = max(self.coef, float(c.max()) if c.numel() else 0.0)
        return self

    @property
    def ok(self):
        return self.coef <= EPS_C


class Slope:
    """Least-squares slope of a deviation on the term it should contain (through the origin), over the nonzero terms."""

    def __init__(self):
        self.sxy = self.sxx = 0.0
        self.n = 0

    def add(self, dev, term):
        dev, term = dev.double(), term.double()
        self.sxy += float((dev * term).sum())
        self.sxx += float((term * term).sum())
        self.n += int(torch.count_nonzero(term))
        return self

    @property
    def value(self):
        return self.sxy / self.sxx if self.sxx > 0 else None

    @property
    def judged(self):
        return self.n >= SLOPE_MIN_TERMS

    @property
    def ok(self):
        return not self.judged or 0.9 <= self.value <= 1.1


# float64 recomputation of each contraction from the operands it read: (product without the checked extra term, extra term, |A|.|B|)
def fwd_a_ref(x, g, delta):
    """Z[n,e,l] = sum_c g[c,e] x[n,c,l] + delta[e] x[n,e,l]      x [n,c,l], g [c,e], delta [e]"""
    x, g, delta = x.double(), g.double(), delta.double()
    base = torch.einsum("ncl,ce->nel", x, g)
    corr = delta[None, :, None] * x
    return base, corr, torch.einsum("ncl,ce->nel", x.abs(), g.abs()) + corr.abs()


def mix_ref(z, hi, lo):
    """U[o,n,e,h] = sum_{d,l} z[d,n,e,l] (hi + lo)[o,d,l,h]"""
    z = z.double()
    return (torch.einsum("dnel,odlh->oneh", z, hi.double()), torch.einsum("dnel,odlh->oneh", z, lo.double()),
            torch.einsum("dnel,odlh->oneh", z.abs(), hi.double().abs() + lo.double().abs()))


def fwd_b_ref(g, u, delta, bias, row0=0):
    """pre[m,e,h] = sum_{o,n} g[o,n,m] u[o,n,e,h] + bias[h] + sum_o delta[o,m] u[o,m-row0,e,h]      u: every row n of the slab of
    origin rows [row0, row0 + R) (the whole layer: R = N), a range of e; g: those rows of G_o; the remainder term only for m in
    the slab; bias None: a raw partial"""
    g, u, delta = g.double(), u.double(), delta.double()
    R = u.shape[1]
    base = torch.einsum("onm,oneh->meh", g, u)
    corr = torch.zeros_like(base)
    corr[row0:row0 + R] = torch.einsum("on,oneh->neh", delta[:, row0:row0 + R], u)
    ab = torch.einsum("onm,oneh->meh", g.abs(), u.abs()) + corr.abs()
    if bias is not None:
        base, ab = base + bias.double(), ab + bias.double().abs()
    return base, corr, ab


def contract(eq, a, b):
    a, b = a.double(), b.double()
    return torch.einsum(eq, a, b), torch.einsum(eq, a.abs(), b.abs())


def _chunks(n, per_item, budget=1 << 24):
    step = max(1, budget // max(1, per_item))
    return [slice(i, min(n, i + step)) for i in range(0, n, step)]


# ------------------------------------------------------------------------------------------------------------------------------
# one layer through the C ABI, workspaces read back
# ------------------------------------------------------------------------------------------------------------------------------
def _garbage(nbytes, dev):
    return torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=dev)      # fp16 NaN / fp32 NaN: unwritten bytes show


def run_layer(X, Go, Gd, W, bias, d_out, dyn):
    """fp16 forward + backward of one layer (ReLU) -> dict of outputs and workspace views."""
    from mpgcn_b200 import _lib
    lib = _lib.load()
    dev = X.device
    B, N, _, C = X.shape
    K, H = Go.shape[-3], W.shape[1]
    nz, Np = (B if dyn else 1), (N + 7) // 8 * 8
    st = torch.cuda.current_stream().cuda_stream
    out = torch.full((B, N, N, H), math.nan, device=dev)
    saved = _garbage(lib.mpgcn_bdgcn_saved_bytes(B, N, K, C, H, 1), dev)
    ws = _garbage(lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, C, H, int(dyn), 1), dev)
    _lib.check(lib.mpgcn_bdgcn_forward(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn), W.data_ptr(), bias.data_ptr(), 1, out.data_ptr(),
                                       saved.data_ptr(), ws.data_ptr(), ws.numel(), B, N, K, C, H, 1, st), "forward")
    r = dict(out=out)
    if d_out is not None:
        dX = torch.full((B, N, N, C), math.nan, device=dev)
        dW = torch.full_like(W, math.nan)
        db = torch.full((H,), math.nan, device=dev)
        dx_amax = torch.full((1,), math.nan, device=dev)
        wsb = _garbage(lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, int(dyn), 1), dev)
        _lib.check(lib.mpgcn_bdgcn_backward_ex(d_out.data_ptr(), out.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn), W.data_ptr(), 1,
                                               saved.data_ptr(), dX.data_ptr(), dW.data_ptr(), db.data_ptr(), wsb.data_ptr(), wsb.numel(),
                                               B, N, K, C, H, 1, None, dx_amax.data_ptr(), st), "backward_ex")
        r.update(dX=dX, dW=dW, db=db, dx_amax=dx_amax)
    torch.cuda.synchronize()
    off = lambda w: lib.mpgcn_debug_tc_workspace_offset(w, B, N, K, int(dyn))

    def h16(buf, w, *shape):
        o = off(w)
        return buf[o:o + 2 * math.prod(shape)].view(torch.float16).view(*shape)

    def f32(buf, w, *shape):
        o = off(w)
        return buf[o:o + 4 * math.prod(shape)].view(torch.float32).view(*shape)

    r.update(x16=h16(ws, 0, B, N, N, 32), gd16=h16(ws, 1, nz, K, N, Np), w16=h16(ws, 3, 2, K, K, 32, 32), u16=h16(ws, 4, B, K, N, N, 32),
             dd=f32(ws, 5, nz, K, N), z16=saved.view(torch.float16).view(B, K, N, N, 32))
    r["go16"], r["dgo"] = (h16(ws, 2, nz, K, N, Np), f32(ws, 6, nz, K, N)) if dyn else (r["gd16"], r["dd"])     # static: one side
    if d_out is not None:
        r.update(dp16=h16(wsb, 10, B, N, N, 32), bgd16=h16(wsb, 11, nz, K, N, Np), v16=h16(wsb, 13, B, K, N, N, 32),
                 y16=h16(wsb, 14, B, K, N, N, 32), wq16=h16(wsb, 15, K, K, 32, 32), scale=f32(wsb, 18, 2))
        r["bgo16"] = h16(wsb, 12, nz, K, N, Np) if dyn else r["bgd16"]
    return r


def _check_support_copy(g16, G, N, what):
    assert torch.equal(bits(g16[..., :N]), bits(f16_sat(G))), f"{what}: fp16 support copy"
    assert not bits(g16[..., N:]).any(), f"{what}: pad columns [N, Np) are not zero"


def check_stages(r, X, Go, Gd, W, bias, d_out, dyn, tag, kind):
    """Every stage of run_layer's result against float64; returns {stage: Bound or Slope}."""
    B, N, _, C = X.shape
    K = Go.shape[-3]
    nz = B if dyn else 1
    Gd4, Go4 = Gd.view(nz, K, N, N), Go.view(nz, K, N, N)
    W4 = W.view(K, K, 32, 32)                               # [o][d][l][h]
    zb = (lambda b: b) if dyn else (lambda b: 0)
    res = {}

    # ---- conversions (bitwise) and the diagonal rule ----
    assert torch.equal(bits(r["x16"]), bits(f16_sat(X))), "x16"
    _check_support_copy(r["gd16"], Gd4, N, "gd16")
    _check_support_copy(r["go16"], Go4, N, "go16")
    hi, lo = hilo(W4)
    assert torch.equal(bits(r["w16"][0]), bits(hi)) and torch.equal(bits(r["w16"][1]), bits(lo)), "w16 hi / lo"
    fired = 0
    for name, G in (("dd", Gd4), ("dgo", Go4)):
        want, near = diag_rule(G.reshape(nz * K, N, N).cpu().numpy())
        got = r[name].reshape(nz * K, N).double().cpu().numpy()
        bad = (got != want) & ~near
        assert not bad.any(), f"{name}: {int(bad.sum())} remainders differ from the tau = 1/16 rule, first at {np.argwhere(bad)[0]}"
        fired = max(fired, int(np.count_nonzero(got)))
    if kind == "diag":
        assert fired >= 0.5 * nz * K * N, f"the inputs were meant to make the remainder correction fire ({fired} of {nz * K * N})"

    x16, gd16, go16 = r["x16"], r["gd16"][..., :N], r["go16"][..., :N]
    dd, dgo, z16, u16, out = r["dd"], r["dgo"], r["z16"], r["u16"], r["out"]

    # ---- FWD_A: Z16 = X16 x2 G_d (+ remainder) ----
    bA, sA = Bound(N, True), Slope()
    for b in range(B):
        for d in range(K):
            for ns in _chunks(N, N * 32):
                base, corr, ab = fwd_a_ref(x16[b, ns], gd16[zb(b), d], dd[zb(b), d])
                y = z16[b, d, ns]
                bA.add(y, base + corr, ab)
                sA.add(y.double() - base, corr)
    res["FWD_A"], res["FWD_A remainder slope"] = bA, sA

    # ---- FWD_MIX: U16 = sum_d Z16_d (hi + lo) ----
    bM, sM = Bound(64 * K, True), Slope()
    for b in range(B):
        for ns in _chunks(N, K * N * 32 * 4):
            base, lpart, ab = mix_ref(z16[b, :, ns], hi, lo)
            y = u16[b, :, ns]
            bM.add(y, base + lpart, ab)
            sM.add(y.double() - base, lpart)
    res["FWD_MIX"], res["FWD_MIX lo slope"] = bM, sM

    # ---- FWD_B: out = relu(sum_o G_o^T U16_o + remainder + b) ----
    bB, sB = Bound(K * N + K + 1, False), Slope()
    for b in range(B):
        for es in _chunks(N, K * N * 32 * 4):
            base, corr, ab = fwd_b_ref(go16[zb(b)], u16[b, :, :, es], dgo[zb(b)], bias)
            y = out[b, :, es]
            bB.add(y, torch.relu(base + corr), ab)
            sB.add(y.double() - base, corr * (y > 0))
    res["FWD_B"], res["FWD_B remainder slope"] = bB, sB
    if d_out is None:
        return res

    # ---- gradient scale, ReLU mask, fp16 dPre, db ----
    amax = float(d_out.abs().max())
    S, invS = expected_scale(amax)
    got = (float(r["scale"][0]), float(r["scale"][1]))
    assert got == (S, invS), f"gradient scale {got} for max|dOut| = {amax:.6e}, want {(S, invS)}"
    if 0 < amax and -100 < 5 - math.frexp(amax)[1] < 100:
        assert 16.0 <= S * amax < 32.0
    d_pre = torch.where(out > 0, d_out, torch.zeros_like(d_out))
    assert torch.equal(bits(r["dp16"]), bits(f16_sat(d_pre * S))), "dp16 != fp16_sat(dOut * [out > 0] * S)"
    ref_db = d_pre.double().sum(dim=(0, 1, 2))
    res["db"] = Bound(B * N * N, False).add(r["db"], ref_db, d_pre.double().abs().sum(dim=(0, 1, 2)))
    _check_support_copy(r["bgd16"], Gd4, N, "backward gd16")
    _check_support_copy(r["bgo16"], Go4, N, "backward go16")
    wq = r["wq16"]
    assert torch.equal(bits(wq), bits(f16_sat(W4.permute(1, 0, 3, 2)))), "wq16 != fp16(W[o][d][l][h]) as [d][o][h][l]"
    dp16, v16, y16 = r["dp16"], r["v16"], r["y16"]
    bgd16, bgo16 = r["bgd16"][..., :N], r["bgo16"][..., :N]

    # ---- BWD_V: V16 = G_o x1 dP16 ----
    bV = Bound(N, True)
    for b in range(B):
        for o in range(K):
            for es in _chunks(N, N * 32 * 2):
                ref, ab = contract("nm,meh->neh", bgo16[zb(b), o], dp16[b, :, es])
                bV.add(v16[b, o, :, es], ref, ab)
    res["BWD_V"] = bV

    # ---- BWD_DW: dW = (sum Z16^T V16) / S ----
    acc = torch.zeros(K, K, 32, 32, dtype=torch.float64, device=X.device)
    aab = torch.zeros_like(acc)
    for b in range(B):
        for ns in _chunks(N, 2 * K * N * 32):
            ref, ab = contract("dnel,oneh->odlh", z16[b, :, ns], v16[b, :, ns])
            acc += ref
            aab += ab
    res["BWD_DW"] = Bound(B * N * N, False).add(r["dW"].view(K, K, 32, 32), acc * invS, aab * invS)

    # ---- BWD_MIX: Y16 = sum_o V16_o Wq ----
    bY = Bound(32 * K, True)
    for b in range(B):
        for ns in _chunks(N, 2 * K * N * 32):
            ref, ab = contract("oneh,dohl->dnel", v16[b, :, ns], wq)
            bY.add(y16[b, :, ns], ref, ab)
    res["BWD_MIX"] = bY

    # ---- BWD_DX: dX = (sum_d Y16_d x2 G_d^T) / S, and its max|dX| hint ----
    bX = Bound(K * N, False)
    for b in range(B):
        for ns in _chunks(N, 2 * K * N * 32):
            ref, ab = contract("dnel,dce->ncl", y16[b, :, ns], bgd16[zb(b)])
            bX.add(r["dX"][b, ns], ref * invS, ab * invS)
    res["BWD_DX"] = bX
    assert float(r["dx_amax"][0]) == float(r["dX"].abs().max()), "dX_absmax hint != max|dX|"
    return res


def _assert_and_record(res, tag):
    bad = []
    for stage, v in res.items():
        if isinstance(v, Bound):
            record_parity(f"stages {tag} {stage}: coef = max err / (2^-24 sqrt(L) |A||B|)", v.coef, v.coef, EPS_C)
            if not v.ok:
                bad.append(f"{stage}: coef {v.coef:.3g} > {EPS_C}")
        elif v.judged:
            record_parity(f"stages {tag} {stage} (n={v.n}): |slope - 1|", abs(v.value - 1), abs(v.value - 1), 0.1)
            if not v.ok:
                bad.append(f"{stage}: slope {v.value:.3f} over {v.n} terms (want 1)")
    assert not bad, f"{tag}: " + "; ".join(bad)


# ------------------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------------------
def _make_cases():
    rows = []          # (N, K, B, dyn, kind, grad)
    shapes = ([(130, K, 2, None) for K in range(1, 9)]                     # every mix mode and tile width R = 1..8
              + [(N, 3, 2, None) for N in (1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129, 255, 256, 257)]
              + [(N, 8, 2, None) for N in (1, 65, 257)]
              + [(130, 3, 3, True),                                        # odd batch, z_inner = K > 1
                 (1000, 3, 8, False),                                      # the benchmarked layer
                 (2000, 8, 1, True)])                                      # longest flat FWD_B, largest streamed mix
    for i, (N, K, B, only) in enumerate(shapes):
        for dyn in ((False, True) if only is None else (only,)):
            kind = "diag" if (i + dyn) % 2 == 0 else "dense"
            grad = 1e4 if (i + 2 * dyn) % 3 == 1 else 1e-5
            rows.append((N, K, B, dyn, kind, grad))
    return rows


CASES = _make_cases()


def _inputs(N, K, B, dyn, kind, seed, dev):
    rng = np.random.default_rng(seed)
    nz = B if dyn else 1
    mk = (lambda: diag_supports(rng, nz * K, N)) if kind == "diag" else (lambda: dense_supports(rng, nz * K, N))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    X = t(np.tanh(rng.standard_normal((B, N, N, 32))).astype(np.float32))
    Gd = t(mk().reshape((B, K, N, N) if dyn else (K, N, N)))
    Go = t(mk().reshape((B, K, N, N))) if dyn else Gd
    W = t((rng.standard_normal((K * K * 32, 32)) * (2.0 / (K * K * 32 + 32)) ** 0.5).astype(np.float32))
    bias = t((rng.standard_normal(32) * 0.1).astype(np.float32))
    return X, Go, Gd, W, bias


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,B,dyn,kind,grad", CASES)
def test_every_stage_matches_float64(N, K, B, dyn, kind, grad, cuda_device):
    X, Go, Gd, W, bias = _inputs(N, K, B, dyn, kind, 7919 * N + 31 * K + 2 * B + dyn, cuda_device)
    d_out = torch.randn(B, N, N, 32, device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(N + K)) * grad
    r = run_layer(X, Go, Gd, W, bias, d_out, dyn)
    tag = f"N={N} K={K} B={B} {'dyn' if dyn else 'static'}/{kind} |dOut|~{grad:g}"
    _assert_and_record(check_stages(r, X, Go, Gd, W, bias, d_out, dyn, tag, kind), tag)


@pytest.mark.gpu
@pytest.mark.parametrize("mag", [0.0, 1e-36, 2.0 ** 118])
def test_gradient_scale_edges(mag, cuda_device):
    """dOut = 0 -> S = 1; max|dOut| ~ 1e-36 and ~ 2^120 hit the +-100 exponent clamp.  dPre stays the saturating cast of the
    scaled gradient, and the gradients stay finite."""
    X, Go, Gd, W, bias = _inputs(40, 2, 1, False, "diag", 5, cuda_device)
    bias = bias + 1.0
    d_out = torch.randn(1, 40, 40, 32, device=cuda_device) * mag
    r = run_layer(X, Go, Gd, W, bias, d_out, False)
    amax = float(d_out.abs().max())
    S, invS = expected_scale(amax)
    assert (float(r["scale"][0]), float(r["scale"][1])) == (S, invS)
    assert S == {0.0: 1.0, 1e-36: 2.0 ** 100, 2.0 ** 118: 2.0 ** -100}[mag]
    d_pre = torch.where(r["out"] > 0, d_out, torch.zeros_like(d_out))
    assert torch.equal(bits(r["dp16"]), bits(f16_sat(d_pre * S)))
    for k in ("dX", "dW", "db"):
        assert torch.isfinite(r[k]).all(), k
    if mag == 0.0:
        assert not r["dX"].any() and not r["dW"].any() and not r["db"].any()


# ---- fp16 range: every fp16 store saturates instead of overflowing to inf (which the next contraction turns into NaN) ----
@pytest.mark.gpu
def test_z16_saturates_and_out_stays_finite(cuda_device):
    N, K, B = 130, 3, 1
    X, Go, Gd, W, bias = _inputs(N, K, B, False, "diag", 11, cuda_device)
    X[0, 5] = 60000.0                         # origin row 5: Z[5, e] = 6e4 * (column sum of G_d) -- beyond fp16 for most e
    r = run_layer(X, Go, Gd, W, bias, None, False)
    zref = torch.einsum("ncl,dce->dnel", r["x16"][0].double(), r["gd16"][0, :, :, :N].double())
    big = zref.abs() > 65520.0
    assert int(big.sum()) > 1000
    z = r["z16"][0].double()
    assert torch.equal(z[big], torch.sign(zref[big]) * HALF_MAX), "Z16 must hold +-65504 where Z overflows fp16"
    assert torch.isfinite(r["u16"].float()).all() and torch.isfinite(r["out"]).all()


@pytest.mark.gpu
def test_v16_saturates_and_gradients_stay_finite(cuda_device):
    """A support row with absolute sum 40 N > 2048 against dPre scaled to [16, 32): V16 = G_o x1 dPre exceeds 65504."""
    N, K, B = 130, 2, 1
    X, Go, Gd, W, bias = _inputs(N, K, B, True, "diag", 12, cuda_device)
    Go[0, :, 3, :] = 40.0
    bias = bias + 200.0                        # every output active: the whole dOut reaches V
    d_out = torch.full((B, N, N, 32), 1e-5, device=cuda_device)
    r = run_layer(X, Go, Gd, W, bias, d_out, True)
    assert bool((r["out"] > 0).all())
    vref = torch.einsum("onm,meh->oneh", r["bgo16"][0, :, :, :N].double(), r["dp16"][0].double())
    big = vref.abs() > 65520.0
    assert int(big.sum()) > 1000
    assert torch.equal(r["v16"][0].double()[big], torch.sign(vref[big]) * HALF_MAX), "V16 must hold +-65504 where V overflows fp16"
    for k in ("dX", "dW", "db"):
        assert torch.isfinite(r[k]).all(), f"{k} is not finite"


@pytest.mark.gpu
def test_x16_keeps_nan_and_saturates_inf(cuda_device):
    X, Go, Gd, W, bias = _inputs(9, 1, 1, False, "dense", 13, cuda_device)
    X[0, 1, 2, 3], X[0, 4, 5, 6], X[0, 7, 8, 9], X[0, 2, 2, 2] = math.nan, math.inf, -math.inf, -70000.0
    r = run_layer(X, Go, Gd, W, bias, None, False)
    x16 = r["x16"][0].float()
    assert math.isnan(float(x16[1, 2, 3])), "NaN must stay NaN"
    assert float(x16[4, 5, 6]) == HALF_MAX and float(x16[7, 8, 9]) == -HALF_MAX and float(x16[2, 2, 2]) == -HALF_MAX
    finite = torch.isfinite(X[0])
    assert torch.equal(bits(r["x16"][0][finite]), bits(f16_sat(X[0][finite])))
    assert torch.isnan(r["z16"][0, :, 1, :, 3].float()).all(), "the epilogue's fp16 store must keep NaN"    # Z[d, 1, e, 3] reads X[1, 2, 3]


# ------------------------------------------------------------------------------------------------------------------------------
# the detectors detect (CPU)
# ------------------------------------------------------------------------------------------------------------------------------
def _simulated(exact, ab, gen, fp16=True):
    """A faithful kernel: the float64 result plus fp32-accumulation-sized noise, stored as fp16."""
    noise = (torch.rand(exact.shape, generator=gen, dtype=torch.float64) * 2 - 1) * 2.0 ** -24 * ab
    y = exact + noise
    return f16_sat(y) if fp16 else y.float()


def test_detectors_accept_a_faithful_kernel_and_reject_each_defect():
    gen = torch.Generator().manual_seed(0)
    rng = np.random.default_rng(0)
    N, K = 96, 2
    x16 = f16_sat(torch.tanh(torch.randn(N, N, 32, generator=gen)))
    G = diag_supports(rng, K, N)
    delta, near = diag_rule(G)
    assert np.count_nonzero(delta) > 0.5 * K * N
    g16 = f16_sat(torch.from_numpy(G))
    W = torch.randn(K, K, 32, 32, generator=gen, dtype=torch.float32) * 0.08
    hi, lo = hilo(W)
    assert not bits(lo).eq(0).all()

    # FWD_A: faithful passes (bound and slope); a dropped k-block and a missing remainder fail
    z_ok, z_drop, z_norem = [], [], []
    bA, bDrop, sA, sNo = Bound(N, True), Bound(N, True), Slope(), Slope()
    for d in range(K):
        base, corr, ab = fwd_a_ref(x16, g16[d], torch.from_numpy(delta[d]))
        y = _simulated(base + corr, ab, gen)
        bA.add(y, base + corr, ab)
        sA.add(y.double() - base, corr)
        g_drop = g16[d].clone()
        g_drop[0:64] = 0                                                  # the first 64-row k-block never arrived
        bd, cd, _ = fwd_a_ref(x16, g_drop, torch.from_numpy(delta[d]))
        bDrop.add(_simulated(bd + cd, ab, gen), base + corr, ab)
        yn = _simulated(base, ab, gen)
        sNo.add(yn.double() - base, corr)
        z_ok.append(y)
    assert bA.ok and sA.judged and sA.ok, (bA.coef, sA.value)
    assert not bDrop.ok
    assert sNo.judged and not sNo.ok and abs(sNo.value) < 0.2, sNo.value

    # FWD_MIX: without the lo half of W the slope collapses
    z = torch.stack(z_ok)
    base, lpart, ab = mix_ref(z, hi, lo)
    sOk, sNoLo, bOk = Slope(), Slope(), Bound(64 * K, True)
    y = _simulated(base + lpart, ab, gen)
    bOk.add(y, base + lpart, ab)
    sOk.add(y.double() - base, lpart)
    sNoLo.add(_simulated(base, ab, gen).double() - base, lpart)
    assert bOk.ok and sOk.ok and sOk.judged
    assert sNoLo.judged and not sNoLo.ok

    # fp32 stage (BWD_DX-like): faithful passes, a result off by a factor 2 (the gradient scale) fails
    ref, ab = contract("dnel,dce->ncl", z, g16)
    assert Bound(K * N, False).add(_simulated(ref, ab, gen, fp16=False), ref, ab).ok
    assert not Bound(K * N, False).add(_simulated(2 * ref, ab, gen, fp16=False), ref, ab).ok

    # gradient scale: S off by a factor of 2 is not the rule
    for amax in (3.1e-7, 1e-5, 0.75, 1.0, 4096.0, 1e-36, 2.0 ** 121):
        S, invS = expected_scale(amax)
        assert S * invS == 1.0 and S == 2.0 ** round(math.log2(S))
        k = 5 - math.frexp(amax)[1]
        if -100 < k < 100:
            assert 16 <= S * amax < 32 and not 16 <= 2 * S * amax < 32
    assert expected_scale(0.0) == (1.0, 1.0) and expected_scale(math.inf) == (1.0, 1.0)

    # the saturating cast itself
    v = torch.tensor([math.nan, math.inf, -math.inf, 65519.0, 65520.0, -1e6, 1.0 + 2.0 ** -12, 3.0e-8])
    h = f16_sat(v)
    assert math.isnan(float(h[0])) and h[1:6].float().tolist() == [HALF_MAX, -HALF_MAX, HALF_MAX, HALF_MAX, -HALF_MAX]
    assert float(h[6]) == 1.0 and float(h[7]) == float(torch.tensor(3.0e-8).half())
