"""Every stage of a layer PART (`mpgcn_bdgcn_forward_part` / `_backward_part`, include/mpgcn_b200.h), checked against float64, in
both kernel families.

The row shard and the K shard evaluate parts, not whole layers, and a part runs code a whole layer does not: FWD_B over an
origin-row slab (one k-segment per support, the support map based at row0, the rows past the slab zero-filled), the origin
remainders masked to the slab, BWD_V / BWD_DX / FWD_A on R-row slabs, channel mixes from Kd*cC to Ko*cH planes when Ko != Kd,
BWD_DW tiling Kd*cC by Ko*cH chunks, and the fp16 dPre prepared by `mpgcn_relu_backward_scatter_f16` with a scale taken from
the global max|dOut| of every rank.  Each case runs one part through the C ABI with every buffer prefilled with a sentinel
inside guard bands, reads every intermediate back from the workspaces (their layouts mirrored by
test_gpu_channel_widths.part_ws_layout / simt_ws_layout and checked against the library's sizes) and recomputes each stage
from the operands it read, with the helpers and bounds of test_gpu_engine_stages.py:

  * tensor cores: conversions bit-exact, the remainders by the tau rule, S by the power-of-two rule, each contraction within
    2^-11 |r| + EPS_C 2^-24 sqrt(L) (|A|.|B|), the remainders and W's `lo` half as regression slopes of 1;
  * prepared fp16 dPre: with a global max|dPre| several times the part's own, the same bounds with that S; with the part's own
    maximum, dW and dX bitwise equal to the call that casts the fp32 dPre itself;
  * fp32 kernels at widths that are not multiples of 32, parts and whole layers: each contraction within EPS_C 2^-24 sqrt(L)
    (|A|.|B|), at N that end the SGEMM's 64-row tiles and 16-deep k slabs partially, and a dW whose split-K slices do not
    divide R*N;
  * no store outside any output or workspace region (guard bands, and the padding between regions), every output written.

The largest coefficient of each bound goes to the parity report ("stages part ...").
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from test_gpu_channel_widths import Layout, backward_stages, check_stages_wide, part_ws_layout, run_layer_wide, simt_ws_layout
from test_gpu_engine_stages import _assert_and_record, bits, dense_supports, diag_supports, expected_scale
from test_gpu_engine_store_bounds import SENTINEL, _gap_intact, _guarded, _guards_intact

from mpgcn_b200 import _lib

GLOBAL_AMAX = 7.3       # a prepared dPre's scale comes from max|dOut| over every rank: here this many times the part's own

# ------------------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------------------
# (C, H, N, K, Ko, Kd, R, row0, B): origin rows [row0, row0 + R) of N, Ko origin / Kd destination supports of a K-support layer
SHAPES = [
    # origin-row slabs (Ko = Kd = K)
    (32, 32, 130, 3, 3, 3, 65, 65, 2),
    (32, 32, 130, 3, 3, 3, 1, 0, 2),
    (32, 32, 257, 3, 3, 3, 1, 256, 1),
    (64, 64, 130, 3, 3, 3, 63, 1, 2),
    (64, 64, 130, 3, 3, 3, 129, 1, 1),
    (64, 64, 257, 3, 3, 3, 128, 129, 1),
    (32, 96, 130, 3, 3, 3, 64, 65, 2),
    (96, 32, 257, 3, 3, 3, 129, 0, 1),
    (128, 64, 257, 3, 3, 3, 65, 65, 1),
    # support subsets over every row: the K shard's Kd < K, and an origin-side subset
    (32, 32, 130, 3, 3, 1, 130, 0, 2),
    (64, 64, 130, 3, 3, 2, 130, 0, 2),
    (32, 96, 130, 9, 9, 4, 130, 0, 1),         # 27 forward mix output planes (four groups), dW 4 x 4 column tiles
    (96, 32, 65, 3, 1, 3, 65, 0, 2),           # one forward mix output plane, nine backward
    (128, 64, 65, 3, 3, 2, 65, 0, 2),
    # slab and subset
    (64, 64, 257, 9, 9, 4, 65, 1, 1),
    (96, 32, 130, 3, 1, 3, 63, 65, 2),
]


def _make_cases():
    rows = []          # (C, H, N, K, Ko, Kd, R, row0, B, dyn, kind, grad)
    for i, shape in enumerate(SHAPES):
        dyn = i % 2 == 1
        kind = "diag" if (i // 2) % 2 == 0 else "dense"
        grad = 1e4 if i % 3 == 1 else 1e-5
        rows.append(shape + (dyn, kind, grad))
    return rows


CASES = _make_cases()

# the fp32 family at widths that are not multiples of 32; row0 None: the whole layer (bias, ReLU)
FP32_SHAPES = [
    (1, 1, 1, 3, 3, 3, 1, None, 2),
    (3, 5, 15, 2, 2, 2, 15, None, 2),
    (8, 12, 16, 3, 3, 3, 16, None, 2),
    (17, 33, 17, 3, 3, 3, 17, None, 1),
    (48, 48, 63, 2, 2, 2, 63, None, 1),
    (100, 36, 64, 1, 1, 1, 64, None, 1),
    (3, 5, 65, 3, 3, 3, 65, None, 2),
    (17, 33, 130, 3, 3, 3, 130, None, 1),      # dW: R*N = 16900 in 8 split-K slices of 2113, the last 2109
    (1, 1, 130, 3, 3, 3, 65, 65, 2),           # R*N = 8450: 4 slices of 2113, the last 2111
    (8, 12, 65, 3, 3, 3, 17, 1, 2),
    (48, 48, 64, 3, 3, 2, 64, 0, 1),
    (100, 36, 17, 3, 1, 3, 17, 0, 2),
    (3, 5, 130, 3, 3, 1, 63, 1, 1),
    (17, 33, 63, 3, 3, 3, 1, 62, 2),
]
FP32_CASES = [s + (i % 2 == 1, "dense" if i % 3 else "diag") for i, s in enumerate(FP32_SHAPES)]


def _simt_ksplit(RN):
    return min(256, max(1, RN // 2048))        # bdgcn_simt.cu BWD_DW


def test_part_cases_cover_slabs_subsets_widths_kinds_and_scales():
    slabs = [c for c in CASES if c[6] < c[2]]
    subsets = [c for c in CASES if c[4] != c[5] or c[4] != c[3]]
    assert {c[6] for c in slabs if c[4] == c[5] == c[3]} == {1, 63, 64, 65, 128, 129}
    assert {0, 1, 65} <= {c[7] for c in slabs} and any(c[7] == c[2] - c[6] for c in slabs)
    assert {c[2] for c in slabs} == {130, 257}
    assert {(c[3], c[4], c[5]) for c in subsets} == {(3, 3, 1), (3, 3, 2), (9, 9, 4), (3, 1, 3)}
    assert [c for c in slabs if c in subsets], "a case that is both a slab and a subset"
    widths = {(c[0], c[1]) for c in CASES}
    assert widths == {(32, 32), (64, 64), (32, 96), (96, 32), (128, 64)}
    for w in widths:
        assert any((c[0], c[1]) == w for c in slabs) and any((c[0], c[1]) == w for c in subsets), w
    assert {c[9] for c in CASES} == {False, True} and {c[10] for c in CASES} == {"diag", "dense"} and {c[11] for c in CASES} == {1e-5, 1e4}
    assert {c[9] for c in subsets} == {False, True} and {c[9] for c in slabs} == {False, True}
    # store bounds: R not a multiple of 8 with row0 != 0, and a subset with an odd number of mix output planes
    assert any(c[6] % 8 and c[7] for c in slabs)
    assert any((c[4] * c[1] // 32) % 2 for c in subsets)
    for row0, R, N in {(c[7], c[6], c[2]) for c in CASES}:
        assert 0 <= row0 and row0 + R <= N

    assert {(c[0], c[1]) for c in FP32_CASES} == {(1, 1), (3, 5), (8, 12), (17, 33), (48, 48), (100, 36)}
    assert {c[2] for c in FP32_CASES} == {1, 15, 16, 17, 63, 64, 65, 130}
    for w in {(c[0], c[1]) for c in FP32_CASES}:
        assert {c[7] is None for c in FP32_CASES if (c[0], c[1]) == w} == {False, True}, w
    assert any(c[7] is not None and c[6] * c[2] >= 4096 and (c[6] * c[2]) % _simt_ksplit(c[6] * c[2]) for c in FP32_CASES)
    assert any(c[4] != c[5] for c in FP32_CASES) and {c[9] for c in FP32_CASES} == {False, True}


def test_fp32_workspace_layouts_match_the_library_sizes():
    """the fp32 layouts of bdgcn_simt.cu (and the tensor-core forward layout, which does not depend on the SM count) against the
    sizes the library reports; the backward tensor-core layout is checked on the GPU, inside run_layer_wide"""
    lib = _lib.load()
    for C, H, N, K, Ko, Kd, R, row0, B, dyn, _ in FP32_CASES:
        part = _lib.BdgcnPart(row0 or 0, R, Ko, Kd)
        fwd, bwd = simt_ws_layout(B, N, C, H, R, Ko, Kd)
        pp = ctypes.addressof(part)
        assert fwd.total == lib.mpgcn_bdgcn_part_fwd_workspace_bytes(B, N, C, H, int(dyn), 0, pp)
        assert bwd.total == lib.mpgcn_bdgcn_part_bwd_workspace_bytes(B, N, C, H, int(dyn), 0, pp)
        assert fwd["u"] == 0 and fwd["z"] % 256 == 0 and bwd["dpre"] == 0
        assert lib.mpgcn_bdgcn_part_saved_bytes(B, N, C, H, 0, pp) == B * Kd * R * N * C * 4
    for C, H, N, K, Ko, Kd, R, row0, B, dyn, *_ in CASES:
        part = _lib.BdgcnPart(row0, R, Ko, Kd)
        fwd, _ = part_ws_layout(B, N, C, H, dyn, R, row0, Ko, Kd, 132)
        assert fwd.total == lib.mpgcn_bdgcn_part_fwd_workspace_bytes(B, N, C, H, int(dyn), 1, ctypes.addressof(part))
    assert Layout([("a", 1), ("b", 1)], 256, 256).total == 768


# ------------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------------
class GuardedAlloc:
    """run_layer_wide's allocator: every buffer inside guard bands, everything prefilled with the sentinel byte"""

    def __init__(self):
        self.bufs = []

    def __call__(self, nbytes, dev, what):
        b, whole = _guarded(nbytes, dev)
        self.bufs.append((what, nbytes, whole))
        return b

    def check(self, tag):
        for what, nbytes, whole in self.bufs:
            _guards_intact(whole, nbytes, f"{tag}: {what}")


def _regions_intact(r, tag):
    """the padding after every workspace region, up to the next one (the layouts align regions), keeps the sentinel"""
    for buf, layout in ((r["bufs"]["ws"], r["layouts"][0]), (r["bufs"].get("wsb"), r["layouts"][1])):
        if buf is None:
            continue
        names = list(layout)
        for name, nxt in zip(names, names[1:] + [None]):
            _gap_intact(buf, layout[name], layout.size[name], layout.total if nxt is None else layout[nxt], f"{tag}: {name}")


def _all_written(r, tag):
    word = int.from_bytes(bytes([SENTINEL] * 4), "little")
    for k in ("out", "dX"):
        if k in r["bufs"]:
            assert not bool((r["bufs"][k].view(torch.int32) == word).any()), f"{tag}: {k}: an element was never written"


def _inputs(C, H, N, K, Ko, Kd, R, row0, B, dyn, kind, seed, dev):
    """X (the slab [B,R,N,C] of a part, [B,N,N,C] of a whole layer), Go = supports [0, Ko) and Gd = supports [d_lo, d_lo + Kd) of
    the layer's K -- static: views of one stack, as the shard passes them (the same buffer when d_lo = 0) --, W [Ko*Kd*C, H], bias [H]"""
    rng = np.random.default_rng(seed)
    mk = (lambda P: diag_supports(rng, P, N)) if kind == "diag" else (lambda P: dense_supports(rng, P, N))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    X = t(np.tanh(rng.standard_normal((B, R, N, C))).astype(np.float32))
    d_lo = (K - Kd) // 2
    if dyn:
        Go = t(mk(B * K).reshape(B, K, N, N)[:, :Ko])
        Gd = t(mk(B * K).reshape(B, K, N, N)[:, d_lo:d_lo + Kd])
    else:
        G = t(mk(K))
        Go, Gd = G[:Ko], G[d_lo:d_lo + Kd]
    W = t((rng.standard_normal((Ko * Kd * C, H)) * (2.0 / (K * K * C + H)) ** 0.5).astype(np.float32))
    bias = t((rng.standard_normal(H) * 0.1).astype(np.float32))
    return X, Go, Gd, W, bias


def _prepare_dpre(d_pre, amax):
    """mpgcn_relu_backward_scatter_f16 at g = 1 over every row (act 0): -> (fp16 S * dPre [B,N,N,H], [S, 1/S]) for max|dOut| = amax"""
    lib = _lib.load()
    B, N, _, H = d_pre.shape
    dev = d_pre.device
    dp16 = torch.full((B, N, N, H), math.nan, dtype=torch.float16, device=dev)
    scale2 = torch.full((2,), math.nan, device=dev)
    amax_t = torch.tensor([amax], dtype=torch.float32, device=dev)
    dsts = (ctypes.c_void_p * 1)(dp16.data_ptr())
    _lib.check(lib.mpgcn_relu_backward_scatter_f16(d_pre.data_ptr(), None, 0, dsts, 1, None, amax_t.data_ptr(), scale2.data_ptr(), B, N, 0, N, H,
                                                   torch.cuda.current_stream().cuda_stream), "relu_backward_scatter_f16")
    return dp16, scale2, float(amax_t)


@pytest.mark.gpu
@pytest.mark.parametrize("C,H,N,K,Ko,Kd,R,row0,B,dyn,kind,grad", CASES)
def test_every_part_stage_matches_float64_on_tensor_cores(C, H, N, K, Ko, Kd, R, row0, B, dyn, kind, grad, cuda_device):
    dev = cuda_device
    X, Go, Gd, W, _ = _inputs(C, H, N, K, Ko, Kd, R, row0, B, dyn, kind, 7919 * N + 31 * K + 7 * Ko + 3 * Kd + R + row0 + C + 5 * H, dev)
    d_pre = torch.randn(B, N, N, H, device=dev, generator=torch.Generator(dev).manual_seed(N + R + C + H)) * grad
    tag = f"part fp16 C={C} H={H} N={N} K={K} Ko={Ko} Kd={Kd} rows [{row0}, {row0 + R}) B={B} {'dyn' if dyn else 'static'}/{kind} |dPre|~{grad:g}"
    guard = GuardedAlloc()
    r = run_layer_wide(X, Go, Gd, W, None, d_pre, dyn, row0, alloc=guard)
    res = check_stages_wide(r, X, Go, Gd, W, None, d_pre, dyn, kind, row0)
    guard.check(tag)
    _regions_intact(r, tag)
    _all_written(r, tag)

    # the fp16 dPre as relu_backward_scatter_f16 prepares it, its S from a global max|dPre| larger than this part's own
    local = float(d_pre.abs().max())
    dp16, scale2, amax = _prepare_dpre(d_pre, local * GLOBAL_AMAX)
    assert expected_scale(amax)[0] < expected_scale(local)[0], "the global maximum was meant to give a smaller S"
    rg = run_layer_wide(X, Go, Gd, W, None, None, dyn, row0, d_pre16=(dp16, scale2))
    for k, v in backward_stages(rg, X, Go, Gd, W, d_pre, dyn, row0, amax=amax).items():
        res[f"{k} (prepared dPre, global S)"] = v
    # ... and with this part's own maximum: the same S, the same bits as the call that casts the fp32 dPre itself
    dp16, scale2, amax = _prepare_dpre(d_pre, local)
    assert amax == local
    rl = run_layer_wide(X, Go, Gd, W, None, None, dyn, row0, d_pre16=(dp16, scale2))
    assert torch.equal(bits(rl["z"]), bits(r["z"])), "the forward is not deterministic"
    assert torch.equal(bits(dp16), bits(r["dp"])), "prepared dP16 != the part's own dP16"
    assert torch.equal(bits(rl["dW"]), bits(r["dW"])) and torch.equal(bits(rl["dX"]), bits(r["dX"])), \
        "backward_part on the prepared fp16 dPre (same S) differs from the call on the fp32 dPre"
    _assert_and_record(res, tag)


@pytest.mark.gpu
@pytest.mark.parametrize("C,H,N,K,Ko,Kd,R,row0,B,dyn,kind", FP32_CASES)
def test_every_stage_matches_float64_on_fp32_kernels(C, H, N, K, Ko, Kd, R, row0, B, dyn, kind, cuda_device):
    dev = cuda_device
    X, Go, Gd, W, bias = _inputs(C, H, N, K, Ko, Kd, R, row0, B, dyn, kind, 104729 * N + 31 * K + R + C + 5 * H, dev)
    d_out = torch.randn(B, N, N, H, device=dev, generator=torch.Generator(dev).manual_seed(N + C + H))
    what = "layer" if row0 is None else f"part rows [{row0}, {row0 + R}) Ko={Ko} Kd={Kd}"
    tag = f"fp32 {what} C={C} H={H} N={N} K={K} B={B} {'dyn' if dyn else 'static'}/{kind}"
    guard = GuardedAlloc()
    r = run_layer_wide(X, Go, Gd, W, bias, d_out, dyn, row0, prec=0, alloc=guard)
    res = check_stages_wide(r, X, Go, Gd, W, bias, d_out, dyn, kind, row0, prec=0)
    guard.check(tag)
    _regions_intact(r, tag)
    _all_written(r, tag)
    _assert_and_record(res, tag)
