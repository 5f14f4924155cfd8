"""The contraction engine writes its output tiles by TMA store, bounded by the output tensor map and nothing else: a map one
row or one chunk too large would write next to an output without changing any value that the stage tests read.

One fp16 layer forward (with the fp16 shadow of `out`) and backward runs at N values that leave partial tiles in both the
row and the chunk dimension.  Every buffer a contraction stores into is placed inside a larger allocation whose guard bands
hold a sentinel byte pattern, and must leave them bit-identical:

* caller buffers: `out` (FWD_B), its fp16 shadow `out_f16` (FWD_B, second output map), `saved` = Z16 (FWD_A), `dX` (BWD_DX);
* workspaces `ws` (U16 of FWD_MIX) and `wsb` (V16 of BWD_V, Y16 of BWD_MIX, the dW partials of BWD_DW) as a whole; inside
  them, the padding between each of these regions and the next (the layout aligns regions to 1 KB) must keep the sentinel
  too, since nothing writes it.

The contraction outputs must also be fully written (no sentinel-valued NaN or stale element left in `out`, `out_f16`, `dX`).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

GUARD = 16384         # bytes on each side (several whole rows of every output layout at these N)
SENTINEL = 0x5A       # 0x5A5A5A5A is a finite fp32 (1.5e16) and 0x5A5A a finite fp16 (203.25): an unwritten element is not NaN


def _guarded(nbytes, dev):
    """-> (uint8 view of nbytes inside the guard bands, the whole allocation); everything prefilled with the sentinel"""
    whole = torch.full((nbytes + 2 * GUARD,), SENTINEL, dtype=torch.uint8, device=dev)
    return whole[GUARD:GUARD + nbytes], whole


def _sentinel(b, what):
    assert bool((b == SENTINEL).all()), f"{what}: {int((b != SENTINEL).sum())} bytes overwritten"


def _guards_intact(whole, nbytes, what):
    _sentinel(whole[:GUARD], f"{what}: bytes before the buffer")
    _sentinel(whole[GUARD + nbytes:], f"{what}: bytes after the buffer")


def _gap_intact(buf, off, nbytes, next_off, what):
    """the padding between a region [off, off + nbytes) and the next region of the same workspace"""
    assert off + nbytes <= next_off, f"{what}: region overlaps the next one"
    _sentinel(buf[off + nbytes:next_off], f"{what}: padding after the region")


CASES = [(130, 3, 3, False), (67, 2, 1, True), (257, 3, 1, False), (9, 1, 2, True), (131, 9, 1, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,B,dyn", CASES)
def test_tile_stores_stay_inside_every_output(N, K, B, dyn, cuda_device):
    from mpgcn_b200 import _lib
    lib = _lib.load()
    dev = cuda_device
    rng = np.random.default_rng(N * 10 + K)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    C = H = 32
    X = t(np.tanh(rng.standard_normal((B, N, N, C))))
    Gd = t(rng.random((B, K, N, N) if dyn else (K, N, N)) / N)
    Go = t(rng.random((B, K, N, N))) / N if dyn else Gd
    W = t(rng.standard_normal((K * K * C, H)) * 0.05)
    bias = t(rng.standard_normal(H) * 0.1)
    d_out = t(rng.standard_normal((B, N, N, H)))
    st = torch.cuda.current_stream().cuda_stream
    cells = B * N * N

    out_b, out_w = _guarded(4 * cells * H, dev)
    o16_b, o16_w = _guarded(2 * cells * H, dev)
    dX_b, dX_w = _guarded(4 * cells * C, dev)
    n_saved = lib.mpgcn_bdgcn_saved_bytes(B, N, K, C, H, 1)
    n_ws = lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, C, H, int(dyn), 1)
    n_wsb = lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, int(dyn), 1)
    saved, saved_w = _guarded(n_saved, dev)
    ws, ws_w = _guarded(n_ws, dev)
    wsb, wsb_w = _guarded(n_wsb, dev)
    out = out_b.view(torch.float32).view(B, N, N, H)
    amax = torch.zeros(1, device=dev)

    ex = _lib.BdgcnExtras()
    ex.out_f16 = o16_b.data_ptr()
    _lib.check(lib.mpgcn_bdgcn_forward_x(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn), W.data_ptr(), bias.data_ptr(), 1,
                                         out.data_ptr(), saved.data_ptr(), ws.data_ptr(), n_ws, B, N, K, C, H, 1, ctypes.addressof(ex), st),
               "forward_x")
    dW, db = torch.empty_like(W), torch.empty(H, device=dev)
    _lib.check(lib.mpgcn_bdgcn_backward_ex(d_out.data_ptr(), out.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dyn), W.data_ptr(), 1,
                                           saved.data_ptr(), dX_b.data_ptr(), dW.data_ptr(), db.data_ptr(), wsb.data_ptr(), n_wsb,
                                           B, N, K, C, H, 1, None, amax.data_ptr(), st), "backward_ex")
    torch.cuda.synchronize()

    for what, nbytes, whole in (("out", 4 * cells * H, out_w), ("out_f16", 2 * cells * H, o16_w), ("dX", 4 * cells * C, dX_w),
                                ("saved (Z16)", n_saved, saved_w), ("forward workspace", n_ws, ws_w), ("backward workspace", n_wsb, wsb_w)):
        _guards_intact(whole, nbytes, what)

    off = lambda w: lib.mpgcn_debug_tc_workspace_offset(w, B, N, K, int(dyn))
    act16 = B * K * N * N * 32 * 2                                      # one [B][K][N][N][32] fp16 activation (32 channels)
    slices = off(17)
    partials = slices * math.ceil(K / 4) * 128 * K * H * 4               # [slice][m tile][128][Ko * H] fp32
    _gap_intact(ws, off(4), act16, off(5), "U16")
    _gap_intact(wsb, off(13), act16, off(14), "V16")
    _gap_intact(wsb, off(14), act16, off(15), "Y16")
    _gap_intact(wsb, off(16), partials, off(18), "dW partials")

    o16 = o16_b.view(torch.float16).view(B, N, N, H)
    dX = dX_b.view(torch.float32).view(B, N, N, C)
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(dX).all())
    assert torch.equal(o16, out.half()), "out_f16 is not the fp16 shadow of out"
    assert not bool((dX_b.view(torch.int32) == 0x5A5A5A5A).any()), "dX: an element was never written"
    assert not bool((out_b.view(torch.int32) == 0x5A5A5A5A).any()), "out: an element was never written"
    assert amax.item() == dX.abs().max().item(), "dX absmax must cover exactly the stored elements"
