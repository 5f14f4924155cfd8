"""The fused FC head (`mpgcn_head_forward` / `mpgcn_head_backward`, head_kernels.cu), checked stage by stage against float64
through the C ABI, and the head inside the model at branch counts and widths the other model tests do not run.

    forward   pre[m,cell] = g_m[cell,:] . w[m,:] + b[m]          y[cell] = (1/M) sum_m relu(pre[m,cell])
    backward  d = fl(dy fl(1/M)) [pre > 0]    dg_m = fl(d w_m)    dw_m = sum_cells d g_m    db_m = sum_cells d

Every output buffer is prefilled with NaN bytes, so an element the kernel leaves unwritten shows.  Sums are judged with the
`Bound` of test_gpu_engine_stages.py (EPS_C 2^-24 sqrt(L) |A|.|B| per element); what the kernel computes without a sum is
checked exactly against an fp32 replay from the kernel's own stash `pre`:
  * y bitwise: acc = fl(acc + max(pre_m, 0)) for m in order, y = fl(acc / M); a forward without the stash gives the same bits;
  * dg by value (so +0 == -0): products only, and the build has no fast-math, so they are IEEE;
  * dg_absmax bitwise max|dg_m| (+0 for a zero dy); the gradient of a branch whose dg pointer is NULL changes nothing else.
The mask is the kernel's own pre > 0, so an exact zero pre-activation (a zero g row with b = 0) takes no gradient, as torch's
ReLU backward gives.

The cases hit the branch-count templates (M = 1..4) and the run-time path (M = 5..8), widths around the 32-channel fast path,
and the grid-stride edges: the grid is capped at SMs * 8 blocks of 32 cells and each thread takes 4 cells a pass, so
S = SMs * 256 cells fill one slot of a pass; S + 1, 4S - 1, 4S + 1 and 10^6 cells hit the later slots and passes.
`test_head_detectors_*` (no GPU) shows that the checks accept a faithful kernel and reject each defect they are meant to find.
"""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

from test_gpu_engine_stages import Bound, _assert_and_record, _garbage

from mpgcn_b200 import _lib

WIDTHS = (4, 8, 28, 32, 36, 64, 100, 128, 256)
CELLS = ("1", "5", "3*47^2", "S", "S+1", "4S-1", "4S+1", "1e6")
SCALES = (1e-5, 1.0, 1e4, 0.0)
BUDGET = 64 << 20          # floats of branch input per case: cells * C * M
SM_MAX = 132               # an H100 SXM; a smaller part only shrinks the cell counts that depend on it


def n_cells(kind, sms):
    S = sms * 256
    return {"1": 1, "5": 5, "3*47^2": 3 * 47 * 47, "S": S, "S+1": S + 1, "4S-1": 4 * S - 1, "4S+1": 4 * S + 1, "1e6": 10 ** 6}[kind]


# (M, C, cells, |dy| scale, zero rows)
CASES = [
    (1, 4, "1", 1.0, False),
    (2, 8, "5", 1e-5, False),
    (3, 28, "3*47^2", 1e4, False),
    (4, 32, "S", 1.0, False),
    (5, 36, "S+1", 0.0, False),
    (6, 64, "4S-1", 1.0, False),
    (7, 64, "4S+1", 1e-5, False),
    (8, 100, "5", 1e4, False),
    (2, 32, "1e6", 1.0, False),
    (1, 256, "4S+1", 1.0, False),
    (4, 128, "S+1", 1e-5, False),
    (8, 256, "3*47^2", 1.0, False),
    (4, 100, "4S-1", 1e4, False),
    (6, 4, "1e6", 0.0, False),
    (3, 8, "4S+1", 1.0, False),
    (5, 36, "S", 1.0, True),
    (3, 32, "3*47^2", 1.0, True),
]


def test_head_stage_cases_cover_every_branch_count_width_edge_and_scale():
    assert {c[0] for c in CASES} == set(range(1, 9))
    assert {c[1] for c in CASES} == set(WIDTHS)
    assert {c[2] for c in CASES} == set(CELLS)
    assert {c[3] for c in CASES} == set(SCALES)
    assert any(c[4] for c in CASES) and any(c[4] and c[0] > 4 for c in CASES)
    assert {c[2] for c in CASES if c[0] > 4} >= {"S+1", "4S-1", "4S+1", "1e6"}        # the run-time path at the pass edges
    assert {c[1] for c in CASES if c[0] > 4} >= {4, 36, 64, 100, 256}
    for M, C, kind, _, _ in CASES:
        assert n_cells(kind, SM_MAX) * C * M <= BUDGET, (M, C, kind)


# ------------------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------------------
def _f32(n, dev):
    return _garbage(4 * n, dev).view(torch.float32)


def _ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[(t.data_ptr() if t is not None else None) for t in ts])


def head_forward(gs, w, b, want_pre=True):
    """-> (y [cells], pre [M, cells] or None), both prefilled with NaN bytes"""
    lib = _lib.load()
    M, (cells, C), dev = len(gs), gs[0].shape, w.device
    y = _f32(cells, dev)
    pre = _f32(M * cells, dev).view(M, cells) if want_pre else None
    _lib.check(lib.mpgcn_head_forward(_ptrs(gs), w.data_ptr(), b.data_ptr(), y.data_ptr(), pre.data_ptr() if want_pre else None, cells,
                                      C, M, torch.cuda.current_stream().cuda_stream), "head_forward")
    return y, pre


def head_backward(gs, w, pre, dy, with_dg=None):
    """-> (dg list, None where with_dg[m] is False; dw [M, C]; db [M]; dg_absmax [M]), all prefilled with NaN bytes"""
    lib = _lib.load()
    M, (cells, C), dev = len(gs), gs[0].shape, w.device
    with_dg = [True] * M if with_dg is None else with_dg
    dgs = [_f32(cells * C, dev).view(cells, C) if k else None for k in with_dg]
    dw, db, amax = _f32(M * C, dev).view(M, C), _f32(M, dev), _f32(M, dev)
    _lib.check(lib.mpgcn_head_backward(_ptrs(gs), w.data_ptr(), pre.data_ptr(), dy.data_ptr(), _ptrs(dgs), dw.data_ptr(), db.data_ptr(),
                                       amax.data_ptr(), cells, C, M, torch.cuda.current_stream().cuda_stream), "head_backward")
    return dgs, dw, db, amax


# ------------------------------------------------------------------------------------------------------------------------------
# checks (device-agnostic)
# ------------------------------------------------------------------------------------------------------------------------------
def _np(t):
    return t.detach().cpu().numpy()


def y_replay(pre):
    """fp32 replay of the forward's branch mean from the stash pre [M, cells] (numpy, IEEE single)"""
    pre = _np(pre)
    M = pre.shape[0]
    acc = np.zeros(pre.shape[1], np.float32)
    for m in range(M):
        acc = acc + np.maximum(pre[m], np.float32(0))
    return acc / np.float32(M)


def d_of(pre, dy):
    """d[m, cell] = fl(dy fl(1/M)) where the kernel's pre > 0, else 0 (float32 numpy)"""
    pre, dy = _np(pre), _np(dy)
    inv = np.float32(1) / np.float32(pre.shape[0])
    return np.where(pre > 0, dy * inv, np.float32(0)).astype(np.float32)


def head_stages(gs, w, b, dy, pre, y, dgs, dw, db, amax):
    """Every output against the operands its stage read -> ({stage: Bound}, [exact-check failures])"""
    M, C = w.shape
    bad = []
    res = {"FWD pre = g.w + b": Bound(C, False), "BWD dw = sum d g": Bound(dy.numel(), False), "BWD db = sum d": Bound(dy.numel(), False)}
    w64, b64 = w.double(), b.double()
    for m in range(M):
        g64 = gs[m].double()
        res["FWD pre = g.w + b"].add(pre[m], g64 @ w64[m] + b64[m], g64.abs() @ w64[m].abs() + b64[m].abs())
    y_exp = y_replay(pre)
    if not np.array_equal(_np(y).view(np.int32), y_exp.view(np.int32)):
        bad.append(f"y != fp32 replay from pre at {int((_np(y) != y_exp).sum())} cells")
    d = d_of(pre, dy)
    wn = _np(w)
    for m in range(M):
        dd = torch.from_numpy(d[m]).to(w.device).double()
        g64 = gs[m].double()
        res["BWD dw = sum d g"].add(dw[m], dd @ g64, dd.abs() @ g64.abs())
        res["BWD db = sum d"].add(db[m:m + 1], dd.sum().reshape(1), dd.abs().sum().reshape(1))
        if dgs[m] is None:
            continue
        dg = _np(dgs[m])
        if not np.array_equal(dg, d[m][:, None] * wn[m][None, :]):
            bad.append(f"dg[{m}] != fl(fl(dy/M) w) [pre > 0]")
        if np.float32(amax[m].item()).view(np.int32) != np.abs(dg).max().view(np.int32):
            bad.append(f"dg_absmax[{m}] = {amax[m].item()!r} != max|dg[{m}]| = {np.abs(dg).max()!r}")
    return res, bad


# ------------------------------------------------------------------------------------------------------------------------------
# the stages on the GPU
# ------------------------------------------------------------------------------------------------------------------------------
def _inputs(M, C, cells, scale, zero_rows, seed, dev):
    gen = torch.Generator(dev).manual_seed(seed)
    gs = [torch.randn(cells, C, device=dev, generator=gen) for _ in range(M)]
    w = torch.randn(M, C, device=dev, generator=gen) / C ** 0.5
    b = torch.randn(M, device=dev, generator=gen) * 0.3
    if zero_rows:            # pre-activations of exactly zero: every 5th cell of every branch, b = 0
        for g in gs:
            g[3::5] = 0
        b.zero_()
    dy = torch.randn(cells, device=dev, generator=gen) * scale if scale else torch.zeros(cells, device=dev)
    return gs, w, b, dy


@pytest.mark.gpu
@pytest.mark.parametrize("M,C,kind,scale,zero_rows", CASES)
def test_head_stages_match_float64(M, C, kind, scale, zero_rows, cuda_device):
    cells = n_cells(kind, torch.cuda.get_device_properties(cuda_device).multi_processor_count)
    gs, w, b, dy = _inputs(M, C, cells, scale, zero_rows, 7919 * M + 31 * C + cells, cuda_device)
    y, pre = head_forward(gs, w, b)
    y_inf, _ = head_forward(gs, w, b, want_pre=False)
    dgs, dw, db, amax = head_backward(gs, w, pre, dy)
    torch.cuda.synchronize()
    tag = f"head M={M} C={C} cells={cells} |dy|~{scale:g}{' zero rows' if zero_rows else ''}"
    res, bad = head_stages(gs, w, b, dy, pre, y, dgs, dw, db, amax)
    if not torch.equal(y_inf.view(torch.int32), y.view(torch.int32)):
        bad.append("y of the forward without the stash != y with it")
    if zero_rows:
        assert bool((pre == 0).any()), "the zero-row case has no exact zero pre-activation"
    if scale == 0:
        for what, t in [("dw", dw), ("db", db), ("dg_absmax", amax)] + [(f"dg[{m}]", d) for m, d in enumerate(dgs)]:
            if not bool((t == 0).all()):
                bad.append(f"{what} is not exactly zero for dy = 0")
        if amax.view(torch.int32).any():
            bad.append("dg_absmax is not +0 for dy = 0")
    if M > 1:                # one branch without a gradient buffer: the others are bitwise those of the call with all of them
        skip = M // 2
        part, _, _, amax_p = head_backward(gs, w, pre, dy, [m != skip for m in range(M)])
        torch.cuda.synchronize()
        for m in range(M):
            if m != skip and not (torch.equal(part[m].view(torch.int32), dgs[m].view(torch.int32)) and torch.equal(amax_p[m], amax[m])):
                bad.append(f"dg[{m}] / dg_absmax[{m}] changed when dg[{skip}] is NULL")
    assert not bad, f"{tag}: " + "; ".join(bad)
    _assert_and_record(res, tag)


# ------------------------------------------------------------------------------------------------------------------------------
# the checks detect (CPU)
# ------------------------------------------------------------------------------------------------------------------------------
def _faithful(gs, w, b, dy):
    """A kernel that does what the head is meant to: fp32 sums, the exact products, the branch mean in order."""
    M = w.shape[0]
    pre = torch.stack([gs[m] @ w[m] + b[m] for m in range(M)])
    y = torch.from_numpy(y_replay(pre))
    d = torch.from_numpy(d_of(pre, dy))
    dgs = [d[m][:, None] * w[m][None, :] for m in range(M)]
    dw = torch.stack([d[m] @ gs[m] for m in range(M)])
    db = d.sum(1)
    amax = torch.stack([g.abs().max() for g in dgs])
    return dict(pre=pre, y=y, dgs=dgs, dw=dw, db=db, amax=amax)


def _verdict(gs, w, b, dy, out):
    res, bad = head_stages(gs, w, b, dy, out["pre"], out["y"], out["dgs"], out["dw"], out["db"], out["amax"])
    return all(v.ok for v in res.values()) and not bad


def test_head_detectors_accept_a_faithful_kernel_and_reject_each_defect():
    torch.manual_seed(0)
    M, C, cells = 3, 64, 203
    gs, w, b, dy = _inputs(M, C, cells, 1.0, True, 5, torch.device("cpu"))
    w[1] *= 3                            # branch maxima of |dg| far apart
    ok = _faithful(gs, w, b, dy)
    assert bool((ok["pre"] == 0).any()) and _verdict(gs, w, b, dy, ok)

    def defect(**changes):
        out = dict(ok)
        out.update(changes)
        return _verdict(gs, w, b, dy, out)

    swapped = _faithful(gs, w[[1, 0, 2]], b, dy)
    assert not defect(pre=swapped["pre"], y=swapped["y"]), "two branches' weight rows swapped"
    assert not defect(y=ok["y"] * M), "1/M missing from y"
    assert not defect(dgs=[d * M for d in ok["dgs"]], amax=ok["amax"] * M), "1/M missing from dg"
    d_ge = torch.where(ok["pre"] >= 0, dy * (np.float32(1) / np.float32(M)), torch.zeros(()))
    assert not defect(dgs=[d_ge[m][:, None] * w[m][None, :] for m in range(M)]), "mask taken as pre >= 0"
    y_tail = ok["y"].clone()
    y_tail[-1] = float("nan")
    assert not defect(y=y_tail), "last cell of a ragged tail left unwritten (y)"
    pre_tail = ok["pre"].clone()
    pre_tail[:, -1] = float("nan")
    assert not defect(pre=pre_tail), "last cell of a ragged tail left unwritten (pre)"
    dg_tail = [d.clone() for d in ok["dgs"]]
    dg_tail[2][-1] = float("nan")
    assert not defect(dgs=dg_tail), "last cell of a ragged tail left unwritten (dg)"
    dw_cut = ok["dw"].clone()
    dw_cut[:, 32:] = 0
    assert not defect(dw=dw_cut), "dw channels >= 32 dropped"
    assert not defect(db=ok["db"] * 8), "db counted once per lane of a cell"
    assert not defect(amax=ok["amax"][[1, 0, 2]]), "dg_absmax taken from the wrong branch"


# ------------------------------------------------------------------------------------------------------------------------------
# argument checks: before any CUDA call (CPU, fake never-dereferenced addresses) and in ops.fc_relu_mean
# ------------------------------------------------------------------------------------------------------------------------------
def test_head_entry_points_refuse_what_the_kernels_cannot_read_without_a_gpu():
    """Every call fails validation, which runs before any CUDA call: the fake device addresses are never touched."""
    lib = _lib.load()
    p = 1 << 20                                   # a plausible, 16-byte aligned, never dereferenced address
    M, C, cells = 3, 32, 100

    def fwd(g=None, w=p, C=C, M=M):
        g = [p] * M if g is None else g
        r = lib.mpgcn_head_forward((ctypes.c_void_p * len(g))(*g), w, p, p, p, cells, C, M, None)
        return r, lib.mpgcn_last_error().decode()

    def bwd(g=None, w=p, dg=None, C=C, M=M):
        g = [p] * M if g is None else g
        dg = [p] * M if dg is None else dg
        r = lib.mpgcn_head_backward((ctypes.c_void_p * len(g))(*g), w, p, p, (ctypes.c_void_p * len(dg))(*dg), p, p, p, cells, C, M, None)
        return r, lib.mpgcn_last_error().decode()

    for call in (fwd, bwd):
        for M_bad in (0, 9):
            r, msg = call(M=M_bad)
            assert r != 0 and "branches unsupported" in msg, (call.__name__, M_bad)
        for C_bad in (0, 30):
            r, msg = call(C=C_bad)
            assert r != 0 and "multiple of 4" in msg, (call.__name__, C_bad)
        r, msg = call(w=p + 4)
        assert r != 0 and "w must be 16-byte aligned" in msg, call.__name__
        r, msg = call(g=[p, None, p])
        assert r != 0 and "branch 1 input is a null pointer" in msg, call.__name__
        r, msg = call(g=[p, p, p + 8])
        assert r != 0 and "branch 2 input must be 16-byte aligned" in msg, call.__name__
    r, msg = bwd(dg=[p, p + 4, p])
    assert r != 0 and "branch 1 gradient must be 16-byte aligned" in msg
    r, msg = bwd(dg=[p + 12, None, p])
    assert r != 0 and "branch 0 gradient must be 16-byte aligned" in msg


@pytest.mark.parametrize("dev", ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)])
def test_fc_relu_mean_refuses_mismatched_operands(dev):
    """Wrong shapes are refused before anything is launched.  Those given to the GPU stay inside their allocations (a wider w,
    a longer b, a branch with more cells), so even without the check they could only compute a wrong answer."""
    from mpgcn_b200 import ops
    if dev == "cuda" and not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    M, C, cells = 2, 8, 20
    gs = [torch.randn(cells, C, device=dev) for _ in range(M)]
    w, b = torch.randn(M, C, device=dev), torch.randn(M, device=dev)
    bad = [(gs, torch.randn(M, C + 4, device=dev), b, "w must be"),
           (gs, w, torch.randn(M + 1, device=dev), "w must be"),
           ([gs[0], torch.randn(cells + 3, C, device=dev)], w, b, "branch 1 has shape")]
    if dev == "cpu":         # never handed to a kernel here
        bad += [([g[:, :6] for g in gs], w[:, :6], b, "multiple of 4"),
                ([torch.randn(cells, C)] * 9, torch.randn(9, C), torch.randn(9), "1 to 8 branches"),
                ([], w, b, "1 to 8 branches"),
                (gs, w[:1], b, "w must be"),
                (gs, w, b.to(torch.device("meta")), "is on meta")]
    for g_, w_, b_, msg in bad:
        with pytest.raises(ValueError, match=msg):
            ops.fc_relu_mean(g_, w_, b_)
    if dev == "cuda":
        y = ops.fc_relu_mean(gs, w, b)
        ref = torch.stack([torch.relu(gs[m].double() @ w[m].double() + b[m].double()) for m in range(M)]).mean(0)
        assert torch.allclose(y[:, 0].double(), ref, rtol=1e-5, atol=1e-6)
    else:
        with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
            ops.fc_relu_mean(gs, w, b)


# ------------------------------------------------------------------------------------------------------------------------------
# the head inside the model (GPU): fused at M = 1, 3, 5, 8; the per-branch modules at M = 9, C = 10 and input_dim = 2
# ------------------------------------------------------------------------------------------------------------------------------
def _model_vs_oracle(M, hid, input_dim, prec, dev, branch_streams=False, seed=0):
    """One forward + backward of an MPGCN (K = 2, two BDGCN layers, static and dynamic supports alternating over the branches)
    against orc.mpgcn_forward_backward with the engine's ReLU masks -> (y, grads)."""
    import MPGCN as shim
    from oracle import mpgcn_oracle as orc
    from test_gpu_parity import TOL, _check, _t
    N, B, T, K, L = 10 + seed % 3, 2, 3, 2, 2
    torch.manual_seed(seed)
    model = shim.MPGCN(M=M, K=K, input_dim=input_dim, lstm_hidden_dim=32, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=L,
                       num_nodes=N, user_bias=True, activation=nn.ReLU)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.05)
    model = model.to(dev)
    model.lstm_precision = prec
    model.branch_streams = branch_streams
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = prec
    rng = np.random.default_rng(seed + M)
    x = (rng.random((B, T, N, N, input_dim)) * 4).astype(np.float32)
    d_y = rng.standard_normal((B, 1, N, N, input_dim)).astype(np.float32)
    GL = [(rng.random((K, N, N)) / N).astype(np.float32) if m % 2 == 0 else
          ((rng.random((B, K, N, N)) / N).astype(np.float32), (rng.random((B, K, N, N)) / N).astype(np.float32)) for m in range(M)]
    to_dev = lambda g: tuple(_t(a, dev) for a in g) if isinstance(g, tuple) else _t(g, dev)
    caps = {m: {"layers": [], "fc": None} for m in range(M)}
    hooks = [layer.register_forward_hook(lambda mod, inp, out, m=m: caps[m]["layers"].append(out.detach().cpu().numpy()))
             for m in range(M) for layer in model.branch_models[m]['spatial']]
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False      # input_dim > 1: nn.LSTM runs the LSTM, in fp32 as the engine's kernels do
    try:
        y = model(x_seq=_t(x, dev), G_list=[to_dev(g) for g in GL])
        y.backward(_t(d_y, dev))
        torch.cuda.synchronize()
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    for h in hooks:
        h.remove()
    assert tuple(y.shape) == (B, 1, N, N, input_dim)
    params = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in model.state_dict().items()}
    for m in range(M):
        fc = model.branch_models[m]['fc'][0]
        caps[m]["fc"] = orc.fc_relu_forward(caps[m]["layers"][-1], fc.weight.detach().cpu().numpy(), fc.bias.detach().cpu().numpy())
    f64 = lambda g: tuple(a.astype(np.float64) for a in g) if isinstance(g, tuple) else g.astype(np.float64)
    y_o, grads_o = orc.mpgcn_forward_backward(params, x.astype(np.float64), [f64(g) for g in GL], M=M, gcn_num_layers=L,
                                              d_y=d_y.astype(np.float64), masks=caps)
    tag = f"model head M={M} hid={hid} input_dim={input_dim} {prec}{' streams' if branch_streams else ''}"
    _check(y, y_o, TOL[prec][0], f"{tag}/y")
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    assert set(grads) == set(grads_o)
    for k, g in grads.items():
        if prec == "fp32":
            _check(g, grads_o[k], 2e-4, f"{tag}/grad:{k}")
        else:
            _check(g, grads_o[k], 5e-3, f"{tag}/grad:{k}", l2_only=True)
    return y.detach(), grads


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 3, 5, 8])
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_model_with_fused_head_matches_oracle(M, prec, cuda_device):
    _model_vs_oracle(M, 32, 1, prec, cuda_device, seed=M)


@pytest.mark.gpu
@pytest.mark.parametrize("M,hid,input_dim", [(9, 32, 1), (3, 10, 1), (2, 32, 2)])
def test_model_with_per_branch_head_matches_oracle(M, hid, input_dim, cuda_device):
    """More than 8 branches, a width that is not a multiple of 4, two input features: the per-branch modules, not the fused kernel."""
    _model_vs_oracle(M, hid, input_dim, "fp32", cuda_device, seed=M + hid)


@pytest.mark.gpu
def test_model_on_branch_streams_agrees_with_one_stream(cuda_device):
    y0, g0 = _model_vs_oracle(5, 32, 1, "fp32", cuda_device, seed=4)
    y1, g1 = _model_vs_oracle(5, 32, 1, "fp32", cuda_device, branch_streams=True, seed=4)
    from test_gpu_parity import _check
    _check(y1, y0.cpu().numpy(), 1e-6, "model head M=5 branch streams vs one stream/y")
    for k in g0:              # the weight gradients add with atomics in an order that varies from run to run
        _check(g1[k], g0[k].cpu().numpy(), 1e-5, f"model head M=5 branch streams vs one stream/grad:{k}", l2_only=True)
