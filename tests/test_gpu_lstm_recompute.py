"""The recomputing LSTM backward (mpgcn_lstm_backward_recompute, ops `recompute=`, MPGCN.lstm_recompute): the training forward
keeps no c_t / h_t and the backward rebuilds them one chunk of tiles at a time (DESIGN.md section 6.5).

  * Same bits as the stored-state path: h_T of the inference forward equals the training forward's, dx equals
    mpgcn_lstm_last_backward_saved / mpgcn_lstm_stack_backward bit for bit, at every chunk size (1 cell, a tile +- 1, one
    wave +- 1, all cells) on cell counts that are not whole tiles and span several waves; the weight gradients agree up to fp32
    summation order and meet the float64 oracle at the width tests' bars (h_T 1e-3, gradients 2e-3).
  * The gradient scale over all cells (tiny, huge and zero d_hT) and the d_hT_absmax hint; deterministic mode.
  * The whole model: recompute on against off (eager, the captured training step, the row-shard model), the memory it saves,
    and one training step at N = 1000 at hidden 96 and 128.
"""
import numpy as np
import pytest
import torch
from torch import nn

import lstm_stack_oracle as sorc
from conftest import record_parity
from oracle import mpgcn_oracle as orc

import MPGCN as shim
from mpgcn_b200 import _lib, ops
from mpgcn_b200.graph_step import GraphedTrainStep

pytestmark = pytest.mark.gpu

H_TOL, G_TOL = 1e-3, 2e-3       # against float64, as tests/test_gpu_lstm_widths.py and test_gpu_lstm_stacked.py
ORDER_TOL = 1e-5                # weight gradients against the stored-state path: fp32 summation order only
TILE = {32: 128, 96: 64, 128: 48}
CONFIGS = [(32, 1), (96, 1), (128, 1), (32, 2), (32, 3), (96, 2), (96, 3)]
PREC = _lib.PREC_FP16_TC


def _wave(C):
    return torch.cuda.get_device_properties(0).multi_processor_count * TILE[C]


def _rel(a, ref):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    return float(np.linalg.norm(a - ref) / max(np.linalg.norm(ref), 1e-300))


def _check(a, ref, tol, what):
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and linf <= tol, f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"


def _weights(C, L, seed):
    rng = np.random.default_rng(seed)
    k = 1.0 / np.sqrt(C)
    return [[rng.uniform(-k, k, s).astype(np.float32) for s in ((4 * C, 1 if l == 0 else C), (4 * C, C), (4 * C,), (4 * C,))]
            for l in range(L)]


class Case:
    """x [B,T,NN], per-layer weights, d_hT on the device, and the three calls: stored-state training pair, inference forward,
    recomputing backward."""

    def __init__(self, C, L, B, T, NN, seed=0, d_scale=1.0, dev="cuda"):
        rng = np.random.default_rng(seed + 1)
        self.C, self.L, self.B, self.T, self.NN, self.cells = C, L, B, T, NN, B * NN
        self.x_np = (rng.random((B, T, NN)) * 4 - 1).astype(np.float32)
        self.w_np = _weights(C, L, seed)
        self.d_np = (rng.standard_normal((self.cells, C)) * d_scale).astype(np.float32)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        self.x, self.d_hT = t(self.x_np), t(self.d_np)
        self.w = [[t(a) for a in layer] for layer in self.w_np]
        self.dev = dev
        self.lib = _lib.load()
        self.st = torch.cuda.current_stream().cuda_stream

    def _ptrs(self, per_layer):
        return [ops._ptr_array([layer[k] for layer in per_layer]) for k in range(4)]

    def _grads(self):
        return [[torch.full_like(a, float("nan")) for a in layer] for layer in self.w]

    def _dx(self):
        return torch.full_like(self.x, float("nan"))

    def stored(self):
        """training forward (saved state) + backward from it -> (h_T, dx, grads)"""
        lib, C, L, B, T, NN = self.lib, self.C, self.L, self.B, self.T, self.NN
        hT = torch.full((self.cells, C), float("nan"), device=self.dev)
        g, dx = self._grads(), self._dx()
        if L == 1:
            n = lib.mpgcn_lstm_saved_bytes(B, T, NN, C, PREC)
            saved = torch.empty(n, dtype=torch.uint8, device=self.dev)
            _lib.check(lib.mpgcn_lstm_last_forward_train(self.x.data_ptr(), *[a.data_ptr() for a in self.w[0]], hT.data_ptr(),
                                                         saved.data_ptr(), n, B, T, NN, C, PREC, self.st), "fwd_train")
            ws = torch.empty(max(lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, PREC) - n, 256), dtype=torch.uint8, device=self.dev)
            _lib.check(lib.mpgcn_lstm_last_backward_saved(self.x.data_ptr(), *[a.data_ptr() for a in self.w[0]], self.d_hT.data_ptr(),
                                                          *[a.data_ptr() for a in g[0]], dx.data_ptr(), saved.data_ptr(), n, ws.data_ptr(),
                                                          ws.numel(), B, T, NN, C, PREC, None, self.st), "bwd_saved")
        else:
            n = lib.mpgcn_lstm_stack_saved_bytes(B, T, NN, C, L, PREC)
            saved = torch.empty(n, dtype=torch.uint8, device=self.dev)
            _lib.check(lib.mpgcn_lstm_stack_forward(self.x.data_ptr(), L, *self._ptrs(self.w), hT.data_ptr(), saved.data_ptr(), n, None, 0,
                                                    B, T, NN, C, PREC, self.st), "stack_fwd_train")
            ws = torch.empty(lib.mpgcn_lstm_stack_bwd_workspace_bytes(B, T, NN, C, L, PREC), dtype=torch.uint8, device=self.dev)
            _lib.check(lib.mpgcn_lstm_stack_backward(self.x.data_ptr(), L, *self._ptrs(self.w), self.d_hT.data_ptr(), *self._ptrs(g),
                                                     dx.data_ptr(), saved.data_ptr(), n, ws.data_ptr(), ws.numel(), B, T, NN, C, PREC, None,
                                                     self.st), "stack_bwd")
        torch.cuda.synchronize()
        return hT, dx, g

    def inference(self):
        lib, C, L, B, T, NN = self.lib, self.C, self.L, self.B, self.T, self.NN
        hT = torch.full((self.cells, C), float("nan"), device=self.dev)
        if L == 1:
            _lib.check(lib.mpgcn_lstm_last_forward(self.x.data_ptr(), *[a.data_ptr() for a in self.w[0]], hT.data_ptr(), B, T, NN, C, PREC,
                                                   self.st), "fwd")
        else:
            ws = torch.empty(lib.mpgcn_lstm_stack_fwd_workspace_bytes(B, T, NN, C, L, PREC), dtype=torch.uint8, device=self.dev)
            _lib.check(lib.mpgcn_lstm_stack_forward(self.x.data_ptr(), L, *self._ptrs(self.w), hT.data_ptr(), None, 0, ws.data_ptr(),
                                                    ws.numel(), B, T, NN, C, PREC, self.st), "stack_fwd")
        torch.cuda.synchronize()
        return hT

    def recompute(self, chunk, hint=None):
        lib, C, L, B, T, NN = self.lib, self.C, self.L, self.B, self.T, self.NN
        g, dx = self._grads(), self._dx()
        nws = lib.mpgcn_lstm_recompute_bwd_workspace_bytes(B, T, NN, C, L, chunk, PREC)
        assert nws > 0
        ws = torch.full((nws,), 0xFF, dtype=torch.uint8, device=self.dev)      # NaN wherever a region is read before it is written
        _lib.check(lib.mpgcn_lstm_backward_recompute(self.x.data_ptr(), L, *self._ptrs(self.w), self.d_hT.data_ptr(), *self._ptrs(g),
                                                     dx.data_ptr(), chunk, ws.data_ptr(), nws, B, T, NN, C, PREC,
                                                     None if hint is None else hint.data_ptr(), self.st), "bwd_recompute")
        torch.cuda.synchronize()
        return dx, g

    def oracle(self):
        """float64: h_T, dx [cells, T], per-layer (dw_ih, dw_hh, db_ih, db_hh)"""
        xs = self.x_np.astype(np.float64).transpose(0, 2, 1).reshape(self.cells, self.T, 1)
        layers = [tuple(a.astype(np.float64) for a in layer) for layer in self.w_np]
        d = self.d_np.astype(np.float64)
        if self.L == 1:
            h = orc.lstm_last_forward(xs, *layers[0])
            dx, *g = orc.lstm_last_backward(xs, *layers[0], d)
            grads = [tuple(g)]
        else:
            h = sorc.lstm_stack_forward(xs, layers)
            dx, grads = sorc.lstm_stack_backward(xs, layers, d)
        return h, dx.reshape(self.cells, self.T), grads

    def dx_cells(self, dx):
        """[B,T,NN] -> [cells, T]"""
        return dx.detach().cpu().numpy().transpose(0, 2, 1).reshape(self.cells, self.T)


def _shape(C, waves, extra):
    """(B, NN) with B NN = waves one-wave chunks + extra cells (ragged: not whole tiles, chunks not at sample boundaries)"""
    cells = int(waves * _wave(C)) + extra
    B = 3
    return B, -(-cells // B)


@pytest.mark.parametrize("T", (1, 7, 256))
@pytest.mark.parametrize("C,L", CONFIGS)
def test_recompute_gives_the_stored_paths_bits(C, L, T, cuda_device):
    B, NN = _shape(C, 2.5 if T < 256 else 1.5, 37)
    case = Case(C, L, B, T, NN, seed=C + L + T)
    hT, dx_ref, g_ref = case.stored()
    assert torch.equal(case.inference(), hT), "the inference forward's h_T differs from the training forward's"
    tile, wave = TILE[C], _wave(C)
    for chunk in (1, tile - 1, tile, tile + 1, wave - 1, wave + 1, 2 * wave + tile + 3, case.cells, 10 ** 12):
        dx, g = case.recompute(chunk)
        assert torch.equal(dx, dx_ref), f"chunk {chunk}: dx differs from the stored-state backward"
        for l in range(L):
            for k in range(4):
                err = _rel(g[l][k].cpu().numpy(), g_ref[l][k].cpu().numpy())
                record_parity(f"recompute C={C} L={L} T={T} chunk={chunk}: grad {k} of layer {l} vs stored", err, err, ORDER_TOL)
                assert err <= ORDER_TOL, (chunk, l, k, err)


@pytest.mark.parametrize("C,L", CONFIGS)
def test_recompute_meets_the_float64_oracle(C, L, cuda_device):
    B, NN = _shape(C, 1.5, 5)       # two chunks of one wave each at chunk_cells = 1
    case = Case(C, L, B, 7, NN, seed=3 * C + L)
    h, dx_ref, g_ref = case.oracle()
    _check(case.inference().cpu().numpy(), h, H_TOL, f"recompute C={C} L={L}: h_T vs float64")
    dx, g = case.recompute(1)
    _check(case.dx_cells(dx), dx_ref, G_TOL, f"recompute C={C} L={L}: dx vs float64")
    for l in range(L):
        for k in range(4):
            _check(g[l][k].cpu().numpy(), g_ref[l][k], G_TOL, f"recompute C={C} L={L}: grad {k} of layer {l} vs float64")


@pytest.mark.parametrize("C,L", [(32, 1), (96, 1), (96, 2)])
def test_gradient_scale_over_all_cells_and_the_hint(C, L, cuda_device):
    B, NN = _shape(C, 2.2, 11)
    for d_scale in (1e-7, 1e4, 0.0):
        case = Case(C, L, B, 7, NN, seed=5, d_scale=d_scale)
        _, dx_ref, g_ref = case.stored()
        dx, g = case.recompute(1)
        assert torch.equal(dx, dx_ref), d_scale
        for l in range(L):
            for k in range(4):
                if d_scale == 0.0:
                    assert not g[l][k].any(), "a zero d_hT gives zero gradients"
                else:
                    assert _rel(g[l][k].cpu().numpy(), g_ref[l][k].cpu().numpy()) <= ORDER_TOL, (d_scale, l, k)
        if d_scale == 0.0:
            assert not dx.any()
    # the hint replaces the absmax pass: one ELEMENTWISE launch fewer, the same bits
    case = Case(C, L, B, 7, NN, seed=6)
    hint = case.d_hT.abs().max().reshape(1).contiguous()
    counts, outs = [], []
    for h in (None, hint):
        torch.cuda.synchronize()
        case.lib.mpgcn_profile_enable(1)
        case.lib.mpgcn_profile_reset()
        outs.append(case.recompute(1, hint=h))
        counts.append(_lib.profile_read()["ELEMENTWISE"]["launches"])
        case.lib.mpgcn_profile_enable(0)
    assert counts[1] == counts[0] - 1, counts
    assert torch.equal(outs[0][0], outs[1][0])


@pytest.mark.parametrize("C,L", [(32, 1), (96, 1), (128, 1), (32, 2), (96, 2)])
def test_deterministic_mode_is_reproducible(C, L, cuda_device):
    B, NN = _shape(C, 2.5, 19)
    case = Case(C, L, B, 7, NN, seed=9)
    h, dx_ref, g_ref = case.oracle()
    prev = case.lib.mpgcn_get_deterministic()
    case.lib.mpgcn_set_deterministic(1)
    try:
        for chunk in (1, 2 * _wave(C) + 1):
            a, b = case.recompute(chunk), case.recompute(chunk)
            assert torch.equal(a[0], b[0])
            for l in range(L):
                for k in range(4):
                    assert torch.equal(a[1][l][k], b[1][l][k]), (chunk, l, k)
                    _check(a[1][l][k].cpu().numpy(), g_ref[l][k], G_TOL, f"recompute det C={C} L={L} chunk={chunk}: grad {k} of layer {l}")
            _check(case.dx_cells(a[0]), dx_ref, G_TOL, f"recompute det C={C} L={L} chunk={chunk}: dx")
    finally:
        case.lib.mpgcn_set_deterministic(prev)


# ------------------------------------------------------------------------------------------------------------------------------
# the whole model
# ------------------------------------------------------------------------------------------------------------------------------
def _model(N, hid, dev, L=1, seed=0):
    torch.manual_seed(seed)
    m = shim.MPGCN(M=2, K=3, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=L, gcn_hidden_dim=hid, gcn_num_layers=3, num_nodes=N,
                   user_bias=True, activation=nn.ReLU).to(dev)
    with torch.no_grad():
        for b in range(2):
            m.branch_models[b]['fc'][0].bias.add_(0.5)
    return m


def _inputs(B, T, N, dev, seed=1):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.rand(B, T, N, N, 1, generator=g) * 6).to(dev)
    y = (torch.rand(B, 1, N, N, 1, generator=g) * 2).to(dev)
    G = (torch.rand(3, N, N, generator=g) / N).to(dev)
    go, gd = ((torch.rand(B, 3, N, N, generator=g) / N).to(dev) for _ in range(2))
    return x, y, G, go, gd


def _step(model, x, y, G, go, gd):
    model.zero_grad(set_to_none=True)
    pred = model(x_seq=x, G_list=[G, (go, gd)])
    loss = nn.functional.mse_loss(pred, y)
    loss.backward()
    torch.cuda.synchronize()
    return pred.detach(), loss.detach(), {k: p.grad.clone() for k, p in model.named_parameters()}


def _compare(a, b, what):
    pred_a, loss_a, g_a = a
    pred_b, loss_b, g_b = b
    assert torch.equal(pred_a, pred_b) and torch.equal(loss_a, loss_b), f"{what}: prediction / loss"
    for k in g_a:
        if "spatial" in k and k.endswith(".W"):
            assert torch.equal(g_a[k], g_b[k]), f"{what}: {k}"
        else:          # LSTM, BDGCN bias and head gradients: atomic flushes (DESIGN.md section 7)
            err = _rel(g_a[k].cpu().numpy(), g_b[k].cpu().numpy())
            record_parity(f"{what}: grad {k}", err, err, ORDER_TOL)
            assert err <= ORDER_TOL, (what, k, err)


@pytest.mark.parametrize("hid,L", [(32, 1), (96, 1), (128, 1), (96, 2)])
def test_model_with_recompute_matches_the_stored_path(hid, L, cuda_device, monkeypatch):
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    N, B, T = 60, 2, 6
    model = _model(N, hid, cuda_device, L)
    data = _inputs(B, T, N, cuda_device)
    off = _step(model, *data)
    model.lstm_recompute = True
    ops.STASH_BYTES.clear()
    on = _step(model, *data)
    assert ops.STASH_BYTES["lstm"] == 2, "with recompute the forward counts the request only, no state"
    _compare(off, on, f"model hidden {hid} L={L}")
    model.lstm_recompute = 7           # a chunk size: raised to one wave, so several chunks at this size
    _compare(off, _step(model, *data), f"model hidden {hid} L={L} chunk 7")


def test_captured_training_step_with_recompute(cuda_device, monkeypatch):
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    N, B, T = 50, 2, 5
    x, y, G, go, gd = _inputs(B, T, N, cuda_device)
    res = []
    for rc in (None, True):
        model = _model(N, 96, cuda_device)
        model.lstm_recompute = rc
        opt = torch.optim.Adam(model.parameters(), lr=0.0, capturable=True)     # lr 0: the weights stay those of both runs
        step = GraphedTrainStep(model, nn.MSELoss(), opt, (x, y, G, (go, gd)), warmup=2)
        loss = step(x, y, go, gd).clone()
        torch.cuda.synchronize()
        pred = model(x_seq=x, G_list=[G, (go, gd)]).detach()
        res.append((pred, loss, {k: p.grad.clone() for k, p in model.named_parameters()}))
    _compare(res[0], res[1], "captured step")


def test_row_shard_model_with_recompute(tmp_path, cuda_device):
    """the NCCL worker of test_gpu_shard.py, with the sharded model's LSTM on the recomputing backward (tests/_recompute_shard_worker.py)"""
    import _recompute_shard_worker as worker
    for world in (1, 2):
        if torch.cuda.device_count() < world:
            continue
        models = [dict(N=40, T=5, hidden=hid, gcn_hidden=32, lstm_layers=L, seed=hid, yardstick="same", cases=[("fp16", "fp32", 1e-3, 8e-2)])
                  for hid, L in ((32, 1), (96, 1), (96, 2))]
        res = worker.run(world, tmp_path, models)
        rows = res["rows"]
        assert rows and res["recompute_calls"] > 0, "the sharded model did not take the recomputing path"
        for row in rows:
            record_parity(row["what"], row["linf"], row["l2"], row["tol"])
            assert row["err"] <= row["tol"], row


def _peak(model, data):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    _step(model, *data)
    return torch.cuda.max_memory_allocated() - base


def test_recompute_lowers_peak_memory(cuda_device, monkeypatch):
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    N, B, T, hid = 200, 4, 12, 96
    lib = _lib.load()
    model = _model(N, hid, cuda_device)
    data = _inputs(B, T, N, cuda_device)
    _step(model, *data)                              # warm: caches, supports, autograd
    off = _peak(model, data)
    model.lstm_recompute = True
    _step(model, *data)
    ops.STASH_BYTES.clear()
    on = _peak(model, data)
    NN = N * N
    saved = lib.mpgcn_lstm_saved_bytes(B, T, NN, hid, PREC)
    da = lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, hid, PREC) - saved - 1024     # the full-size records (after the 1 KB scale)
    chunk = ops.lstm_recompute_chunk_cells(True, T, hid, 1)
    ws = lib.mpgcn_lstm_recompute_bwd_workspace_bytes(B, T, NN, hid, 1, chunk, PREC)
    print(f"peak allocated, N={N} B={B} hidden {hid}: stored {off / 2**30:.2f} GiB, recompute {on / 2**30:.2f} GiB "
          f"(saved 2 x {saved / 2**30:.2f}, records {da / 2**30:.2f}, recompute workspace {ws / 2**30:.2f} GiB)")
    assert ops.STASH_BYTES["lstm"] == 2
    assert off - on >= 2 * saved + da - ws, (off, on, saved, da, ws)


@pytest.mark.parametrize("hid", (96, 128))
def test_training_step_at_n1000_with_recompute(hid, cuda_device, monkeypatch):
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    N, B, T = 1000, 4, 12
    model = _model(N, hid, cuda_device)
    model.lstm_recompute = True
    data = _inputs(B, T, N, cuda_device)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    _, loss, grads = _step(model, *data)
    peak = torch.cuda.max_memory_allocated()
    print(f"N=1000 B=4 hidden {hid} with recompute: loss {float(loss):.6g}, peak allocated {peak / 2**30:.2f} GiB")
    assert torch.isfinite(loss)
    assert all(torch.isfinite(g).all() for g in grads.values())
