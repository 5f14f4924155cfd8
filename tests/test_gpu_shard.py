"""Layer PARTS on the GPU (`mpgcn_bdgcn_forward_part` / `_backward_part`, include/mpgcn_b200.h) -- what one rank of an origin-row
shard or of a K shard evaluates (SURVEY.md section 8(e)) -- against an independent float64 evaluation of the same part
(tests/shard_standin.py), rank by rank on ONE GPU, and the parts of all ranks summed against the whole layer.  The NCCL run of the
sharded model over 2 GPUs is `test_sharded_model_nccl_world2` (skipped on a 1-GPU box)."""
import numpy as np
import pytest
import torch

import _shard_nccl_worker as nccl_worker
import abi
from conftest import record_parity
from oracle import mpgcn_oracle as orc
from shard_standin import TorchEngine

from mpgcn_b200 import shard

pytestmark = pytest.mark.gpu
TOL = {"fp32": (2e-5, 1e-4), "fp16": (1e-3, 2e-3)}


def _check(a, ref, tol, what):
    linf, l2 = orc.rel_errors(a.detach().cpu().numpy(), ref.detach().cpu().numpy())
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and linf <= tol and l2 <= tol, f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"


@pytest.mark.parametrize("kind,N,world,K,dyn", [("row", 130, 2, 3, False), ("row", 256, 4, 3, True), ("row", 300, 2, 3, False),
                                                 ("row", 1000, 8, 3, True), ("k", 130, 2, 3, True), ("k", 201, 3, 3, False),
                                                 ("k", 300, 4, 6, False), ("k", 132, 4, 3, False)])
def test_layer_parts_match_standin_and_sum_to_the_whole_layer(kind, N, world, K, dyn, cuda_device):
    dev = cuda_device
    torch.manual_seed(N + world)
    B, C = 2 if N <= 300 else 1, 32
    X = torch.tanh(torch.randn(B, N, N, C, device=dev))
    mk = (lambda: torch.randn(B, K, N, N, device=dev) / N ** 0.5) if dyn else (lambda: torch.randn(K, N, N, device=dev) / N ** 0.5)
    Go = mk()
    Gd = mk() if dyn else Go
    W = torch.randn(K * K * C, C, device=dev) * (2.0 / (K * K * C + C)) ** 0.5
    bias = torch.randn(C, device=dev) * 0.1
    d_pre = torch.randn(B, N, N, C, device=dev) * 1e-4
    cuda, ref = shard.CudaEngine(), TorchEngine()
    for prec_name, prec in (("fp32", 0), ("fp16", 1)):
        tf, tb = TOL[prec_name]
        total = torch.zeros(B, N, N, C, device=dev)
        dX_all = torch.zeros(B, N, N, C, device=dev)
        dW_all = torch.zeros(K, K, C, C, device=dev)
        for r in range(world):
            plan = shard.ShardPlan(kind, r, world, N, K)
            if kind == "row":
                Xp, row0, rows, Kd, Gdp, Wp = X[:, plan.row_lo:plan.row_hi].contiguous(), plan.row_lo, plan.rows, K, Gd, W
            else:
                if plan.Kd == 0:
                    continue
                Xp, row0, rows, Kd = X, 0, N, plan.Kd
                Gdp = (Gd[:, plan.d_lo:plan.d_hi] if dyn else Gd[plan.d_lo:plan.d_hi]).contiguous()
                Wp = W.view(K, K, C, C)[:, plan.d_lo:plan.d_hi].reshape(K * Kd * C, C).contiguous()
            pre, saved = cuda.forward_part(Xp, Go, Gdp, dyn, Wp, N, row0, K, Kd, prec, True)
            pre_r, Z_r = ref.forward_part(Xp, Go, Gdp, dyn, Wp, N, row0, K, Kd, 0, True)
            _check(pre, pre_r, tf, f"part {kind} N={N} rank {r}/{world} {prec_name} partial pre")
            total += pre
            dX, dW = cuda.backward_part(d_pre, Go, Gdp, dyn, Wp, saved, N, row0, rows, K, Kd, C, prec, True)
            dX_r, dW_r = ref.backward_part(d_pre, Go, Gdp, dyn, Wp, Z_r, N, row0, rows, K, Kd, C, 0, True)
            _check(dX, dX_r, tb, f"part {kind} N={N} rank {r}/{world} {prec_name} dX")
            _check(dW, dW_r, tb, f"part {kind} N={N} rank {r}/{world} {prec_name} dW")
            if kind == "row":
                dX_all[:, plan.row_lo:plan.row_hi] = dX
                dW_all += dW.view(K, K, C, C)
            else:
                dX_all += dX
                dW_all[:, plan.d_lo:plan.d_hi] = dW.view(K, Kd, C, C)
        # the parts of all ranks, exchanged (= summed) and finished with bias + ReLU, are the whole layer
        cuda.bias_act(total, bias, 1)
        Go_, Gd_ = (Go, Gd) if dyn else (Go, Go)
        whole, saved_w = abi.forward(X, Go_, Gd_, W, bias, True, "fp32")
        _check(total, whole, tf, f"parts {kind} N={N} x{world} {prec_name}: sum of partials == whole layer")
        # ... and so are their gradients (whole layer fed d_pre through a linear epilogue: act = None)
        lin, saved_l = abi.forward(X, Go_, Gd_, W, bias, False, "fp32")
        dXw, dWw, _ = abi.backward(d_pre, lin, Go_, Gd_, W, False, saved_l, "fp32")
        _check(dX_all, dXw, tb, f"parts {kind} N={N} x{world} {prec_name}: dX")
        _check(dW_all.view(K * K * C, C), dWw, tb, f"parts {kind} N={N} x{world} {prec_name}: dW")


@pytest.mark.parametrize("N,dyn", [(130, False), (258, True)])
def test_row_shard_fp16_partials_on_dominant_diagonals_sum_to_the_whole_layer(N, dyn, cuda_device):
    """Row shard over 2 ranks on supports whose diagonal remainder correction fires: the fp16 partial pre-activations of both
    ranks, summed, equal the fp16 whole layer (no bias, no activation) to 1e-5.  A slab's Z16 and U16 rows come from the same
    kernels on the same bits as the whole layer's; only the FWD_B accumulation order differs.  So this pins what the slab adds:
    the origin remainders masked to the slab's rows and the zero-filled rows past the slab edge."""
    from test_gpu_engine_stages import diag_supports
    dev = cuda_device
    rng = np.random.default_rng(N)
    B, K, C, world = 2, 3, 32, 2
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    X = t(np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32))
    shape = (B, K, N, N) if dyn else (K, N, N)
    Gd = t(diag_supports(rng, (B if dyn else 1) * K, N).reshape(shape))
    Go = t(diag_supports(rng, B * K, N).reshape(shape)) if dyn else Gd
    W = t((rng.standard_normal((K * K * C, C)) * (2.0 / (K * K * C + C)) ** 0.5).astype(np.float32))
    cuda = shard.CudaEngine()
    total = torch.zeros(B, N, N, C, dtype=torch.float64, device=dev)
    for r in range(world):
        plan = shard.ShardPlan("row", r, world, N, K)
        pre, _ = cuda.forward_part(X[:, plan.row_lo:plan.row_hi].contiguous(), Go, Gd, dyn, W, N, plan.row_lo, K, K, 1, False)
        total += pre.double()
    whole, _ = abi.forward(X, Go, Gd, W, torch.zeros(C, device=dev), False, "fp16", want_saved=False)
    _check(total, whole, 1e-5, f"row shard N={N} x{world} {'dyn' if dyn else 'static'}/diag fp16: sum of partials == fp16 whole layer")


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def _masked(d, out):
    return torch.where(out > 0, d, torch.zeros_like(d))


def _check_db(db, d_pre, what):
    """db [H] against the float64 per-channel sum of d_pre [..., H], relative to the sum of magnitudes"""
    x = d_pre.double().reshape(-1, d_pre.shape[-1])
    err = (db.double() - x.sum(0)).abs()
    assert bool((err <= 2e-6 * x.abs().sum(0) + 1e-30).all()), f"{what}: db error {float(err.max()):.3e}"


def test_bias_act_and_relu_backward_kernels(cuda_device):
    """`mpgcn_bias_act` and `mpgcn_relu_backward` at widths 1 .. 1024; offset 1 places the tensors one float past a 16-byte boundary,
    which takes the scalar kernels"""
    eng = shard.CudaEngine()
    for H, offset in ((1, 0), (3, 0), (32, 0), (96, 0), (1024, 0), (32, 1)):
        torch.manual_seed(H)
        shape = (3, 17, 19, H)

        def at(t):      # a copy of t starting `offset` floats into its allocation
            v = torch.empty(t.numel() + offset, device=cuda_device)[offset:].view(t.shape)
            return v.copy_(t)

        x = torch.randn(shape, device=cuda_device)
        b = torch.randn(H, device=cuda_device)
        want = torch.relu(x + b)
        assert torch.equal(_bits(eng.bias_act(at(x), b, 1)), _bits(want)), f"H={H} offset={offset}: bias + ReLU"
        assert torch.equal(_bits(eng.bias_act(at(x), None, 0)), _bits(x)), f"H={H} offset={offset}: identity"
        d = torch.randn_like(x)
        d_pre, db = eng.relu_backward(at(d), at(want), 1, True)
        assert torch.equal(_bits(d_pre), _bits(_masked(d, want))), f"H={H} offset={offset}: masked dOut"
        _check_db(db, _masked(d, want), f"H={H} offset={offset}")


@pytest.mark.parametrize("kind,peer", [("row", True), ("row", False), ("k", False)])
def test_sharded_model_nccl_world2(kind, peer, tmp_path):
    """The sharded model on 2 GPUs vs the whole model on one GPU: fp32 engine <= 1e-5 forward (2e-3 rel_L2 gradients: summation
    order + the handful of ReLU-mask flips at fp32 noise level), fp16 engine <= 1e-3 forward.  Row shard: once with the exchange
    inside our own kernels over NVLink peer memory (symmetric memory), once with the NCCL collectives."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    res = nccl_worker.run(2, tmp_path, kind=kind, peer=peer)
    if peer:
        assert res["peer_exchange"], "symmetric-memory peer exchange could not be enabled on this box (the NCCL path is tested separately)"
    for row in res["rows"]:
        record_parity(row["what"], row["linf"], row["l2"], row["tol"])
        assert row["err"] <= row["tol"], row


def test_peer_exchange_kernels_on_one_gpu(cuda_device):
    """`mpgcn_rows_reduce_bias_act`, `mpgcn_relu_backward_scatter(_f16)` and the prepared-fp16-dPre entry of `backward_part`, with the g
    "ranks'" buffers all on one GPU (the kernels only see pointers): reduce-scatter + bias + ReLU, mask + all-gather, and the fp16
    flavour bit-identical to the fp32 route through the library's own cast.  The exchange steps at layer widths 32, 96 (an LSTM
    width) and 100 (not a multiple of 32); the fp16 backward_part at 32."""
    dev = cuda_device
    B, N, g, K = 2, 136, 4, 3
    rows, r = N // g, 2
    eng = shard.CudaEngine()
    for H in (32, 96, 100):
        torch.manual_seed(3)
        parts = [torch.randn(B, N, N, H, device=dev) for _ in range(g)]
        bias = torch.randn(H, device=dev)
        for rr in range(g):
            out = eng.rows_reduce_bias_act([p.data_ptr() for p in parts], B, N, rr * rows, rows, H, bias, 1, dev)
            want = torch.relu(torch.stack([p[:, rr * rows:(rr + 1) * rows] for p in parts]).sum(0) + bias)
            torch.testing.assert_close(out, want, rtol=1e-6, atol=1e-6, msg=lambda m: f"H={H} rows_reduce_bias_act: {m}")
        del parts
        # scatter (fp32): every destination receives the masked rows, nothing else is touched
        d_out = torch.randn(B, rows, N, H, device=dev) * 1e-5
        out_slab = torch.relu(torch.randn(B, rows, N, H, device=dev))
        dsts = [torch.full((B, N, N, H), 7.0, device=dev) for _ in range(g)]
        db = eng.relu_backward_scatter(d_out, out_slab, 1, [d.data_ptr() for d in dsts], N, r * rows, True)
        want = _masked(d_out, out_slab)
        for d in dsts:
            assert torch.equal(_bits(d[:, r * rows:(r + 1) * rows]), _bits(want)), f"H={H}: scattered rows"
            assert float((d[:, :r * rows] - 7.0).abs().max()) == 0.0 and float((d[:, (r + 1) * rows:] - 7.0).abs().max()) == 0.0, \
                f"H={H}: rows outside the slab were written"
        _check_db(db, want, f"H={H} scatter")
        del dsts
        # scatter (fp16): S = 2^k with S * absmax in [16, 32)
        amax = eng.absmax(d_out)
        assert float(amax) == float(d_out.abs().max())
        dsts16 = [torch.zeros(B, N, N, H, device=dev, dtype=torch.float16) for _ in range(g)]
        db16, scale2 = eng.relu_backward_scatter_f16(d_out, out_slab, 1, [d.data_ptr() for d in dsts16], N, r * rows, True, amax)
        S = float(scale2[0])
        assert 16.0 <= S * float(amax) < 32.0 and abs(np.log2(S) - round(np.log2(S))) < 1e-9 and float(scale2[1]) == 1.0 / S
        for d in dsts16:
            assert torch.equal(_bits(d[:, r * rows:(r + 1) * rows]), _bits((want * S).to(torch.float16))), f"H={H}: fp16 scattered rows"
        _check_db(db16, want, f"H={H} scatter_f16")
        torch.testing.assert_close(db16, db, rtol=1e-5, atol=1e-9)
    # backward_part fed the prepared fp16 dPre == backward_part casting the fp32 dPre itself (same S, same bits)
    H = 32
    out_slab = torch.relu(torch.randn(B, rows, N, H, device=dev))
    X = torch.tanh(torch.randn(B, rows, N, 32, device=dev))
    G = torch.randn(K, N, N, device=dev) / N ** 0.5
    W = torch.randn(K * K * 32, 32, device=dev) * 0.05
    _, saved = eng.forward_part(X, G, G, False, W, N, r * rows, K, K, 1, True)
    d_pre = torch.randn(B, N, N, H, device=dev) * 1e-5
    am = eng.absmax(d_pre)
    full16 = torch.zeros(B, N, N, H, device=dev, dtype=torch.float16)
    sc = None
    for rr in range(g):       # fill the "gathered" fp16 tensor slab by slab, as g ranks would
        _, sc = eng.relu_backward_scatter_f16(d_pre[:, rr * rows:(rr + 1) * rows].contiguous(), out_slab, 0, [full16.data_ptr()], N, rr * rows, False, am)
    dX_a, dW_a = eng.backward_part(d_pre, G, G, False, W, saved, N, r * rows, rows, K, K, 32, 1, True)
    dX_b, dW_b = eng.backward_part(None, G, G, False, W, saved, N, r * rows, rows, K, K, 32, 1, True, d_pre16=full16, scale2=sc)
    assert torch.equal(dX_a, dX_b) and torch.equal(dW_a, dW_b)


def test_hybrid_row_x_batch_shard_nccl_world4(tmp_path):
    """world 4 = 2 batch groups x 2 row ranks (bench.py --shard row --row-ranks 2) on 4 GPUs: the row exchange (peer memory) stays
    inside a group, the gradients are summed over all ranks and averaged over the groups; vs the whole model on one GPU.
    (Round 2, 4 GPUs, K = 4 dense supports: fp32 engine y 1.3e-6, every gradient inside its bound; fp16 engine y rel_L2 8.4e-4 with
    rel_Linf 8.9e-4 .. 1.02e-3 on a slab -- the fp16 engine's own error at K = 4 dense supports, the K shard measures the same on the
    whole output -- hence K = 3 here, like the world-2 row test.)"""
    if torch.cuda.device_count() < 4:
        pytest.skip("needs four GPUs")
    res = nccl_worker.run(4, tmp_path, kind="rowhyb", peer=True)
    for row in res["rows"]:
        record_parity(row["what"], row["linf"], row["l2"], row["tol"])
        assert row["err"] <= row["tol"], row
