"""The tensor-core BDGCN layer (precision 1) with more than 8 supports.

The trainer builds K = k + 1 supports for Chebyshev / random-walk diffusion of order k and 2k + 1 for dual random-walk
diffusion, so `-kernel dual_random_walk_diffusion -K 4` already gives 9.  Beyond 8 supports the engine splits what one tile
cannot hold: the channel mixes evaluate their output supports in ceil(Kout / 8) balanced groups, BWD_DW tiles its Ko chunks in
column groups, and the FWD_B epilogue walks its diagonal remainders 8 segments at a time (DESIGN.md section 6.1).

  * CPU: the oracle against fixtures of the unmodified reference with 9 and 11 dual random-walk supports
    (`tests/golden/many_bdgcn_*`, tools/gen_golden_many.py); the host-side shape checks.
  * GPU: every stage against float64 (the helpers and bounds of test_gpu_engine_stages.py) at K = 9 .. 17, plus the
    remainder of supports 8 and up on its own; the layer against the fixtures and the factored oracle; the whole model on
    dual random-walk supports; a row shard.
"""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

import abi
import test_gpu_at_size as at_size
from conftest import golden_names, load_golden, record_parity
from oracle import mpgcn_oracle as orc
from oracle.gen_golden import layer_fixture
from test_gpu_engine_stages import Slope, _assert_and_record, _inputs, check_stages, diag_supports, run_layer

import GCN as gshim
import MPGCN as shim
from mpgcn_b200 import _lib, shard

FIXTURE_TOL = 2e-5      # oracle vs reference fixtures (as tests/test_oracle_golden.py)
FWD_TOL = {"fp32": 5e-5, "fp16": 1e-3}
BWD_TOL = {"fp32": 2e-4, "fp16": 2e-3}
LOOSE_FP16_GRAD = 8e-2  # fp16 gradients against another ReLU mask (DESIGN.md section 3)


def _rel_check(a, ref, tol, what, l2_only=False):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    ref = ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol), f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"


def _graph(g):
    return (g["G_o"], g["G_d"]) if int(g["dynamic"]) else g["G"]


# ------------------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------------------
def test_many_support_fixtures_exist_and_stay_out_of_the_small_layer_set():
    names = golden_names("many_bdgcn_")
    assert len(names) >= 3 and max(int(load_golden(n)["K"]) for n in names) >= 11
    assert not set(names) & set(golden_names("bdgcn_")) and not set(names) & set(golden_names("big_bdgcn_"))


@pytest.mark.parametrize("name", golden_names("many_bdgcn_"))
def test_oracle_matches_reference_with_many_supports(name):
    g = layer_fixture(load_golden(name))
    assert int(g["K"]) > 8 and g["W"].shape == (int(g["K"]) ** 2 * 32, 32)
    out = orc.bdgcn_forward(g["X"], _graph(g), g["W"], g["b"], "relu")
    _rel_check(out, g["out"], FIXTURE_TOL, f"{name}: out")
    dX, dW, db = orc.bdgcn_backward(g["X"], _graph(g), g["W"], g["b"], "relu", g["d_out"])
    for a, k in ((dX, "dX"), (dW, "dW"), (db, "db")):
        _rel_check(a, g[k], FIXTURE_TOL, f"{name}: {k}")
    fac = orc.bdgcn_backward_factored(g["X"], _graph(g), g["W"], g["b"], "relu", g["d_out"])
    for a, k in zip(fac, ("out", "dX", "dW", "db")):
        _rel_check(a, g[k], FIXTURE_TOL, f"{name}: factored {k}")


@pytest.mark.parametrize("K", [9, 16, 17])
def test_tensor_path_accepts_more_than_eight_supports(K):
    lib = _lib.load()
    assert lib.mpgcn_bdgcn_precision_supported(2, 50, K, 32, 32, 1) == 1
    assert lib.mpgcn_bdgcn_precision_supported(2, 50, K, 16, 32, 1) == 0
    assert lib.mpgcn_bdgcn_precision_supported(2, 50, K, 32, 16, 1) == 0
    from mpgcn_b200 import ops
    assert ops.resolve_precision("auto", 2, 50, K, 32, 32) == _lib.PREC_FP16_TC
    assert ops.resolve_precision("fp16", 2, 50, K, 32, 32) == _lib.PREC_FP16_TC
    with pytest.raises(RuntimeError, match="C == H == 32"):
        ops.resolve_precision("fp16", 2, 50, K, 16, 32)


def test_layer_part_with_nine_supports_passes_validation():
    """check_part runs before any pointer is looked at: a Ko = 9 part gets as far as the null-pointer check, a C = 16 one does not."""
    lib = _lib.load()
    one = ctypes.c_void_p(256)

    def err():
        return lib.mpgcn_last_error().decode()
    for Ko, Kd in ((9, 9), (9, 5), (17, 3)):
        part = _lib.BdgcnPart(0, 4, Ko, Kd)
        rc = lib.mpgcn_bdgcn_forward_part(one, one, one, 0, one, None, None, one, 1 << 20, 2, 8, 32, 32, 1, ctypes.addressof(part), None, None)
        assert rc != 0 and "null pointer" in err(), err()
        assert lib.mpgcn_bdgcn_part_saved_bytes(2, 8, 32, 32, 1, ctypes.addressof(part)) == 2 * Kd * 4 * 8 * 32 * 2
    part = _lib.BdgcnPart(0, 4, 9, 9)
    rc = lib.mpgcn_bdgcn_forward_part(one, one, one, 0, one, one, None, one, 1 << 20, 2, 8, 16, 32, 1, ctypes.addressof(part), None, None)
    assert rc != 0 and "C == H == 32" in err()


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: every stage against float64
# ------------------------------------------------------------------------------------------------------------------------------
def _make_cases():
    rows = []          # (N, K, B, dyn, kind, grad)
    shapes = ([(130, K, 2, None) for K in (9, 10, 12, 16, 17)]          # mix groups 5+4, 5+5, 6+6, 8+8, 6+6+5; dW column tiles
              + [(N, 9, 2, None) for N in (1, 65, 257)]                 # tile edges
              + [(130, 17, 3, True),                                    # odd batch
                 (1000, 9, 1, False)])                                  # at size
    for i, (N, K, B, only) in enumerate(shapes):
        for dyn in ((False, True) if only is None else (only,)):
            kind = "diag" if (i + dyn) % 2 == 0 else "dense"
            grad = 1e4 if (i + 2 * dyn) % 3 == 1 else 1e-5
            rows.append((N, K, B, dyn, kind, grad))
    return rows


CASES = _make_cases()


def test_stage_cases_cover_both_kinds_and_both_gradient_scales_at_every_k():
    for K in (9, 10, 12, 16, 17):
        rows = [c for c in CASES if c[1] == K]
        assert {c[4] for c in rows} == {"diag", "dense"}, K
        assert {c[3] for c in rows} == {False, True}, K
    assert {c[5] for c in CASES} == {1e-5, 1e4}
    assert any(c[1] == 17 and c[2] % 2 == 1 for c in CASES)


def _high_segment_remainder_slope(r, bias, B, N, dyn):
    """The FWD_B remainder of supports 8 .. K-1 on its own: the kernel's deviation from the product plus the remainders of
    supports 0..7 must have slope 1 on the remainders of the rest (0 when the epilogue stops after 8 segments)."""
    go16 = r["go16"][..., :N].double()
    dgo, out = r["dgo"].double(), r["out"]
    s = Slope()
    for b in range(B):
        zb = b if dyn else 0
        for e0 in range(0, N, 32):
            es = slice(e0, min(N, e0 + 32))
            u = r["u16"][b, :, :, es].double()         # [o][n][e][h]; the remainder of support o at destination m reads row n = m
            base = torch.einsum("onm,oneh->meh", go16[zb], u) + bias.double()
            lo = torch.einsum("om,omeh->meh", dgo[zb, :8], u[:8])
            hi = torch.einsum("om,omeh->meh", dgo[zb, 8:], u[8:])
            y = out[b, :, es].double()
            s.add((y - base - lo) * (y > 0), hi * (y > 0))
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,B,dyn,kind,grad", CASES)
def test_every_stage_matches_float64_with_many_supports(N, K, B, dyn, kind, grad, cuda_device):
    X, Go, Gd, W, bias = _inputs(N, K, B, dyn, kind, 7919 * N + 31 * K + 2 * B + dyn + 5, cuda_device)
    d_out = torch.randn(B, N, N, 32, device=cuda_device, generator=torch.Generator(cuda_device).manual_seed(N + K + 1)) * grad
    r = run_layer(X, Go, Gd, W, bias, d_out, dyn)
    tag = f"N={N} K={K} B={B} {'dyn' if dyn else 'static'}/{kind} |dOut|~{grad:g}"
    res = check_stages(r, X, Go, Gd, W, bias, d_out, dyn, tag, kind)
    s = _high_segment_remainder_slope(r, bias, B, N, dyn)
    res["FWD_B remainder slope, supports 8+"] = s
    if kind == "diag" and N >= 130:
        assert s.judged, f"{tag}: only {s.n} remainder terms of supports 8+"
    _assert_and_record(res, tag)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: end to end
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("many_bdgcn_"))
def test_layer_matches_reference_fixture_with_many_supports(name, cuda_device):
    g = layer_fixture(load_golden(name))
    X, G, W, b, d_out = g["X"], _graph(g), g["W"], g["b"], g["d_out"]
    for prec in ("fp32", "fp16"):
        out, dX, dW, db = at_size._run_layer(X, G, W, b, d_out, prec, cuda_device)
        _rel_check(out, g["out"], FWD_TOL[prec], f"{name}/{prec}/out vs reference")
        if prec == "fp32":
            for a, k in ((dX, "dX"), (dW, "dW"), (db, "db")):
                _rel_check(a, g[k], BWD_TOL[prec], f"{name}/{prec}/{k} vs reference")
        else:
            refs = orc.bdgcn_backward_factored(X.astype(np.float64), tuple(a.astype(np.float64) for a in G) if isinstance(G, tuple)
                                               else G.astype(np.float64), W.astype(np.float64), b.astype(np.float64), "relu",
                                               d_out.astype(np.float64), mask_from=out)[1:]
            for a, ref, k in zip((dX, dW, db), refs, ("dX", "dW", "db")):
                _rel_check(a, ref, BWD_TOL[prec], f"{name}/{prec}/{k} (engine mask)")
                _rel_check(a, g[k], LOOSE_FP16_GRAD, f"{name}/{prec}/{k} vs reference", l2_only=True)


@pytest.mark.gpu
@pytest.mark.parametrize("N,K,B,dyn,kind", [
    (200, 9, 2, False, "diag"), (200, 12, 2, True, "dense"), (200, 17, 1, False, "rw"),
    (500, 9, 1, True, "rw"), (500, 12, 1, False, "diag"), (500, 17, 1, False, "dense"),
])
def test_layer_matches_oracle_with_many_supports(N, K, B, dyn, kind, cuda_device):
    """The at-size oracle comparison of test_gpu_at_size.py (forward <= 1e-3, gradients <= 2e-3 against the oracle on the
    engine's ReLU mask, for fp32 and fp16), at 9, 12 and 17 supports."""
    at_size.test_layer_matches_oracle_at_size(N, K, B, dyn, kind, cuda_device)


def _run_model(model, x_seq, G_list, d_y, prec):
    at_size._set_precision(model, prec)
    model.zero_grad(set_to_none=True)
    y = model(x_seq=x_seq, G_list=G_list)
    y.backward(d_y)
    torch.cuda.synchronize()
    return y.detach().clone(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}


@pytest.mark.gpu
@pytest.mark.parametrize("order", [2, 3, 4])
def test_model_on_dual_random_walk_supports_fp16_matches_fp32(order, cuda_device):
    """The whole model with the trainer's `dual_random_walk_diffusion` supports of order 4 (K = 9; orders 2 and 3, K = 5 and 7,
    for comparison): static graph and dynamic graphs, forward and backward, the fp16 tensor-core engine against the fp32 engine.
    The forward is held to 1e-3 in rel_L2 (its rel_Linf, recorded in the parity report, is above 1e-3 on this model at K = 5
    already); gradients to 8e-2 in rel_L2 (another forward's ReLU mask, DESIGN.md section 3).  The default init can leave a
    branch's FC ReLU dead, so the first seed whose fp32 run gives every parameter a gradient is used."""
    dev = cuda_device
    N, T, B, K = 40, 4, 2, 2 * order + 1
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    proc = gshim.Adj_Processor("dual_random_walk_diffusion", order)
    assert proc.num_supports() == K
    for seed in range(99, 2000, 100):
        rng = np.random.default_rng(seed)
        torch.manual_seed(seed)
        g_static = proc.process(t(rng.random((1, N, N)).astype(np.float32)))[0]
        G_list = [g_static, (proc.process(t(rng.random((B, N, N)).astype(np.float32))), proc.process(t(rng.random((B, N, N)).astype(np.float32))))]
        assert tuple(g_static.shape) == (K, N, N) and tuple(G_list[1][0].shape) == (B, K, N, N)
        model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=32, lstm_num_layers=1, gcn_hidden_dim=32, gcn_num_layers=3,
                           num_nodes=N, user_bias=True, activation=nn.ReLU).to(dev)
        x_seq = t((rng.random((B, T, N, N, 1)) * 8).astype(np.float32))
        d_y = t(rng.standard_normal((B, 1, N, N, 1)).astype(np.float32))
        y32, g32 = _run_model(model, x_seq, G_list, d_y, "fp32")
        if all(float(g.abs().max()) > 0 for g in g32.values()):
            break
    else:
        pytest.fail("no seed gives both branches a gradient")
    y16, g16 = _run_model(model, x_seq, G_list, d_y, "fp16")
    _rel_check(y16, y32, FWD_TOL["fp16"], f"model K={K} dual random walk (seed {seed}): fp16 y vs fp32", l2_only=True)
    for k, g in g32.items():
        _rel_check(g16[k], g, LOOSE_FP16_GRAD, f"model K={K} dual random walk: fp16 grad:{k} vs fp32", l2_only=True)


@pytest.mark.gpu
@pytest.mark.parametrize("N,dyn", [(130, False), (258, True)])
def test_row_shard_with_nine_supports_sums_to_the_whole_layer(N, dyn, cuda_device):
    """Row shard over 2 ranks at K = 9 on supports whose diagonal remainders fire: the fp16 partial pre-activations summed equal
    the fp16 whole layer to 1e-5 (as test_gpu_shard.py at K = 3), so the slab path's mixes and remainders of supports 8+ agree."""
    dev = cuda_device
    rng = np.random.default_rng(N + 9)
    B, K, C, world = 2, 9, 32, 2
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
    _rel_check(total, whole.double(), 1e-5, f"row shard K=9 N={N} x{world} {'dyn' if dyn else 'static'}/diag fp16: sum of partials == whole")
