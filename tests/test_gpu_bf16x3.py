"""Precision 2, "bf16x3", of the BDGCN layer on the GPU (DESIGN.md section 3): every operand a bf16 hi / lo pair, three products
per contraction on the tensor cores.

  * the layer fixtures of the unmodified reference, static and dynamic, K up to 11, C != H: forward within 1e-4 (rel_Linf and
    rel_L2), dX / dW / db within 2e-4 of the float64 oracle on the engine's ReLU mask;
  * at size: N = 1000, K = 3, C = H = 32 and N = 500, C = H = 128 against the oracle;
  * the whole model at hidden 128 (mpgcnw_* fixture) within the project's 1e-3 forward gate, and the mpgcn_* model fixtures;
  * training-mode behaviour: no stash under torch.no_grad(), CUDA-graph rollout equal to the eager loop, bitwise repeats in
    the deterministic mode."""
import numpy as np
import pytest
import torch

import test_gpu_at_size as at_size
import test_gpu_lstm_widths as widths
from conftest import golden_names, load_golden, record_parity
from oracle import mpgcn_oracle as orc
from oracle.gen_golden import layer_fixture
from test_oracle_golden import load_big

from mpgcn_b200 import _lib, ops

pytestmark = pytest.mark.gpu

FWD_BAR, GRAD_BAR = 1e-4, 2e-4
MODEL_FWD_GATE = 1e-3           # BASELINE.md section 3.6


def _check(a, ref, tol, what, l2_only=False):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    ref = ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol), f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"


def _f64(a):
    return tuple(x.astype(np.float64) for x in a) if isinstance(a, tuple) else a.astype(np.float64)


def _layer(X, G, W, b, d_out, relu, dev, precision="bf16x3"):
    """forward + backward of ops.bdgcn -> numpy (out, dX, dW, db)."""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    Xt = t(X).requires_grad_(True)
    Wt = t(W).requires_grad_(True)
    bt = None if b is None else t(b).requires_grad_(True)
    Gt = (t(G[0]), t(G[1])) if isinstance(G, tuple) else t(G)
    out = ops.bdgcn(Xt, Gt, Wt, bt, relu, precision=precision)
    out.backward(t(d_out))
    torch.cuda.synchronize()
    return [None if a is None else a.detach().cpu().numpy() for a in (out, Xt.grad, Wt.grad, None if bt is None else bt.grad)]


def _tc_fixtures():
    names = golden_names("bdgcn_") + golden_names("wide_bdgcn_") + golden_names("many_bdgcn_")
    return [n for n in names if all(d % 32 == 0 for d in (layer_fixture(load_golden(n))["X"].shape[-1], layer_fixture(load_golden(n))["W"].shape[1]))]


def test_fixture_set_covers_static_dynamic_many_supports_and_unequal_widths():
    gs = [layer_fixture(load_golden(n)) for n in _tc_fixtures()]
    assert {int(g["dynamic"]) for g in gs} == {0, 1} and max(int(g["K"]) for g in gs) >= 11
    assert any(g["X"].shape[-1] != g["W"].shape[1] for g in gs)


@pytest.mark.parametrize("name", _tc_fixtures())
def test_layer_matches_reference_fixture(name, cuda_device):
    g = layer_fixture(load_golden(name))
    G = (g["G_o"], g["G_d"]) if int(g["dynamic"]) else g["G"]
    act = str(g["act"])
    b = g.get("b")
    out, dX, dW, db = _layer(g["X"], G, g["W"], b, g["d_out"], act == "relu", cuda_device)
    _check(out, g["out"], FWD_BAR, f"{name}/bf16x3/out vs reference")
    refs = orc.bdgcn_backward_factored(_f64(g["X"]), _f64(G), _f64(g["W"]), None if b is None else _f64(b), act, _f64(g["d_out"]),
                                       mask_from=out)[1:]
    for a, r, k in zip((dX, dW, db), refs, ("dX", "dW", "db")):
        if r is not None:
            _check(a, r, GRAD_BAR, f"{name}/bf16x3/{k} (engine mask)")


@pytest.mark.parametrize("name", golden_names("big_bdgcn_"))
def test_layer_matches_big_reference_fixture(name, cuda_device):
    g, X, d_out, G = load_big(name)
    out, dX, dW, db = _layer(X, G, g["W"], g["b"], d_out, True, cuda_device)
    _check(out[:, g["rows"]], g["out_rows"], FWD_BAR, f"{name}/bf16x3/out rows vs reference")
    refs = orc.bdgcn_backward_factored(_f64(X), _f64(G), _f64(g["W"]), _f64(g["b"]), "relu", _f64(d_out), mask_from=out)[1:]
    for a, r, k in zip((dX, dW, db), refs, ("dX", "dW", "db")):
        _check(a, r, GRAD_BAR, f"{name}/bf16x3/{k} (engine mask)")


@pytest.mark.parametrize("N,K,B,dyn,kind,C", [(1000, 3, 1, False, "dense", 32), (500, 3, 1, True, "rw", 128), (300, 11, 1, False, "rw", 32),
                                              (129, 4, 2, True, "dense", 64)])
def test_layer_matches_oracle_at_size(N, K, B, dyn, kind, C, cuda_device):
    """The oracle comparison of test_gpu_at_size.py, in bf16x3.  (The oracle runs in float64 up to N = 300, in float32 BLAS above,
    whose own summation error, ~1e-6, is far below the bars.)"""
    rng = np.random.default_rng(1000 * N + 10 * K + dyn + C)
    H = C
    X = np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32)
    G = (at_size._supports(rng, kind, K, N, B), at_size._supports(rng, kind, K, N, B)) if dyn else at_size._supports(rng, kind, K, N, 0)
    W = (rng.standard_normal((K * K * C, H)) * (2.0 / (K * K * C + H)) ** 0.5).astype(np.float32)
    b = (rng.standard_normal(H) * 0.1).astype(np.float32)
    d_out = (rng.standard_normal((B, N, N, H)) * 1e-5).astype(np.float32)
    cast = (lambda a: a.astype(np.float64)) if N <= 300 else (lambda a: a)
    Gc = tuple(cast(a) for a in G) if dyn else cast(G)
    out, dX, dW, db = _layer(X, G, W, b, d_out, True, cuda_device)
    tag = f"layer N={N} K={K} B={B} C=H={C} {'dyn' if dyn else 'static'}/{kind}/bf16x3"
    out_o = orc.bdgcn_forward_factored(cast(X), Gc, cast(W), cast(b), "relu")
    _check(out, out_o, FWD_BAR, f"{tag}/out vs oracle")
    refs = orc.bdgcn_backward_factored(cast(X), Gc, cast(W), cast(b), "relu", cast(d_out), mask_from=out)[1:]
    for a, r, k in zip((dX, dW, db), refs, ("dX", "dW", "db")):
        _check(a, r, GRAD_BAR, f"{tag}/{k} (engine mask)")


@pytest.mark.parametrize("name", golden_names("mpgcnw_"))
def test_model_at_hidden_128_meets_the_forward_gate(name, cuda_device):
    """bf16x3 layers behind the tensor-core LSTM ("bf16x3" reads as "auto" for the LSTM): the forward within the project's 1e-3
    gate of the reference (rel_L2; rel_Linf recorded), which the fp16 layers miss here (DESIGN.md section 3); gradients against the
    oracle on the engine's ReLU masks as the fp16 model is held (5e-3)."""
    g = load_golden(name)
    params = widths._model_params(g)
    y, grads, grads_m = widths._run_fixture_model(g, params, "bf16x3", "bf16x3", cuda_device)
    _check(y, g["y"], MODEL_FWD_GATE, f"{name}/bf16x3/y", l2_only=True)
    for k, v in grads.items():
        _check(v, grads_m[k], widths.MODEL_GRAD_TOL, f"{name}/bf16x3/grad:{k} (engine masks)", l2_only=True)


@pytest.mark.parametrize("name", golden_names("mpgcn_"))
def test_model_fixtures(name, cuda_device):
    """The reference's model checkpoints with every layer in bf16x3 (the LSTM as under "auto"): the forward within the 1e-3 gate of
    the reference in rel_L2, gradients against the oracle on the engine's ReLU masks (5e-3, as the fp16 model)."""
    import MPGCN as shim
    from torch import nn
    g = load_golden(name)
    K, hid = int(g["K"]), int(g["hidden"])
    if hid % 32:
        pytest.skip(f"hidden {hid}: the tensor-core layers take multiples of 32")
    N = g["x_seq"].shape[2]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    params = {k[6:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("param:")}
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU)
    model.load_state_dict(params)
    model = model.to(cuda_device)
    at_size._set_precision(model, "bf16x3")
    caps = {m: {"layers": [], "fc": None} for m in range(2)}
    hooks = [layer.register_forward_hook(lambda mod, inp, out, m=m: caps[m]["layers"].append(out.detach().cpu().numpy()))
             for m in range(2) for layer in model.branch_models[m]['spatial']]
    y = model(x_seq=t(g["x_seq"]), G_list=[t(g["G_static"]), (t(g["G_o"]), t(g["G_d"]))])
    y.backward(t(g["d_y"]))
    torch.cuda.synchronize()
    for h in hooks:
        h.remove()
    for m in range(2):
        fc = model.branch_models[m]['fc'][0]
        caps[m]["fc"] = orc.fc_relu_forward(caps[m]["layers"][-1], fc.weight.detach().cpu().numpy(), fc.bias.detach().cpu().numpy())
    _check(y, g["y"], MODEL_FWD_GATE, f"{name}/bf16x3/y", l2_only=True)
    params_np = {k[6:]: v for k, v in g.items() if k.startswith("param:")}
    _, grads_m = orc.mpgcn_forward_backward(params_np, g["x_seq"], [g["G_static"], (g["G_o"], g["G_d"])], M=2, gcn_num_layers=3,
                                            d_y=g["d_y"], masks=caps)
    for k, p in model.named_parameters():
        _check(p.grad, grads_m[k], widths.MODEL_GRAD_TOL, f"{name}/bf16x3/grad:{k} (engine masks)", l2_only=True)


def _small_model(dev):
    return widths._model(23, 3, 32, 3, dev)


def test_no_grad_allocates_no_stash_and_graph_rollout_equals_eager(cuda_device):
    from mpgcn_b200 import rollout
    dev = cuda_device
    N, K, B, T, P = 23, 3, 2, 5, 3
    model = _small_model(dev)
    at_size._set_precision(model, "bf16x3")
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
    assert torch.equal(eager, graphed)


@pytest.mark.parametrize("dyn", [False, True])
def test_deterministic_backward_repeats_bitwise(dyn, cuda_device):
    dev = cuda_device
    rng = np.random.default_rng(7 + dyn)
    B, N, K, C, H = 2, 150, 3, 64, 32
    X = np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32)
    G = (at_size._supports(rng, "dense", K, N, B), at_size._supports(rng, "dense", K, N, B)) if dyn else at_size._supports(rng, "dense", K, N, 0)
    W = (rng.standard_normal((K * K * C, H)) * 0.05).astype(np.float32)
    b = (rng.standard_normal(H) * 0.1).astype(np.float32)
    d_out = (rng.standard_normal((B, N, N, H)) * 1e-4).astype(np.float32)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = [_layer(X, G, W, b, d_out, True, dev) for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, c in zip(*runs):
        assert np.array_equal(a, c)


def test_profile_tags_report_algorithmic_flops(cuda_device):
    """The stage tags count the flops of the algorithm, the same in every precision (not the three products of bf16x3)."""
    dev = cuda_device
    rng = np.random.default_rng(3)
    B, N, K, C, H = 1, 100, 2, 32, 64
    X = rng.standard_normal((B, N, N, C)).astype(np.float32)
    G = at_size._supports(rng, "dense", K, N, 0)
    W = (rng.standard_normal((K * K * C, H)) * 0.05).astype(np.float32)
    d_out = rng.standard_normal((B, N, N, H)).astype(np.float32)
    flops = {}
    for prec in ("fp16", "bf16x3"):
        _lib.load().mpgcn_profile_reset()
        _layer(X, G, W, None, d_out, True, dev, precision=prec)
        flops[prec] = {k: v["flops"] for k, v in _lib.profile_read().items() if k in _lib.PROFILE_TAGS[:7]}
    assert flops["fp16"] == flops["bf16x3"] and all(v > 0 for v in flops["bf16x3"].values())
