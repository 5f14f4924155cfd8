"""Gradients with respect to the supports G of a BDGCN layer (`support_grad=True`), in both kernel families.

CPU: the float64 factored dG (tests/support_grad_oracle.py) against the reference's autograd fixtures `sgrad_*`, the C-ABI
surface of the new entry point and its argument checks.  GPU: the engine's dG against float64 at ragged sizes, supports counts
and channel widths, at size, against the fixtures (layer and whole model), unchanged dX / dW / db / out, the default refusal,
re-staging of a learnable support after an optimiser step, a few Adam steps against the reference model, and the whole model's dG
against float64 on the engine's own ReLU masks in both precisions.  The dG stages in isolation: test_gpu_support_grad_stages.py.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch
from torch import nn

from conftest import ROOT, golden_names, load_golden, record_parity
from oracle import mpgcn_oracle as orc
from oracle.gen_golden import layer_fixture
from support_grad_oracle import support_grads

import MPGCN as shim
from mpgcn_b200 import _lib, ops

TOL = {"fp32": 5e-5, "fp16": 2e-3}          # gradient tolerances of test_gpu_parity.py
LOOSE_FP16_GRAD = 8e-2                       # fp16 against the reference: a flipped ReLU mask element is an O(1) local change
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def _check(a, ref, tol, what, l2_only=False):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol), f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"


# ------------------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------------------
def test_fixture_prefix_is_its_own():
    names = golden_names("sgrad_")
    assert len([n for n in names if n.startswith("sgrad_bdgcn_")]) >= 7 and any(n.startswith("sgrad_mpgcn_") for n in names)
    for prefix in ("bdgcn_", "mpgcn_", "wide_", "many_", "big_", "lstm_", "lstms_", "mpgcns_", "adj_"):
        assert not set(names) & set(golden_names(prefix))
    for n in names:
        assert os.path.getsize(os.path.join(ROOT, "tests", "golden", n + ".npz")) < 1 << 20


@pytest.mark.parametrize("name", [n for n in golden_names("sgrad_bdgcn_")])
def test_float64_support_grad_matches_reference_fixture(name):
    g = layer_fixture(load_golden(name))
    dyn = int(g["dynamic"])
    G = (g["G_o"], g["G_d"]) if dyn else g["G"]
    ref = support_grads(g["X"], G, g["W"], g["b"], "relu", g["d_out"])
    if dyn:
        _check(ref[0], g["dG_o"], 1e-5, f"{name}/oracle dG_o")
        _check(ref[1], g["dG_d"], 1e-5, f"{name}/oracle dG_d")
    else:
        _check(ref, g["dG"], 1e-5, f"{name}/oracle dG")


def test_new_symbols_are_exported_and_bound():
    for sym in ("mpgcn_bdgcn_support_grad_workspace_bytes", "mpgcn_bdgcn_backward_supports"):
        assert sym in _lib.EXPORTED_SYMBOLS
        with open(os.path.join(ROOT, "include", "mpgcn_b200.h")) as f:
            assert sym + "(" in f.read()
    assert "BWD_DG" in _lib.PROFILE_TAGS and _lib.PROFILE_TAGS.index("BWD_DG") == len(_lib.PROFILE_TAGS) - 1
    lib = _lib.load()
    assert lib.mpgcn_abi_version() == 4
    for prec in (0, 1):
        for dyn in (0, 1):
            need = lib.mpgcn_bdgcn_support_grad_workspace_bytes(2, 33, 3, 64, 32, dyn, prec)
            assert need > lib.mpgcn_bdgcn_bwd_workspace_bytes(2, 33, 3, 64, 32, dyn, prec) > 0
    assert lib.mpgcn_bdgcn_support_grad_workspace_bytes(2, 33, 3, 48, 32, 0, 1) == 0      # no tensor-core layer at C = 48


def test_entry_point_rejects_bad_arguments_without_a_gpu():
    """Every case fails validation, which runs before any CUDA call: fake device addresses are never touched."""
    lib = _lib.load()
    B, N, K, C, H = 2, 9, 3, 32, 32
    p = 1 << 20                                   # a plausible, never dereferenced address
    ex = _lib.BdgcnExtras()

    def call(prec=1, dyn=0, ws_bytes=None, **kw):
        a = dict(d_out=p, out=p, go=p, gd=p, W=p, saved=p, dX=p, dW=p, db=p, ws=p, X=p, dGo=p, dGd=None)
        a.update(kw)
        if ws_bytes is None:
            ws_bytes = lib.mpgcn_bdgcn_support_grad_workspace_bytes(B, N, K, C, H, dyn, prec) - 1
        r = lib.mpgcn_bdgcn_backward_supports(a["d_out"], a["out"], a["go"], a["gd"], dyn, a["W"], 1, a["saved"], a["dX"], a["dW"], a["db"],
                                              a["ws"], ws_bytes, B, N, K, C, H, prec, ctypes.addressof(ex), a["X"], a["dGo"], a["dGd"], None)
        return r, lib.mpgcn_last_error().decode()

    for prec in (0, 1):
        r, msg = call(prec, X=None)
        assert r != 0 and "null pointer" in msg
        r, msg = call(prec, saved=None)
        assert r != 0 and "null pointer" in msg
        r, msg = call(prec, dGd=p)                     # static supports: one gradient, in dG_o
        assert r != 0 and "dG_d must be NULL" in msg
        r, msg = call(prec, dGo=None)
        assert r != 0 and "dG_d must be NULL" in msg
        r, msg = call(prec)                            # one byte short
        assert r != 0 and "workspace too small" in msg
        r, msg = call(prec, dyn=1, dGo=None, dGd=p)
        assert r != 0 and "workspace too small" in msg
    ex.d_pre_f16 = p                                   # a part's prepared dPre has no place in a whole-layer call
    r, msg = call(1, ws_bytes=1 << 40)
    assert r != 0 and "prepared fp16 dPre" in msg
    ex.d_pre_f16 = None
    r = lib.mpgcn_bdgcn_backward_supports(p, p, p, p, 0, p, 1, p, p, p, p, p, 1 << 40, B, N, K, 48, H, 1, None, p, p, None, None)
    assert r != 0 and "multiples of 32" in lib.mpgcn_last_error().decode()


# ------------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------------
def _inputs(seed, B, N, K, C, H, dyn, dev):
    rng = np.random.default_rng(seed)
    X = np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32)
    d_out = rng.standard_normal((B, N, N, H)).astype(np.float32)
    shape = (B, K, N, N) if dyn else (K, N, N)
    gs = [(rng.standard_normal(shape) / np.sqrt(N)).astype(np.float32) for _ in range(2 if dyn else 1)]
    W = (rng.standard_normal((K * K * C, H)) * np.sqrt(2.0 / (K * K * C + H))).astype(np.float32)
    b = (rng.standard_normal(H) * 0.1).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(dev)
    return X, (gs[0], gs[1]) if dyn else gs[0], W, b, d_out, t


def _run(X, G, W, b, d_out, prec, dev, support_grad=True, g_grad=True):
    """One layer forward + backward through ops.bdgcn -> (out, dX, dW, db, dG) with dG None / a tensor / a pair."""
    Xt = torch.from_numpy(X).to(dev).requires_grad_(True)
    Wt = torch.from_numpy(W).to(dev).requires_grad_(True)
    bt = torch.from_numpy(b).to(dev).requires_grad_(True)
    if isinstance(G, tuple):
        Gt = tuple(torch.from_numpy(g).to(dev).requires_grad_(g_grad) for g in G)
    else:
        Gt = torch.from_numpy(G).to(dev).requires_grad_(g_grad)
    out = ops.bdgcn(Xt, Gt, Wt, bt, relu=True, precision=prec, support_grad=support_grad)
    out.backward(torch.from_numpy(d_out).to(dev))
    torch.cuda.synchronize()
    dG = tuple(g.grad for g in Gt) if isinstance(Gt, tuple) else Gt.grad
    return out.detach(), Xt.grad, Wt.grad, bt.grad, dG


def _check_dg(dG, ref, tol, what):
    if isinstance(ref, tuple):
        _check(dG[0], ref[0], tol, what + "/dG_o")
        _check(dG[1], ref[1], tol, what + "/dG_d")
    else:
        _check(dG, ref, tol, what + "/dG")


LAYER_CASES = [
    # N, K, dynamic, C, H, B
    (1, 1, False, 32, 32, 2),
    (7, 3, False, 32, 32, 2),
    (7, 9, True, 32, 32, 2),
    (65, 3, True, 64, 32, 2),
    (65, 1, False, 32, 96, 3),
    (129, 3, False, 96, 64, 1),
    (129, 9, False, 32, 32, 1),
    (129, 3, True, 32, 32, 2),
    (200, 3, False, 32, 32, 2),
    (200, 1, True, 64, 96, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("N,K,dyn,C,H,B", LAYER_CASES)
def test_layer_support_grad_against_float64(N, K, dyn, C, H, B, prec, cuda_device):
    X, G, W, b, d_out, _ = _inputs(100 * N + 10 * K + int(dyn), B, N, K, C, H, dyn, cuda_device)
    out, dX, dW, db, dG = _run(X, G, W, b, d_out, prec, cuda_device)
    ref = support_grads(X, G, W, b, "relu", d_out, mask_from=out.cpu().numpy(), device=cuda_device)
    _check_dg(dG, ref, TOL[prec], f"sgrad N={N} K={K} dyn={dyn} C={C} H={H}/{prec}")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("dyn", [False, True])
def test_support_grad_at_size(dyn, prec, cuda_device):
    """N = 1000, K = 3, B = 2: sampled rows of dG (tile edges and a spread) against the factored float64 oracle."""
    B, N, K, C, H = 2, 1000, 3, 32, 32
    X, G, W, b, d_out, _ = _inputs(77 + int(dyn), B, N, K, C, H, dyn, cuda_device)
    out, _, _, _, dG = _run(X, G, W, b, d_out, prec, cuda_device)
    ref = support_grads(X, G, W, b, "relu", d_out, mask_from=out.cpu().numpy(), device=cuda_device)
    rows = np.asarray(sorted({0, 1, 31, 32, 63, 64, 127, 128, 255, 256, 511, 512, 767, 768, 895, 896, 998, 999} | set(range(5, N, 97))))
    if dyn:
        for got, want, side in ((dG[0], ref[0], "dG_o"), (dG[1], ref[1], "dG_d")):
            got = got.cpu().numpy()
            _check(got[:, :, rows], want[:, :, rows], TOL[prec], f"sgrad at size/{prec}/{side} rows")
            _check(got[:, :, :, rows], want[:, :, :, rows], TOL[prec], f"sgrad at size/{prec}/{side} columns")
    else:
        got = dG.cpu().numpy()
        _check(got[:, rows], ref[:, rows], TOL[prec], f"sgrad at size/{prec}/dG rows")
        _check(got[:, :, rows], ref[:, :, rows], TOL[prec], f"sgrad at size/{prec}/dG columns")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("N,K,dyn,C,H", [(65, 3, False, 32, 32), (33, 2, True, 64, 32), (129, 1, False, 32, 96)])
def test_other_results_unchanged_by_support_grad(N, K, dyn, C, H, prec, cuda_device):
    """out and dX (and the tensor-core dW): bitwise the same with the dG stages as without them, and support_grad=True with a G
    that does not require grad is exactly today's call.  db, and the fp32 path's split-K dW, are summed with atomics (their
    order varies from run to run, with or without the dG stages), so they are held to fp32 rounding."""
    X, G, W, b, d_out, _ = _inputs(5 + N, 2, N, K, C, H, dyn, cuda_device)
    base = _run(X, G, W, b, d_out, prec, cuda_device, support_grad=False, g_grad=False)
    with_dg = _run(X, G, W, b, d_out, prec, cuda_device, support_grad=True, g_grad=True)
    opted_in = _run(X, G, W, b, d_out, prec, cuda_device, support_grad=True, g_grad=False)
    exact = ("out", "dX", "dW") if prec == "fp16" else ("out", "dX")
    for i, what in enumerate(("out", "dX", "dW", "db")):
        for run, how in ((with_dg, "by the dG stages"), (opted_in, "by support_grad=True without a G that requires grad")):
            if what in exact:
                assert torch.equal(base[i], run[i]), f"{what} changed {how}"
            else:
                torch.testing.assert_close(run[i], base[i], rtol=1e-5, atol=1e-5 * float(base[i].abs().max()), msg=f"{what} changed {how}")
    none = lambda d: d is None or (isinstance(d, tuple) and all(x is None for x in d))
    assert not none(with_dg[4]) and none(opted_in[4])


@pytest.mark.gpu
def test_dynamic_pair_as_one_tensor_gets_the_sum(cuda_device):
    X, G, W, b, d_out, _ = _inputs(11, 2, 20, 3, 32, 32, True, cuda_device)
    Xt = torch.from_numpy(X).to(cuda_device)
    g = torch.from_numpy(G[0]).to(cuda_device).requires_grad_(True)
    y = ops.bdgcn(Xt, (g, g), torch.from_numpy(W).to(cuda_device), torch.from_numpy(b).to(cuda_device), relu=True, precision="fp32",
                  support_grad=True)
    y.backward(torch.from_numpy(d_out).to(cuda_device))
    G1 = (G[0], G[0])
    _, _, _, _, (a, c) = _run(X, G1, W, b, d_out, "fp32", cuda_device)
    torch.testing.assert_close(g.grad, a + c, rtol=1e-6, atol=1e-7)


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("sgrad_bdgcn_"))
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_layer_matches_reference_fixture(name, prec, cuda_device):
    g = layer_fixture(load_golden(name))
    dyn = int(g["dynamic"])
    K, C, H = int(g["K"]), int(g["C"]), int(g["H"])
    layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=H, use_bias=True, activation=nn.ReLU).to(cuda_device)
    layer.precision, layer.support_grad = prec, True
    with torch.no_grad():
        layer.W.copy_(torch.from_numpy(g["W"]))
        layer.b.copy_(torch.from_numpy(g["b"]))
    X = torch.from_numpy(g["X"]).to(cuda_device).requires_grad_(True)
    if dyn:
        G = tuple(torch.from_numpy(g[k]).to(cuda_device).requires_grad_(True) for k in ("G_o", "G_d"))
    else:
        G = torch.from_numpy(g["G"]).to(cuda_device).requires_grad_(True)
    out = layer(X, G)
    out.backward(torch.from_numpy(g["d_out"]).to(cuda_device))
    torch.cuda.synchronize()
    got = (G[0].grad, G[1].grad) if dyn else G.grad
    want = (g["dG_o"], g["dG_d"]) if dyn else g["dG"]
    if prec == "fp32":
        _check_dg(got, want, TOL[prec], f"{name}/{prec}")
    else:
        Gn = (g["G_o"], g["G_d"]) if dyn else g["G"]
        ref = support_grads(g["X"], Gn, g["W"], g["b"], "relu", g["d_out"], mask_from=out.detach().cpu().numpy())
        _check_dg(got, ref, TOL[prec], f"{name}/{prec} (engine mask)")
        if dyn:
            _check(got[0], want[0], LOOSE_FP16_GRAD, f"{name}/{prec}/dG_o vs reference", l2_only=True)
            _check(got[1], want[1], LOOSE_FP16_GRAD, f"{name}/{prec}/dG_d vs reference", l2_only=True)
        else:
            _check(got, want, LOOSE_FP16_GRAD, f"{name}/{prec}/dG vs reference", l2_only=True)


def _model(g, N, K, hid, prec, dev):
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU)
    if g is not None:
        model.load_state_dict({k[6:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("param:")})
    model = model.to(dev)
    model.lstm_precision = prec
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision, mod.support_grad = prec, True
    return model


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("sgrad_mpgcn_"))
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_model_matches_reference_fixture(name, prec, cuda_device):
    """The three layers of branch 0 share one learnable static support: their gradients add into one dG."""
    g = load_golden(name)
    K, hid, N = int(g["K"]), int(g["hidden"]), g["x_seq"].shape[2]
    model = _model(g, N, K, hid, prec, cuda_device)
    gs = torch.from_numpy(g["G_static"]).to(cuda_device).requires_grad_(True)
    G_list = [gs, (torch.from_numpy(g["G_o"]).to(cuda_device), torch.from_numpy(g["G_d"]).to(cuda_device))]
    y = model(x_seq=torch.from_numpy(g["x_seq"]).to(cuda_device), G_list=G_list)
    y.backward(torch.from_numpy(g["d_y"]).to(cuda_device))
    torch.cuda.synchronize()
    if prec == "fp32":
        _check(y, g["y"], 5e-5, f"{name}/{prec}/y")
        _check(gs.grad, g["dG_static"], 2e-4, f"{name}/{prec}/dG_static")       # summation-order noise only
        for k, p in model.named_parameters():
            _check(p.grad, g["grad:" + k], 2e-4, f"{name}/{prec}/grad:{k}")
    else:
        _check(y, g["y"], 1e-3, f"{name}/{prec}/y")
        _check(gs.grad, g["dG_static"], LOOSE_FP16_GRAD, f"{name}/{prec}/dG_static vs reference", l2_only=True)


@pytest.mark.gpu
def test_support_grad_is_refused_by_default(cuda_device):
    X = torch.zeros(2, 9, 9, 32, device=cuda_device)
    G = torch.rand(3, 9, 9, device=cuda_device).requires_grad_(True)
    layer = shim.BDGCN(K=3, input_dim=32, hidden_dim=32, use_bias=True, activation=nn.ReLU).to(cuda_device)
    with pytest.raises(NotImplementedError):
        layer(X, G)
    with pytest.raises(NotImplementedError):
        ops.bdgcn(X, (G.expand(2, 3, 9, 9), G.expand(2, 3, 9, 9)), layer.W, layer.b, relu=True)
    with torch.no_grad():                  # no gradient asked for: nothing to refuse
        layer(X, G)
    layer.support_grad = True
    layer(X, G).sum().backward()
    assert G.grad is not None and G.grad.shape == G.shape


@pytest.mark.gpu
def test_prepared_supports_restaged_after_an_optimiser_step(cuda_device):
    """fp16 layers stage each support tensor once (a cache keyed on the tensor and its version): an in-place optimiser step on
    a learnable G must re-stage it, so the next forward equals one on a fresh copy of the updated G."""
    X, G, W, b, d_out, t = _inputs(3, 2, 40, 3, 32, 32, False, cuda_device)
    layer = shim.BDGCN(K=3, input_dim=32, hidden_dim=32, use_bias=True, activation=nn.ReLU).to(cuda_device)
    layer.precision, layer.support_grad = "fp16", True
    Gp = nn.Parameter(t(G))
    opt = torch.optim.SGD([Gp], lr=0.5)
    Xt = t(X)
    layer(Xt, Gp).backward(t(d_out))
    opt.step()
    after = layer(Xt, Gp)
    fresh = layer(Xt, Gp.detach().clone())
    assert not torch.equal(Gp.detach(), t(G))
    assert torch.equal(after, fresh)


def _load_reference_mpgcn():
    if not os.path.isfile(os.path.join(REF_DIR, "MPGCN.py")):
        pytest.skip("oracle/_ref (the unmodified reference) is not installed")
    spec = importlib.util.spec_from_file_location("_ref_MPGCN_sgrad", os.path.join(REF_DIR, "MPGCN.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.gpu
def test_adam_on_a_learnable_support_tracks_the_reference(cuda_device):
    """A few Adam steps on the model with a learnable static support (an nn.Parameter G, every model parameter trained too),
    ours in fp32 against the reference model in float32 on the GPU from the same initial state."""
    ref_mpgcn = _load_reference_mpgcn()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    B, T, N, K, hid = 2, 4, 12, 3, 32
    rng = np.random.default_rng(2024)
    torch.manual_seed(2024)
    ref = ref_mpgcn.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                          num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    with torch.no_grad():                  # live heads: a dead FC ReLU would leave the support without a gradient
        for branch in ref.branch_models:
            branch['fc'][0].bias.fill_(0.5)
    ours = _model(None, N, K, hid, "fp32", cuda_device)
    ours.load_state_dict(ref.state_dict())
    x = torch.from_numpy((rng.random((B, T, N, N, 1)) * 4).astype(np.float32)).to(cuda_device)
    target = torch.from_numpy(rng.random((B, 1, N, N, 1)).astype(np.float32)).to(cuda_device)
    g0 = torch.from_numpy((rng.random((K, N, N)) / N).astype(np.float32)).to(cuda_device)
    gd = (torch.from_numpy((rng.random((B, K, N, N)) / N).astype(np.float32)).to(cuda_device),) * 2
    runs = {}
    for tag, model in (("ref", ref), ("ours", ours)):
        G = nn.Parameter(g0.clone())
        opt = torch.optim.Adam(list(model.parameters()) + [G], lr=1e-3)
        losses = []
        for _ in range(4):
            opt.zero_grad()
            loss = torch.mean((model(x, [G * 1.0, gd]) - target) ** 2)     # the reference takes a plain Tensor, not a Parameter
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        runs[tag] = (losses, G.detach().cpu().numpy())
    np.testing.assert_allclose(runs["ours"][0], runs["ref"][0], rtol=1e-4)
    moved = runs["ref"][1] - g0.cpu().numpy()
    assert np.abs(moved).max() > 1e-4
    _check(runs["ours"][1] - g0.cpu().numpy(), moved, 1e-3, "adam: G update", l2_only=True)


def capture_layer_grads(model, m):
    """Forward hooks on branch m's BDGCN layers -> [(layer, {"X", "out", "d_out"})] filled by the next forward / backward: each
    layer's input and output, and by a tensor hook on the output its upstream gradient."""
    caps = []

    def hook(layer, inp, out):
        rec = {"X": inp[0].detach(), "out": out.detach()}
        out.register_hook(lambda g: rec.__setitem__("d_out", g.detach().clone()))
        caps.append((layer, rec))
    handles = [layer.register_forward_hook(hook) for layer in model.branch_models[m]['spatial']]
    return caps, handles


def model_support_grad_float64(caps, G, dev):
    """sum over the captured layers of support_grads on each layer's own ReLU mask: the float64 dL/dG of the function the engine
    computed (static: [K,N,N]; dynamic: (dG_o, dG_d))."""
    total = None
    G = tuple(g.detach() for g in G) if isinstance(G, tuple) else G.detach()
    for layer, rec in caps:
        r = support_grads(rec["X"], G, layer.W.detach(), layer.b.detach(), "relu", rec["d_out"], mask_from=rec["out"], device=dev)
        total = r if total is None else (tuple(a + b for a, b in zip(total, r)) if isinstance(r, tuple) else total + r)
    return total


def _live_model(N, K, hid, prec, dev, seed=5):
    """The trainer's model (M = 2, three layers) with support gradients on and live heads (a dead FC ReLU would leave the supports
    without a gradient); prec None keeps every layer at the default precision."""
    torch.manual_seed(seed)
    model = _model(None, N, K, hid, prec, dev)
    with torch.no_grad():
        for branch in model.branch_models:
            branch['fc'][0].bias.fill_(0.5)
    return model


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "fp16"])
@pytest.mark.parametrize("dyn", [False, True])
def test_model_support_grad_against_float64_on_the_engine_masks(dyn, prec, cuda_device):
    """A learnable static G (an nn.Parameter in branch 0), or a learnable dynamic pair (branch 1): G.grad, which the three layers'
    gradients add into, against the float64 sum over the layers of support_grads on each layer's captured input, output (its ReLU
    mask) and upstream gradient, on rel_L2 and rel_Linf at TOL (on an H100 the largest error was 3.4e-4 in fp16, 7.0e-7 in fp32)."""
    B, T, N, K, hid = 2, 4, 20, 3, 32
    rng = np.random.default_rng(31 + int(dyn))
    t = lambda a: torch.from_numpy(a.astype(np.float32)).to(cuda_device)
    model = _live_model(N, K, hid, prec, cuda_device)
    G = nn.Parameter(t(rng.random((K, N, N)) / N))
    pair = tuple(nn.Parameter(t(rng.random((B, K, N, N)) / N)) for _ in range(2))
    G_list = [G, pair] if not dyn else [G.detach(), pair]
    caps, handles = capture_layer_grads(model, 1 if dyn else 0)
    model(x_seq=t(rng.random((B, T, N, N, 1)) * 4), G_list=G_list).backward(t(rng.standard_normal((B, 1, N, N, 1))))
    torch.cuda.synchronize()
    for h in handles:
        h.remove()
    assert len(caps) == 3
    ref = model_support_grad_float64(caps, pair if dyn else G, cuda_device)
    what = f"model {'dynamic pair' if dyn else 'static G'}/{prec}: dG vs float64 on the engine masks"
    if dyn:
        _check(pair[0].grad, ref[0], TOL[prec], what + "/dG_o")
        _check(pair[1].grad, ref[1], TOL[prec], what + "/dG_d")
    else:
        _check(G.grad, ref, TOL[prec], what)
