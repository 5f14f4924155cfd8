"""Gradients through the support-matrix builder: `GCN.Adj_Processor.process(flow)` differentiable with respect to `flow`.

CPU: the float64 adjoint (tests/adj_grad_oracle.py) against the reference's autograd fixtures `agrad_*` and against central
finite differences of the forward, the C-ABI surface and the entry point's argument checks.  GPU: the engine's d_flow against
float64 for every kernel type across sizes, the fixtures, the zero-row rule, the unchanged forward, when a gradient is (not)
tracked, CPU leaves, a flow feeding both sides of a dynamic pair, Adam steps on a learnable adjacency against the reference
model fed by the reference's Adj_Processor, the whole chain flow -> supports -> model at the default (fp16) precision, and Adam on a
learnable adjacency in fp16 against fp32.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch
from torch import nn

from adj_grad_oracle import adj_process_grad
from conftest import ROOT, golden_names, load_golden, record_parity
from oracle import mpgcn_oracle as orc

import MPGCN as shim
from mpgcn_b200 import _lib
from mpgcn_b200.GCN import Adj_Processor

KINDS = ("localpool", "chebyshev", "random_walk_diffusion", "dual_random_walk_diffusion")
KT = {k: i for i, k in enumerate(KINDS)}
TOL = 2e-5          # the forward's bar (test_gpu_parity.py); see test_dflow_against_float64 for the gradient's margin
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def _check(a, ref, tol, what, l2_only=False):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol), f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"


def _check_grad(got, ref, flow, d_sup, tol, what):
    """_check, except where the exact gradient is 0 and both sides are rounding noise (N = 1: every support is constant in the
    flow).  There d_flow is the difference of two equal terms of size |gx| / rowsum, with |gx| <= (K+1)^3 max|d_supports| (the
    Chebyshev adjoint at x = +-1), and it must stay within tol of that size."""
    scale = float(np.abs(d_sup).max())
    if np.abs(ref).max() <= 1e-6 * scale:
        got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got
        terms = scale * d_sup.shape[1] ** 3 / float(np.abs(np.asarray(flow).sum(axis=2)).min())
        assert np.abs(got).max() <= tol * terms, f"{what}: max|d_flow| = {np.abs(got).max():.3e} where the gradient is 0"
        return
    _check(got, ref, tol, what)


def _num_supports(kind, K):
    return 1 if kind == "localpool" else (2 * K + 1 if kind == "dual_random_walk_diffusion" else K + 1)


def _flow(rng, B, N):
    return (rng.random((B, N, N)) + 0.05).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------------------
def test_fixture_prefix_is_its_own():
    names = golden_names("agrad_")
    assert len(names) >= 16
    for kind in ("lp", "cheb", "rw", "drw"):
        assert any(n.startswith(f"agrad_{kind}_") for n in names)
    assert {"agrad_rw_k2_b2_n12_zero", "agrad_drw_k2_b2_n12_zero"} <= set(names)
    for prefix in ("adj_", "sgrad_", "bdgcn_", "mpgcn_"):
        assert not set(names) & set(golden_names(prefix))
    for n in names:
        assert os.path.getsize(os.path.join(ROOT, "tests", "golden", n + ".npz")) < 1 << 20


def _zero_sums(flow):
    """(b, i) of rows and (b, j) of columns whose sum's inverse is inf: where the random-walk normalisation masks."""
    with np.errstate(divide="ignore"):
        return np.isinf(1.0 / flow.sum(axis=2)), np.isinf(1.0 / flow.sum(axis=1))


@pytest.mark.parametrize("name", golden_names("agrad_"))
def test_oracle_matches_reference_fixture(name):
    g = load_golden(name)
    kind, K = str(g["kernel_type"]), int(g["K"])
    _check(orc.adj_process(g["flow"], kind, K), g["supports"], 1e-12, f"{name}/oracle supports")
    got = adj_process_grad(g["flow"], g["d_supports"], kind, K)
    ref = g["d_flow"]
    nan = np.isnan(ref)
    assert np.isfinite(got).all()
    _check_grad(np.where(nan, 0, got), np.where(nan, 0, ref), g["flow"], g["d_supports"], 1e-10, f"{name}/oracle d_flow (finite entries)")
    if not nan.any():
        return
    # NaN only where the reference's random-walk normalisation divided by a zero sum; there, that series contributes exactly 0
    zrow, zcol = _zero_sums(g["flow"])
    assert not (nan & ~(zrow[:, :, None] | zcol[:, None, :])).any()
    fwd = adj_process_grad(g["flow"], g["d_supports"], kind, K, series="forward")
    assert (fwd[zrow] == 0).all() and zrow.any()
    if kind == "random_walk_diffusion":
        assert (got[nan] == 0).all()
    else:
        bwd = adj_process_grad(g["flow"], g["d_supports"], kind, K, series="backward")
        assert (bwd.transpose(0, 2, 1)[zcol] == 0).all() and zcol.any()
        np.testing.assert_array_equal(fwd + bwd, got)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [1, 2, 3])
def test_oracle_matches_finite_differences(kind, K):
    if kind == "localpool" and K != 1:
        pytest.skip("localpool has one support whatever K is")
    rng = np.random.default_rng(31 * K + KT[kind])
    B, N, eps = 2, 6, 1e-6
    flow = rng.random((B, N, N)) + 0.2
    d_sup = rng.standard_normal((B, _num_supports(kind, K), N, N))
    loss = lambda f: float((orc.adj_process(f, kind, K) * d_sup).sum())
    fd = np.zeros_like(flow)
    for idx in np.ndindex(*flow.shape):
        fp, fm = flow.copy(), flow.copy()
        fp[idx] += eps
        fm[idx] -= eps
        fd[idx] = (loss(fp) - loss(fm)) / (2 * eps)
    _check(adj_process_grad(flow, d_sup, kind, K), fd, 1e-7, f"oracle vs finite differences {kind} K={K}")


def test_new_symbols_are_exported_and_bound():
    for sym in ("mpgcn_adj_backward_workspace_bytes", "mpgcn_adj_process_backward"):
        assert sym in _lib.EXPORTED_SYMBOLS
        with open(os.path.join(ROOT, "include", "mpgcn_b200.h")) as f:
            assert sym + "(" in f.read()
    lib = _lib.load()
    assert lib.mpgcn_abi_version() == 4
    for kt in range(4):
        for K in (0, 1, 3):
            assert lib.mpgcn_adj_backward_workspace_bytes(2, 33, kt, K) >= lib.mpgcn_adj_workspace_bytes(2, 33, kt, K) > 0
    # the recursion's working copy of d_supports: [B][Ks][N][N] floats from K = 2 on
    assert lib.mpgcn_adj_backward_workspace_bytes(2, 33, 3, 3) >= 2 * 7 * 33 * 33 * 4
    assert lib.mpgcn_adj_backward_workspace_bytes(2, 33, 4, 1) == 0
    assert lib.mpgcn_adj_backward_workspace_bytes(0, 33, 1, 1) == 0


def test_entry_point_rejects_bad_arguments_without_a_gpu():
    """Every case fails validation, which runs before any CUDA call: fake device addresses are never touched."""
    lib = _lib.load()
    B, N, kt, K = 2, 9, 3, 3
    p = 1 << 20                                   # a plausible, never dereferenced address

    def call(B=B, N=N, kt=kt, K=K, ws_bytes=None, **kw):
        a = dict(flow=p, sup=p, dsup=p, dflow=p, ws=p)
        a.update(kw)
        if ws_bytes is None:
            ws_bytes = 1 << 40
        r = lib.mpgcn_adj_process_backward(a["flow"], a["sup"], a["dsup"], a["dflow"], B, N, kt, K, a["ws"], ws_bytes, None)
        return r, lib.mpgcn_last_error().decode()

    for ptr in ("flow", "sup", "dsup", "dflow", "ws"):
        r, msg = call(**{ptr: None})
        assert r != 0 and "null pointer" in msg, ptr
    for bad_kt in (-1, 4):
        r, msg = call(kt=bad_kt)
        assert r != 0 and "Invalid kernel_type" in msg
    for shape in (dict(B=0), dict(N=0), dict(N=-3), dict(K=-1)):
        r, msg = call(**shape)
        assert r != 0 and "bad shape" in msg, shape
    for kt_ in range(4):
        need = lib.mpgcn_adj_backward_workspace_bytes(B, N, kt_, K)
        r, msg = call(kt=kt_, ws_bytes=need - 1)
        assert r != 0 and "workspace too small" in msg


# ------------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------------
def _engine_grad(kind, K, flow, d_sup, dev):
    """-> (supports, d_flow) from the engine, flow / d_sup float32 numpy."""
    f = torch.from_numpy(flow).to(dev).requires_grad_(True)
    S = Adj_Processor(kind, K, device=dev).process(f)
    S.backward(torch.from_numpy(d_sup.astype(np.float32)).to(dev))
    torch.cuda.synchronize()
    return S.detach(), f.grad


GRAD_CASES = [(kind, N, K, B) for kind in KINDS for N in (1, 2, 7, 33, 129, 500) for K in (1, 2, 4) for B in (1, 3)
              if not (kind == "localpool" and K != 1)]
GRAD_CASES += [("random_walk_diffusion", 1000, 3, 2), ("dual_random_walk_diffusion", 1000, 3, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,N,K,B", GRAD_CASES)
def test_dflow_against_float64(kind, N, K, B, cuda_device):
    """d_flow against the float64 adjoint of the same float32 flow, at the forward's 2e-5 bar on both rel_L2 and rel_Linf.
    The adjoint is exact fp32 SGEMMs plus length-N reductions, like the forward, so the forward's bar applies unchanged: on an
    H100 the largest errors measured were rel_Linf 9.6e-7 and rel_L2 8.8e-7 (random walk N = 500 K = 4, chebyshev
    N = 2 K = 4), a margin of 20x."""
    rng = np.random.default_rng(1000 * N + 10 * K + B + KT[kind])
    flow = _flow(rng, B, N)
    d_sup = rng.standard_normal((B, _num_supports(kind, K), N, N)).astype(np.float32)
    _, got = _engine_grad(kind, K, flow, d_sup, cuda_device)
    _check_grad(got, adj_process_grad(flow, d_sup, kind, K), flow, d_sup, TOL, f"adj grad {kind} N={N} K={K} B={B}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("agrad_"))
def test_reference_fixture(name, cuda_device):
    g = load_golden(name)
    kind, K = str(g["kernel_type"]), int(g["K"])
    S, got = _engine_grad(kind, K, g["flow"].astype(np.float32), g["d_supports"], cuda_device)
    _check(S, g["supports"], TOL, f"{name}/supports")
    got = got.cpu().numpy()
    ref = g["d_flow"]
    nan = np.isnan(ref)
    assert np.isfinite(got).all()
    _check_grad(np.where(nan, 0, got), np.where(nan, 0, ref), g["flow"], g["d_supports"], TOL, f"{name}/d_flow (finite entries)")
    if kind == "random_walk_diffusion":
        assert (got[nan] == 0).all()
    _check_grad(got, adj_process_grad(g["flow"], g["d_supports"].astype(np.float32), kind, K), g["flow"], g["d_supports"], TOL,
                f"{name}/d_flow vs oracle")


@pytest.mark.gpu
def test_masked_rows_and_columns_contribute_exact_zeros(cuda_device):
    """Random walk: an empty row, and a row whose sum is an fp32 subnormal (1/sum overflows, so the forward masks it too), get
    exactly 0.  Dual: an empty row gets exactly 0 from the forward series and an empty column from the backward series (the other
    series' upstream gradient is zeroed to isolate each); with both series live the result is finite and matches the oracle."""
    rng = np.random.default_rng(7)
    B, N, K = 2, 40, 3
    flow = _flow(rng, B, N)
    flow[0, 5, :] = 0
    flow[1, 17, :] = 0
    flow[1, 17, 3] = 1e-39                          # subnormal in fp32: 1 / 1e-39 = inf
    d_sup = rng.standard_normal((B, K + 1, N, N)).astype(np.float32)
    S, got = _engine_grad("random_walk_diffusion", K, flow, d_sup, cuda_device)
    got = got.cpu().numpy()
    assert np.isfinite(S.cpu().numpy()).all() and np.isfinite(got).all()
    assert (got[0, 5] == 0).all() and (got[1, 17] == 0).all()
    ref_flow = flow.copy()
    ref_flow[1, 17, 3] = 0                          # the function the fp32 forward computed
    _check(got, adj_process_grad(ref_flow, d_sup, "random_walk_diffusion", K), TOL, "zero rows/random walk")

    flow = _flow(rng, B, N)
    flow[0, 9, :] = 0
    flow[1, :, 22] = 0
    d_sup = rng.standard_normal((B, 2 * K + 1, N, N)).astype(np.float32)
    fwd_only, bwd_only = d_sup.copy(), d_sup.copy()
    fwd_only[:, K + 1:] = 0
    bwd_only[:, 1:K + 1] = 0
    _, g_f = _engine_grad("dual_random_walk_diffusion", K, flow, fwd_only, cuda_device)
    _, g_b = _engine_grad("dual_random_walk_diffusion", K, flow, bwd_only, cuda_device)
    assert (g_f[0, 9] == 0).all() and (g_b[1, :, 22] == 0).all()
    _, both = _engine_grad("dual_random_walk_diffusion", K, flow, d_sup, cuda_device)
    assert torch.isfinite(both).all()
    _check(both, adj_process_grad(flow, d_sup, "dual_random_walk_diffusion", K), TOL, "zero rows/dual")


@pytest.mark.gpu
def test_symmetric_kernels_give_nan_on_a_zero_row(cuda_device):
    """A zero-sum row makes the symmetric normalisation's forward non-finite; the gradient then holds NaN (as the reference's)."""
    rng = np.random.default_rng(8)
    flow = _flow(rng, 1, 12)
    flow[0, 4, :] = 0
    for kind, K in (("localpool", 1), ("chebyshev", 1), ("chebyshev", 3)):
        d_sup = rng.standard_normal((1, _num_supports(kind, K), 12, 12)).astype(np.float32)
        _, got = _engine_grad(kind, K, flow, d_sup, cuda_device)
        assert torch.isnan(got).any(), (kind, K)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_supports_unchanged_by_gradient_tracking(kind, cuda_device):
    """Bitwise the same supports whether the flow requires grad or not, and under no_grad (no grad_fn there)."""
    rng = np.random.default_rng(KT[kind])
    flow = torch.from_numpy(_flow(rng, 3, 57)).to(cuda_device)
    proc = Adj_Processor(kind, 3)
    plain = proc.process(flow)
    assert plain.grad_fn is None
    tracked = proc.process(flow.clone().requires_grad_(True))
    assert tracked.grad_fn is not None and torch.equal(plain, tracked)
    with torch.no_grad():
        nog = proc.process(flow.clone().requires_grad_(True))
    assert nog.grad_fn is None and not nog.requires_grad and torch.equal(plain, nog)
    f64 = flow.double().requires_grad_(True)
    assert torch.equal(proc.process(f64).detach(), plain)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["chebyshev", "random_walk_diffusion", "dual_random_walk_diffusion"])
def test_identity_alone_carries_no_gradient(kind, cuda_device):
    """K = 0: only T_0 = I, which does not depend on the flow -- no grad_fn, as in the reference."""
    flow = torch.rand(2, 9, 9, device=cuda_device, requires_grad=True)
    S = Adj_Processor(kind, 0).process(flow)
    assert S.grad_fn is None and not S.requires_grad
    assert torch.equal(S, torch.eye(9, device=cuda_device).expand(2, 1, 9, 9))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_cpu_leaf_gets_a_cpu_grad(dtype, cuda_device):
    rng = np.random.default_rng(3)
    flow = _flow(rng, 2, 20)
    d_sup = rng.standard_normal((2, 7, 20, 20)).astype(np.float32)
    leaf = torch.from_numpy(flow).to(dtype).requires_grad_(True)
    proc = Adj_Processor("dual_random_walk_diffusion", 3, device=cuda_device)
    S = proc.process(leaf)
    assert S.is_cuda
    S.backward(torch.from_numpy(d_sup).to(cuda_device))
    assert leaf.grad.device.type == "cpu" and leaf.grad.dtype == dtype
    _, on_gpu = _engine_grad("dual_random_walk_diffusion", 3, flow, d_sup, cuda_device)
    assert torch.equal(leaf.grad.float(), on_gpu.cpu())


@pytest.mark.gpu
def test_one_flow_on_both_sides_of_a_dynamic_pair_gets_the_sum(cuda_device):
    B, N, K, C = 2, 15, 3, 32
    rng = np.random.default_rng(4)
    flow = torch.from_numpy(_flow(rng, B, N)).to(cuda_device)
    X = torch.from_numpy(np.tanh(rng.standard_normal((B, N, N, C))).astype(np.float32)).to(cuda_device)
    layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=C, use_bias=True, activation=nn.ReLU).to(cuda_device)
    layer.precision, layer.support_grad = "fp32", True
    proc = Adj_Processor("random_walk_diffusion", K - 1)
    d_out = torch.from_numpy(rng.standard_normal((B, N, N, C)).astype(np.float32)).to(cuda_device)
    one = flow.clone().requires_grad_(True)
    G = proc.process(one)
    layer(X, (G, G)).backward(d_out)
    two = flow.clone().requires_grad_(True), flow.clone().requires_grad_(True)
    layer(X, (proc.process(two[0]), proc.process(two[1]))).backward(d_out)
    torch.cuda.synchronize()
    assert float(two[0].grad.abs().max()) > 0 and float(two[1].grad.abs().max()) > 0
    torch.testing.assert_close(one.grad, two[0].grad + two[1].grad, rtol=1e-5, atol=1e-6 * float(one.grad.abs().max()))


def _load_reference(name):
    if not os.path.isfile(os.path.join(REF_DIR, f"{name}.py")):
        pytest.skip("oracle/_ref (the unmodified reference) is not installed")
    spec = importlib.util.spec_from_file_location(f"_ref_{name}_agrad", os.path.join(REF_DIR, f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _adam_runs(learn_static, cuda_device):
    """A few Adam steps on the whole model plus a learnable flow, ours in fp32 against the reference model fed by the reference's
    Adj_Processor (float32 on the CPU, then .to(device)), from the same initial state."""
    ref_mpgcn, ref_gcn = _load_reference("MPGCN"), _load_reference("GCN")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    B, T, N, K, hid = 2, 4, 12, 3, 32
    rng = np.random.default_rng(2025 + int(learn_static))
    torch.manual_seed(2025)
    ref = ref_mpgcn.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                          num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    with torch.no_grad():                  # live heads: a dead FC ReLU would leave the supports without a gradient
        for branch in ref.branch_models:
            branch['fc'][0].bias.fill_(0.5)
    ours = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                      num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    ours.load_state_dict(ref.state_dict())
    ours.lstm_precision = "fp32"
    for mod in ours.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision, mod.support_grad = "fp32", True
    x = torch.from_numpy((rng.random((B, T, N, N, 1)) * 4).astype(np.float32)).to(cuda_device)
    target = torch.from_numpy(rng.random((B, 1, N, N, 1)).astype(np.float32)).to(cuda_device)
    adj0 = torch.from_numpy(_flow(rng, 1, N))
    od0 = torch.from_numpy(_flow(rng, B, N)), torch.from_numpy(_flow(rng, B, N))
    runs = {}
    for tag, model, procs in (("ref", ref, (ref_gcn.Adj_Processor("random_walk_diffusion", K - 1),
                                            ref_gcn.Adj_Processor("dual_random_walk_diffusion", 1))),
                              ("ours", ours, (Adj_Processor("random_walk_diffusion", K - 1), Adj_Processor("dual_random_walk_diffusion", 1)))):
        on_dev = tag == "ours"
        adj = nn.Parameter(adj0.clone().to(cuda_device) if on_dev else adj0.clone())
        od = tuple(nn.Parameter(t.clone().to(cuda_device) if on_dev else t.clone()) for t in od0)
        learnable = [adj] if learn_static else list(od)
        opt = torch.optim.Adam(list(model.parameters()) + learnable, lr=1e-3)
        losses = []
        for _ in range(4):
            opt.zero_grad()
            G = procs[0].process(adj if learn_static else adj.detach()).to(cuda_device)[0]
            pair = tuple(procs[1].process(t if not learn_static else t.detach()).to(cuda_device) for t in od)
            loss = torch.mean((model(x, [G, pair]) - target) ** 2)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        runs[tag] = (losses, [p.detach().cpu().numpy() for p in learnable])
    start = [adj0.numpy()] if learn_static else [t.numpy() for t in od0]
    np.testing.assert_allclose(runs["ours"][0], runs["ref"][0], rtol=1e-4)
    for i, s in enumerate(start):
        moved = runs["ref"][1][i] - s
        assert np.abs(moved).max() > 1e-4
        _check(runs["ours"][1][i] - s, moved, 1e-3, f"adam: flow {i} update ({'static' if learn_static else 'dynamic'})",
               l2_only=True)


@pytest.mark.gpu
def test_adam_on_a_learnable_static_adjacency_tracks_the_reference(cuda_device):
    _adam_runs(True, cuda_device)


@pytest.mark.gpu
def test_adam_on_a_learnable_dynamic_pair_tracks_the_reference(cuda_device):
    _adam_runs(False, cuda_device)


def _chain(model, procs, flows, x, d_y, dev):
    """flow -> Adj_Processor -> model, one forward / backward: procs / flows for the static adjacency [1,N,N] (branch 0) and the OD
    pair [B,N,N] x 2 (branch 1).  -> (captured layers of both branches, the supports, their gradients captured by tensor hooks)."""
    from test_support_grad import capture_layer_grads
    sups, grads = [], {}
    for i, f in enumerate(flows):
        S = procs[0 if i == 0 else 1].process(f)
        S.register_hook(lambda g, i=i: grads.__setitem__(i, g.detach().clone()))
        sups.append(S)
    caps = [capture_layer_grads(model, m) for m in range(2)]
    model(x_seq=x, G_list=[sups[0][0], (sups[1], sups[2])]).backward(d_y)
    torch.cuda.synchronize()
    for _, handles in caps:
        for h in handles:
            h.remove()
    return [c for c, _ in caps], sups, [grads[i] for i in range(len(flows))]


@pytest.mark.gpu
def test_learnable_adjacency_chain_at_the_default_precision(cuda_device):
    """flow -> Adj_Processor (random walk: static adjacency; dual random walk: OD pair) -> model with every layer at the default
    precision, which resolves to the fp16 tensor cores at hidden 32: each flow's gradient is the builder's adjoint of its supports'
    own gradient (captured by a tensor hook) at TOL, and that support gradient passes the float64 model check at fp16's 2e-3
    (on an H100 the largest errors were 3.8e-6 and 4.5e-4)."""
    from test_support_grad import TOL as SG_TOL, _live_model, model_support_grad_float64
    from mpgcn_b200 import ops
    B, T, N, K, hid = 2, 4, 20, 3, 32
    rng = np.random.default_rng(77)
    model = _live_model(N, K, hid, None, cuda_device)
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            assert mod.precision is None and ops.resolve_precision(mod.precision, B, N, K, hid, hid) == _lib.PREC_FP16_TC
    t = lambda a: torch.from_numpy(a).to(cuda_device)
    flows = [t(_flow(rng, 1, N)).requires_grad_(True)] + [t(_flow(rng, B, N)).requires_grad_(True) for _ in range(2)]
    procs = (Adj_Processor("random_walk_diffusion", K - 1), Adj_Processor("dual_random_walk_diffusion", 1))
    x = t((rng.random((B, T, N, N, 1)) * 4).astype(np.float32))
    d_y = t(rng.standard_normal((B, 1, N, N, 1)).astype(np.float32))
    caps, sups, d_sups = _chain(model, procs, flows, x, d_y, cuda_device)
    for i, (f, d) in enumerate(zip(flows, d_sups)):
        kind, order = ("random_walk_diffusion", K - 1) if i == 0 else ("dual_random_walk_diffusion", 1)
        assert float(d.abs().max()) > 0
        _check(f.grad, adj_process_grad(f.detach().cpu().numpy(), d.cpu().numpy(), kind, order), TOL, f"chain/auto: flow {i} grad")
    ref_s = model_support_grad_float64(caps[0], sups[0][0], cuda_device)
    _check(d_sups[0][0], ref_s, SG_TOL["fp16"], "chain/auto: static support grad vs float64 on the engine masks")
    ref_o, ref_d = model_support_grad_float64(caps[1], (sups[1], sups[2]), cuda_device)
    _check(d_sups[1], ref_o, SG_TOL["fp16"], "chain/auto: G_o support grad vs float64 on the engine masks")
    _check(d_sups[2], ref_d, SG_TOL["fp16"], "chain/auto: G_d support grad vs float64 on the engine masks")


# Adam divides each element's update by its own gradient's running magnitude, so flow elements whose gradient is near zero move
# by a near-random sign in either precision: on an H100 (80GB HBM3, 700 W) the fp16 update differs from the fp32 one by rel_L2
# 0.23; the bar is 4x that, so it mostly catches an update that stays at zero (rel_L2 1).  The elements whose gradient kept its
# sign (the fp32 run moved them at least half its largest move) have a determined update: there the difference measured 0.092,
# and the bar of 4x that rejects an update off by a factor of 2 or of the wrong sign.
ADAM_FLOW_UPDATE_TOL = 0.95
ADAM_STEADY_UPDATE_TOL = 0.4


@pytest.mark.gpu
def test_adam_on_a_learnable_adjacency_is_equivalent_in_fp16_and_fp32(cuda_device):
    """20 Adam steps on the model plus a learnable static adjacency (random walk), every layer and the LSTM on the fp16 tensor
    cores against the fp32 kernels, from one initial state: the loss curves within test_gpu_at_size's 2e-2 (max relative
    difference; measured 2.1e-3), and the flow's update in rel_L2 within ADAM_FLOW_UPDATE_TOL over every element (measured 0.23)
    and within ADAM_STEADY_UPDATE_TOL over the elements the fp32 run moved steadily (measured 0.092)."""
    B, T, N, K, hid = 2, 4, 12, 3, 32
    rng = np.random.default_rng(2026)
    x = torch.from_numpy((rng.random((B, T, N, N, 1)) * 4).astype(np.float32)).to(cuda_device)
    target = torch.from_numpy(rng.random((B, 1, N, N, 1)).astype(np.float32)).to(cuda_device)
    adj0 = torch.from_numpy(_flow(rng, 1, N)).to(cuda_device)
    od = tuple(torch.from_numpy(_flow(rng, B, N)).to(cuda_device) for _ in range(2))
    from test_support_grad import _live_model
    runs = {}
    for prec in ("fp32", "fp16"):
        model = _live_model(N, K, hid, prec, cuda_device, seed=2026)
        adj = nn.Parameter(adj0.clone())
        opt = torch.optim.Adam(list(model.parameters()) + [adj], lr=1e-3)
        pair = tuple(Adj_Processor("dual_random_walk_diffusion", 1).process(t) for t in od)
        proc = Adj_Processor("random_walk_diffusion", K - 1)
        losses = []
        for _ in range(20):
            opt.zero_grad()
            loss = torch.mean((model(x, [proc.process(adj)[0], pair]) - target) ** 2)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        runs[prec] = (np.asarray(losses), (adj.detach() - adj0).cpu().numpy())
    a, r = runs["fp16"][0], runs["fp32"][0]
    assert np.all(np.isfinite(a)) and r[-1] < r[0], f"fp32 loss did not move: {r[0]:.4f} -> {r[-1]:.4f}"
    rel = np.abs(a - r) / r
    record_parity("adam-20 learnable adjacency: loss curve fp16 vs fp32 (max rel diff)", float(rel.max()),
                  float(np.linalg.norm(a - r) / np.linalg.norm(r)), 2e-2)
    assert rel.max() <= 2e-2, f"loss curves diverge: max rel diff {rel.max():.3e} at step {int(rel.argmax())}"
    moved = runs["fp32"][1]
    assert np.abs(moved).max() > 1e-4
    _check(runs["fp16"][1], moved, ADAM_FLOW_UPDATE_TOL, "adam-20 learnable adjacency: flow update fp16 vs fp32", l2_only=True)
    steady = np.abs(moved) >= 0.5 * np.abs(moved).max()          # elements whose gradient kept its sign over the steps
    assert steady.sum() >= 10
    _check(runs["fp16"][1][steady], moved[steady], ADAM_STEADY_UPDATE_TOL,
           "adam-20 learnable adjacency: flow update fp16 vs fp32 where fp32 moved >= half its largest move", l2_only=True)
