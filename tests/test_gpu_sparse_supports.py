"""Sparse static supports on the GPU (DESIGN.md section 12): the CSR / CSC build, the four gather stages of the fp32 layer against
float64, the layer at size against the dense fp32 layer, the reference fixtures with G.to_sparse(), and the model-level behaviour
(no stash without grad, CUDA-graph paths, deterministic mode, refusals, cache invalidation, the trainer)."""
import math
import os
import zlib

import numpy as np
import pytest
import torch
from torch import nn

from conftest import golden_names, load_golden, record_parity
from oracle import mpgcn_oracle as orc
from oracle.gen_golden import layer_fixture
from test_oracle_golden import load_big

import MPGCN as shim
from mpgcn_b200 import _lib, ops, rollout, shard
from mpgcn_b200.graph_step import GraphedTrainStep

pytestmark = pytest.mark.gpu

FWD_TOL, BWD_TOL = 5e-5, 2e-4        # the fp32 bars (test_gpu_channel_widths.py)


def _check(a, ref, tol, what):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(f"sparse {what}", linf, l2, tol)
    assert np.isfinite(linf) and linf <= tol and l2 <= tol, f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"


def _knn_adjacency(rng, N, k):
    """symmetric k-nearest-neighbour graph of random points in the plane, with self loops"""
    p = rng.random((N, 2))
    d = ((p[:, None] - p[None]) ** 2).sum(-1)
    A = np.zeros((N, N))
    nb = np.argsort(d, axis=1)[:, 1:k + 1] if N > 1 else np.zeros((N, 0), int)
    A[np.repeat(np.arange(N), nb.shape[1]), nb.ravel()] = 1.0
    A = np.maximum(A, A.T)
    np.fill_diagonal(A, 1.0)
    return A


def _random_sparse(rng, K, N, density):
    G = rng.standard_normal((K, N, N)) * (rng.random((K, N, N)) < density)
    return (G / math.sqrt(max(1.0, density * N))).astype(np.float32)


def _supports(kind, rng, K, N):
    if kind in ("localpool", "chebyshev", "random_walk_diffusion", "dual_random_walk_diffusion"):
        order = {"localpool": 1, "chebyshev": K - 1, "random_walk_diffusion": K - 1, "dual_random_walk_diffusion": (K - 1) // 2}[kind]
        return orc.adj_process(_knn_adjacency(rng, N, 4)[None], kind, order)[0].astype(np.float32)
    if kind == "identity":
        return np.eye(N, dtype=np.float32)[None].repeat(K, 0)
    if kind == "dense":
        return (rng.standard_normal((K, N, N)) / math.sqrt(N)).astype(np.float32)
    return _random_sparse(rng, K, N, float(kind))


def _sparse(G, dev):
    return torch.from_numpy(np.ascontiguousarray(G)).to(dev).to_sparse()


def _nan(shape, dev):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=dev)


def run_sparse_layer(X, G, W, b, act, d_out, dev):
    """One forward and backward through the C ABI on NaN-prefilled outputs, stash and workspaces -> out, Z, dX, dW, db."""
    lib = _lib.load()
    B, N, _, C = X.shape
    K, H = G.shape[0], W.shape[1]
    Gs = _sparse(G, dev)
    sp, nnz = ops._sparse_supports(lib, Gs, K, N)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    Xt, Wt, bt, dt = t(X), t(W), (None if b is None else t(b)), t(d_out)
    out = _nan((B, N, N, H), dev)
    saved = _nan((lib.mpgcn_bdgcn_saved_bytes(B, N, K, C, H, 0) // 4,), dev)
    ws = _nan((lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, C, H, 0, 0) // 4 + 1,), dev)
    p = lambda x: None if x is None else x.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.mpgcn_bdgcn_forward_sparse(p(Xt), p(sp), sp.numel(), nnz, p(Wt), p(bt), act, p(out), p(saved), p(ws), ws.numel() * 4,
                                              B, N, K, C, H, st), "forward_sparse")
    dX, dW = _nan((B, N, N, C), dev), _nan(tuple(W.shape), dev)
    db = None if b is None else _nan((H,), dev)
    ws = _nan((lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, 0, 0) // 4 + 1,), dev)
    _lib.check(lib.mpgcn_bdgcn_backward_sparse(p(dt), p(out), p(sp), sp.numel(), nnz, p(Wt), act, p(saved), p(dX), p(dW), p(db), p(ws),
                                               ws.numel() * 4, B, N, K, C, H, st), "backward_sparse")
    torch.cuda.synchronize()
    Z = saved[:B * K * N * N * C].view(B, K, N, N, C)
    return out, Z, dX, dW, db


# ------------------------------------------------------------------------------------------------------------------------------
# 1. structure readback
# ------------------------------------------------------------------------------------------------------------------------------
def _read_structure(sp, K, N, nnz):
    """CSR and CSC of the built buffer, in the layout of bdgcn_sparse.cu's sparse_layout"""
    def take(off, nbytes):
        off = (off + 255) // 256 * 256
        return off, off + nbytes
    off, parts = 0, []
    for nbytes in [K * (N + 1) * 4, nnz * 4, nnz * 4] * 2:
        start, off = take(off, nbytes)
        parts.append(sp[start:off])
    i32 = lambda x: x.view(torch.int32).cpu().numpy()
    f32 = lambda x: x.view(torch.float32).cpu().numpy()
    return [(i32(parts[0 + 3 * f]).reshape(K, N + 1), i32(parts[1 + 3 * f]), f32(parts[2 + 3 * f])) for f in range(2)]


STRUCT_CASES = [(K, N) for K in range(1, 10) for N in (1, 2, 47, 129, 1000)]


@pytest.mark.parametrize("K,N", STRUCT_CASES)
def test_structure_equals_torch_conversion(K, N, cuda_device):
    rng = np.random.default_rng(K * 1000 + N)
    G = _random_sparse(rng, K, N, min(1.0, 8.0 / N))
    G[0] = 0.0                                     # an all-zero support
    if N > 2:
        G[:, N // 2, :] = 0.0                      # an empty row and an empty column in every support
        G[:, :, N // 3] = 0.0
    # duplicate COO entries: every stored entry twice, halves of it, uncoalesced
    Gd = torch.from_numpy(G).to_sparse()
    idx, val = Gd.indices(), Gd.values()
    dup = torch.sparse_coo_tensor(torch.cat([idx, idx], 1), torch.cat([val * 0.5, val * 0.5]), G.shape).to(cuda_device)
    assert Gd._nnz() == 0 or not dup.is_coalesced()
    lib = _lib.load()
    sp, nnz = ops._sparse_supports(lib, dup, K, N)
    torch.cuda.synchronize()
    assert nnz == Gd._nnz()
    (rp, ci, rv), (cp, ri, cv) = _read_structure(sp, K, N, nnz)
    for k in range(K):
        ref = torch.from_numpy(G[k]).to_sparse_csr()
        base = rp[k, 0]
        np.testing.assert_array_equal(rp[k] - base, ref.crow_indices().numpy())
        np.testing.assert_array_equal(ci[rp[k, 0]:rp[k, N]], ref.col_indices().numpy())
        np.testing.assert_array_equal(rv[rp[k, 0]:rp[k, N]], ref.values().numpy())
        reft = torch.from_numpy(np.ascontiguousarray(G[k].T)).to_sparse_csr()
        np.testing.assert_array_equal(cp[k] - cp[k, 0], reft.crow_indices().numpy())
        np.testing.assert_array_equal(ri[cp[k, 0]:cp[k, N]], reft.col_indices().numpy())
        np.testing.assert_array_equal(cv[cp[k, 0]:cp[k, N]], reft.values().numpy())
    assert rp[K - 1, N] == cp[K - 1, N] == nnz and rp[0, 0] == cp[0, 0] == 0


# ------------------------------------------------------------------------------------------------------------------------------
# 2. stages against float64
# ------------------------------------------------------------------------------------------------------------------------------
KINDS = ["localpool", "chebyshev", "random_walk_diffusion", "dual_random_walk_diffusion", "identity", "0.001", "0.05", "0.3", "dense"]
WIDTHS = [(1, 5), (5, 1), (32, 48), (48, 32), (64, 96), (96, 64), (5, 32), (1, 96), (96, 1)]
STAGE_CASES = []
for i, kind in enumerate(KINDS):
    for j in range(2):
        C, H = WIDTHS[(2 * i + j) % len(WIDTHS)]
        K = {"localpool": 1, "dual_random_walk_diffusion": 5}.get(kind, 3)
        N = (47, 129, 20, 63)[(i + j) % 4] if kind != "0.001" else 400       # 0.1 %: 160 entries per support
        STAGE_CASES.append((kind, K, N, C, H, (i + j) % 2, j == 0, 2 if N < 200 else 1))


def test_stage_cases_cover_the_issue():
    assert {c[0] for c in STAGE_CASES} == set(KINDS)
    assert {c[3] for c in STAGE_CASES} >= {1, 5, 32, 48, 64, 96} and {c[4] for c in STAGE_CASES} >= {1, 5, 32, 48, 64, 96}
    assert all(c[3] != c[4] for c in STAGE_CASES)
    assert {c[5] for c in STAGE_CASES} == {0, 1} and {c[6] for c in STAGE_CASES} == {False, True}


@pytest.mark.parametrize("kind,K,N,C,H,act,bias,B", STAGE_CASES)
def test_stages_against_float64(kind, K, N, C, H, act, bias, B, cuda_device):
    rng = np.random.default_rng(zlib.crc32(f"{kind} {C} {H}".encode()))
    G = _supports(kind, rng, K, N)
    K = G.shape[0]
    X = rng.standard_normal((B, N, N, C)).astype(np.float32)
    W = (rng.standard_normal((K * K * C, H)) / math.sqrt(K * K * C)).astype(np.float32)
    b = rng.standard_normal(H).astype(np.float32) if bias else None
    d_out = rng.standard_normal((B, N, N, H)).astype(np.float32)
    out, Z, dX, dW, db = run_sparse_layer(X, G, W, b, act, d_out, cuda_device)
    G64, X64 = G.astype(np.float64), X.astype(np.float64)
    Z_ref = np.einsum("bncl,dce->bdnel", X64, G64, optimize=True)
    _check(Z, Z_ref, FWD_TOL, f"{kind} C={C} H={H} Z")
    mode = "relu" if act else None
    ref_out, rdX, rdW, rdb = orc.bdgcn_backward_factored(X64, G64, W.astype(np.float64), b, mode, d_out.astype(np.float64),
                                                         mask_from=out.cpu().numpy() if act else None)
    _check(out, ref_out, FWD_TOL, f"{kind} C={C} H={H} out")
    _check(dX, rdX, BWD_TOL, f"{kind} C={C} H={H} dX")
    _check(dW, rdW, BWD_TOL, f"{kind} C={C} H={H} dW")
    if bias:
        _check(db, rdb, BWD_TOL, f"{kind} C={C} H={H} db")


# ------------------------------------------------------------------------------------------------------------------------------
# 3. identity and empty rows
# ------------------------------------------------------------------------------------------------------------------------------
def test_identity_passes_x_through_and_empty_rows_give_act_bias(cuda_device):
    rng = np.random.default_rng(3)
    B, N, C, H = 2, 33, 5, 7
    X = rng.standard_normal((B, N, N, C)).astype(np.float32)
    W = rng.standard_normal((C, H)).astype(np.float32)
    b = rng.standard_normal(H).astype(np.float32)
    d_out = rng.standard_normal((B, N, N, H)).astype(np.float32)
    _, Z, _, _, _ = run_sparse_layer(X, np.eye(N, dtype=np.float32)[None], W, b, 1, d_out, cuda_device)
    assert torch.equal(Z[:, 0], torch.from_numpy(X).to(cuda_device)), "Z = X x_2 I must be X bitwise"
    G = _random_sparse(rng, 1, N, 0.2)
    G[0, :, 4] = 0.0           # column 4 empty: out[:, 4] (origin m = 4) has no term
    G[0, 9, :] = 0.0           # row 9 empty: no Z / dX term from destination c = 9
    out, Z, dX, _, _ = run_sparse_layer(X, G, W, b, 1, d_out, cuda_device)
    want = torch.from_numpy(np.maximum(b, 0)).to(cuda_device).expand(B, N, H)
    assert torch.equal(out[:, 4], want), "an empty column of G_o gives act(bias) exactly"
    assert torch.equal(Z[:, 0, :, 4], torch.zeros_like(Z[:, 0, :, 4])), "an empty column of G_d gives a zero Z row"
    assert torch.equal(dX[:, :, 9], torch.zeros_like(dX[:, :, 9])), "an empty row of G_d gives a zero dX row"


def test_non_finite_x_does_not_leak_through_zeros(cuda_device):
    rng = np.random.default_rng(4)
    N, C, H = 12, 3, 4
    G = np.eye(N, dtype=np.float32)[None]
    X = rng.standard_normal((1, N, N, C)).astype(np.float32)
    X[0, 2, 5, :] = np.inf            # X[b, n = 2, c = 5]: reaches Z only through G[5, e] != 0, i.e. e = 5
    W = rng.standard_normal((C, H)).astype(np.float32)
    out, Z, _, _, _ = run_sparse_layer(X, G, W, None, 0, np.zeros((1, N, N, H), np.float32), cuda_device)
    Zc = Z.cpu().numpy()[0, 0, 2]
    assert np.isinf(Zc[5]).all() and np.isfinite(np.delete(Zc, 5, axis=0)).all()


# ------------------------------------------------------------------------------------------------------------------------------
# 4. at size against the dense precision-0 layer
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1000, 2000])
def test_at_size_against_dense_fp32_layer(N, cuda_device):
    rng = np.random.default_rng(N)
    K, C, H, B = 3, 64, 64, 1
    G = orc.adj_process(_knn_adjacency(rng, N, 6)[None], "random_walk_diffusion", K - 1)[0].astype(np.float32)
    torch.manual_seed(0)
    layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=H, use_bias=True, activation=nn.ReLU).to(cuda_device)
    layer.precision = "fp32"
    with torch.no_grad():
        layer.b.normal_()
    X = torch.randn(B, N, N, C, device=cuda_device)
    d_out = torch.randn(B, N, N, H, device=cuda_device)
    Gd = torch.from_numpy(G).to(cuda_device)
    res = {}
    for name, g in (("dense", Gd), ("sparse", Gd.to_sparse())):
        Xg = X.clone().requires_grad_(True)
        layer.zero_grad()
        out = layer(Xg, g)
        out.backward(d_out)
        torch.cuda.synchronize()
        res[name] = [out.detach().cpu().numpy(), Xg.grad.cpu().numpy(), layer.W.grad.cpu().numpy(), layer.b.grad.cpu().numpy()]
        del out, Xg
    for what, a, r, tol in zip(("out", "dX", "dW", "db"), res["sparse"], res["dense"], (FWD_TOL, BWD_TOL, BWD_TOL, BWD_TOL)):
        _check(a, r, tol, f"N={N} {what} vs dense fp32")


# ------------------------------------------------------------------------------------------------------------------------------
# 5. reference fixtures with G.to_sparse()
# ------------------------------------------------------------------------------------------------------------------------------
STATIC_LAYER_FIXTURES = [n for p in ("bdgcn_", "big_bdgcn_", "many_bdgcn_", "wide_bdgcn_") for n in golden_names(p) if "bdgcn_s_" in n]


def test_every_static_layer_fixture_is_listed():
    assert len(STATIC_LAYER_FIXTURES) >= 14


@pytest.mark.parametrize("name", STATIC_LAYER_FIXTURES)
def test_static_layer_fixture_with_sparse_supports(name, cuda_device):
    if name.startswith("big_"):     # at-size fixtures: X / d_out from the seed, a subset of origin rows of out / dX
        g, X, d_out, G = load_big(name)
        g = dict(g, X=X, d_out=d_out, out=g["out_rows"], dX=g["dX_rows"])
    else:
        g = layer_fixture(load_golden(name))
    assert not int(g["dynamic"])
    K = int(g["K"])
    C, H = g["X"].shape[-1], g["W"].shape[1]
    layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=H, use_bias="b" in g,
                       activation=nn.ReLU if str(g["act"]) == "relu" else None).to(cuda_device)
    with torch.no_grad():
        layer.W.copy_(torch.from_numpy(g["W"]))
        if "b" in g:
            layer.b.copy_(torch.from_numpy(g["b"]))
    X = torch.from_numpy(g["X"]).to(cuda_device).requires_grad_(True)
    out = layer(X, torch.from_numpy(g["G"]).to(cuda_device).to_sparse())
    out.backward(torch.from_numpy(g["d_out"]).to(cuda_device))
    torch.cuda.synchronize()
    rows = g.get("rows")        # at-size fixtures keep a subset of origin rows of out / dX
    sel = (lambda a: a[:, rows]) if rows is not None else (lambda a: a)
    _check(sel(out.detach().cpu().numpy()), g["out"], FWD_TOL, f"{name} out")
    _check(sel(X.grad.cpu().numpy()), g["dX"], BWD_TOL, f"{name} dX")
    _check(layer.W.grad, g["dW"], BWD_TOL, f"{name} dW")
    if "b" in g:
        _check(layer.b.grad, g["db"], BWD_TOL, f"{name} db")


def _fixture_model(g, dev):
    K, hid = int(g["K"]), int(g["hidden"])
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                       num_nodes=g["x_seq"].shape[2], user_bias=True, activation=nn.ReLU)
    model.load_state_dict({k[6:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("param:")})
    model = model.to(dev)
    model.lstm_precision = "fp32"
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = "fp32"
    return model


@pytest.mark.parametrize("name", golden_names("mpgcn_"))
def test_model_fixture_with_sparse_static_branch(name, cuda_device):
    g = load_golden(name)
    model = _fixture_model(g, cuda_device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)
    G_list = [t(g["G_static"]).to_sparse(), (t(g["G_o"]), t(g["G_d"]))]
    y = model(x_seq=t(g["x_seq"]), G_list=G_list)
    y.backward(t(g["d_y"]))
    torch.cuda.synchronize()
    _check(y, g["y"], FWD_TOL, f"{name} y")
    for k, p in model.named_parameters():
        _check(p.grad, g["grad:" + k], BWD_TOL, f"{name} grad:{k}")


# ------------------------------------------------------------------------------------------------------------------------------
# 6. model behaviour
# ------------------------------------------------------------------------------------------------------------------------------
def _small_model(dev, N=20, K=3, hid=32):
    torch.manual_seed(0)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU).to(dev)
    rng = np.random.default_rng(5)
    G = torch.from_numpy(orc.adj_process(_knn_adjacency(rng, N, 3)[None], "random_walk_diffusion", K - 1)[0].astype(np.float32)).to(dev)
    return model, G.to_sparse(), rng


def _inputs(rng, dev, B, T, N, K):
    t = lambda a: torch.from_numpy(a.astype(np.float32)).to(dev)
    return (t(rng.random((B, T, N, N, 1)) * 4), t(rng.random((B, 1, N, N, 1)) * 4), t(rng.random((B, K, N, N)) / N),
            t(rng.random((B, K, N, N)) / N))


def test_no_grad_allocates_no_stash_and_rollout_matches_eager(cuda_device):
    model, Gs, rng = _small_model(cuda_device)
    x, _, go, gd = _inputs(rng, cuda_device, 2, 4, 20, 3)
    ops.STASH_BYTES.clear()
    with torch.no_grad():
        eager = rollout._eager(model.eval(), x, [Gs, (go, gd)], 3)
    assert ops.STASH_BYTES["bdgcn"] == 0
    graphed = rollout.forecast(model, x, [Gs, (go, gd)], 3, use_cuda_graph=True)
    assert torch.equal(graphed, eager)
    rollout.install(model)
    try:
        with torch.no_grad():
            a, b = model(x_seq=x, G_list=[Gs, (go, gd)]), model(x_seq=x, G_list=[Gs, (go, gd)])
        assert torch.equal(a, eager[:, :1]) and torch.equal(b, a) and model.forward.replays == 2
    finally:
        rollout.uninstall(model)


def test_graphed_train_step_matches_eager(cuda_device):
    # bitwise comparison: the rest of the model (LSTM, head, bias gradients) sums with atomics unless the deterministic mode is on
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        _graphed_vs_eager(cuda_device)
    finally:
        torch.use_deterministic_algorithms(prev)


def _graphed_vs_eager(cuda_device):
    losses = {}
    for graphed in (False, True):
        model, Gs, rng = _small_model(cuda_device)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3, capturable=True)
        batches = [_inputs(rng, cuda_device, 2, 4, 20, 3) for _ in range(3)]
        crit = nn.MSELoss()
        if graphed:
            state = {k: v.clone() for k, v in model.state_dict().items()}
            step = GraphedTrainStep(model, crit, opt, example=(batches[0][0], batches[0][1], Gs, batches[0][2:]), warmup=2)
            with torch.no_grad():      # the warm-up trained: start the replays from the eager run's initial state
                for k, v in model.state_dict().items():
                    v.copy_(state[k])
                for s in opt.state.values():
                    for v in s.values():
                        if torch.is_tensor(v):
                            v.zero_()
            losses[graphed] = [step(*b_).detach().clone() for b_ in batches]
        else:
            out = []
            for x, y, go, gd in batches:
                loss = crit(model(x_seq=x, G_list=[Gs, (go, gd)]), y)
                opt.zero_grad(set_to_none=False)
                loss.backward()
                opt.step()
                out.append(loss.detach().clone())
            losses[graphed] = out
    assert all(torch.equal(a, b) for a, b in zip(losses[False], losses[True])), (losses[False], losses[True])


def test_deterministic_training_steps_are_bitwise_equal(cuda_device):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = []
        for _ in range(2):
            model, Gs, rng = _small_model(cuda_device)
            for mod in model.modules():
                if isinstance(mod, shim.BDGCN):
                    mod.precision = "fp32"
            opt = torch.optim.Adam(model.parameters(), lr=1e-3)
            for _ in range(2):
                x, y, go, gd = _inputs(rng, cuda_device, 2, 4, 20, 3)
                loss = nn.functional.mse_loss(model(x_seq=x, G_list=[Gs, (go, gd)]), y)
                opt.zero_grad()
                loss.backward()
                opt.step()
            runs.append([p.detach().clone() for p in model.parameters()] + [loss.detach()])
        assert all(torch.equal(a, b) for a, b in zip(*runs))
    finally:
        torch.use_deterministic_algorithms(prev)


def test_refusals(cuda_device):
    N, K, C, H = 9, 2, 4, 5
    X = torch.randn(1, N, N, C, device=cuda_device)
    W = torch.randn(K * K * C, H, device=cuda_device)
    G = torch.rand(K, N, N, device=cuda_device)
    Gs = G.to_sparse()
    with pytest.raises(NotImplementedError, match="dynamic"):
        ops.bdgcn(X, (Gs.unsqueeze(0), G.unsqueeze(0)), W, None, True)
    with pytest.raises(NotImplementedError, match="no gradient"):
        ops.bdgcn(X, Gs.clone().requires_grad_(True), W, None, True, support_grad=True)
    with pytest.raises(RuntimeError, match="no fp16 sparse kernels"):
        ops.bdgcn(X, Gs, W, None, True, precision="fp16")
    with pytest.raises(NotImplementedError, match="COO"):
        ops.bdgcn(X, G.to_sparse_csr(), W, None, True)
    with pytest.raises(NotImplementedError, match="COO"):
        ops.bdgcn(X, G.cpu().to_sparse_bsr((1, 1)).to(cuda_device), W, None, True)
    with pytest.raises(ValueError, match="dense"):
        ops.bdgcn(X, G.unsqueeze(-1).to_sparse(3), W, None, True)
    with pytest.raises(ValueError, match="floating"):
        ops.bdgcn(X, (G > 0.5).to(torch.int32).to_sparse(), W, None, True)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.bdgcn(X, Gs.cpu(), W, None, True)
    layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=H, activation=nn.ReLU).to(cuda_device)
    with pytest.raises(NotImplementedError, match="sharded layers take dense supports"):
        shard.sharded_bdgcn(layer, X, Gs, plan=None)


def test_in_place_edit_of_sparse_values_is_picked_up(cuda_device):
    N, K, C, H = 15, 2, 3, 4
    X = torch.randn(1, N, N, C, device=cuda_device)
    W = torch.randn(K * K * C, H, device=cuda_device)
    G = (torch.rand(K, N, N, device=cuda_device) * (torch.rand(K, N, N, device=cuda_device) < 0.3)).to_sparse()
    with torch.no_grad():
        a = ops.bdgcn(X, G, W, None, False)
        G._values().mul_(2.0)
        b = ops.bdgcn(X, G, W, None, False)
        ref = ops.bdgcn(X, G.to_dense(), W, None, False, precision="fp32")
    torch.testing.assert_close(b, 4 * a, rtol=1e-5, atol=1e-5)       # G enters twice (G_o^T X G_d)
    torch.testing.assert_close(b, ref, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------------------------------------
# 7. the trainer
# ------------------------------------------------------------------------------------------------------------------------------
REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "Main.py")), reason="oracle/_ref (the unmodified reference) is not installed")
def test_trainer_with_sparse_static_supports_matches_dense(tmp_path, monkeypatch):
    from test_trainer_dropin import run_main, val_losses, write_synthetic_data
    data = tmp_path / "data"
    data.mkdir()
    write_synthetic_data(str(data))
    monkeypatch.setenv("MPGCN_B200_PRECISION", "fp32")
    losses = {}
    for flag in ([], ["--sparse-static-supports"]):
        out = tmp_path / ("out" + "".join(flag))
        common = ["-GPU", "cuda:0", "-in", str(data), "-out", str(out), "-batch", "4", "-lr", "1e-3", "-mode", "train", "-epoch", "2"]
        losses[bool(flag)] = val_losses(run_main(["--seed", "0"] + flag, common))
    assert len(losses[True]) == len(losses[False]) == 2, losses
    np.testing.assert_allclose(losses[True], losses[False], rtol=1e-4)
