"""Stacked LSTMs (lstm_num_layers = L >= 2) on the tensor cores at hidden 32 and 96.

Every layer runs the width-generic kernels of lstm_tc.cu (hidden 32 as one 32-unit slice); a layer above the first takes
h^{l-1}_t of the layer below as a second H-deep block of its gate GEMM, and its backward walk hands d(h^{l-1}_t) down.
Hidden 128 and every other configuration keep nn.LSTM, in the model and in the sharded model alike (ops.lstm_runs_on_engine).

  * CPU: the float64 stacked oracle (tests/lstm_stack_oracle.py) against fixtures of the unmodified reference
    (`tests/golden/lstms_*`, `mpgcns_*`, tools/gen_golden_stacked_lstm.py); the support query and sizes; the dispatch rule.
  * GPU: the stack against the fixtures and against float64 (ragged cell counts, T = 1, 7, 256, tiny / huge gradients,
    saturated gates); a row slab; refused buffers; the whole model (no nn.LSTM, fixtures, no stash under no_grad, CUDA-graph
    rollout); the dispatch of everything the engine does not run; the sharded model with NCCL.

Bounds are those of the single-layer path: h_T 1e-3, gradients 2e-3.
"""
import numpy as np
import pytest
import torch
from torch import nn

import _shard_nccl_worker as nccl_worker
from conftest import golden_names, load_golden, record_parity
from oracle import lstm_tc_oracle as emu
from oracle import mpgcn_oracle as orc
import lstm_stack_oracle as sorc

import MPGCN as shim
from mpgcn_b200 import _lib, ops
from tools.gen_golden_stacked_lstm import KEYS, stacked_lstm_params
from tools.gen_golden_wide import params_checksum, wide_model_params

FIXTURE_TOL = 2e-5
H_TOL, G_TOL = 1e-3, 2e-3
FP16_MODEL_FWD_TOL = 3.5e-3     # whole model in fp16 against the reference (test_gpu_lstm_widths.py, DESIGN.md section 3)
MODEL_GRAD_TOL = 5e-3           # whole model, against the oracle on the engine's ReLU masks
WIDTHS = (32, 96)


def _rel_check(a, ref, tol, what, l2_only=False):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    ref = ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol), f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"
    return linf, l2


def _fixture_params(g):
    params = stacked_lstm_params(int(g["seed"]), int(g["C"]), int(g["L"]))
    assert abs(float(params_checksum(params)) - float(g["params_checksum"])) < 1e-6, "numpy RNG stream changed: regenerate the fixture"
    return params


def _layers(params, L, dtype=np.float64):
    return [tuple(params[f"{k}_l{l}"].astype(dtype) for k in KEYS) for l in range(L)]


def _check_fixture_grad(a, g, key, tol, what):
    """One gradient against an `lstms_` fixture: on its stored rows and in norm when only those were kept, else in full."""
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    if key in g:
        return _rel_check(a, g[key], tol, f"{what}/{key}")
    _rel_check(a[g[key + "_row_ids"]], g[key + "_rows"], tol, f"{what}/{key} rows")
    ref = float(g[key + "_norm"])
    assert abs(float(np.linalg.norm(a.astype(np.float64))) - ref) <= tol * ref, f"{what}/{key}: norm of the whole tensor"


def _model(N, K, hid, seed, dev, L=2, **kw):
    torch.manual_seed(seed)
    m = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=L, gcn_hidden_dim=hid, gcn_num_layers=3, num_nodes=N,
                   user_bias=True, activation=nn.ReLU)
    for branch in m.branch_models:          # nn.LSTM's dropout between layers is a constructor argument of the module
        if "dropout" in kw:
            branch['temporal'].dropout = kw["dropout"]
    return m.to(dev)


def _model_params(g):
    hid, K, N, L = int(g["hidden"]), int(g["K"]), g["x_seq"].shape[2], int(g["lstm_num_layers"])
    shapes = {k: v.shape for k, v in _model(N, K, hid, 0, "cpu", L).state_dict().items()}
    params = wide_model_params(int(g["seed"]), shapes)
    assert abs(float(params_checksum(params)) - float(g["params_checksum"])) < 1e-6, "numpy RNG stream changed: regenerate the fixture"
    return params


def _check_model_grads(grads, g, tol, what, l2_only=False):
    assert set(grads) == {k.split(":", 1)[1] for k in g if k.startswith(("grad:", "grad_rows:"))}
    for k, v in grads.items():
        v = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        if "grad_rows:" + k in g:
            _rel_check(v[g["grad_row_ids:" + k]], g["grad_rows:" + k], tol, f"{what}/grad:{k} rows", l2_only)
            ref = float(g["grad_norm:" + k])
            assert abs(float(np.linalg.norm(v.astype(np.float64))) - ref) <= tol * ref, f"{what}/grad:{k}: norm of the whole tensor"
        else:
            _rel_check(v, g["grad:" + k], tol, f"{what}/grad:{k}", l2_only)


# ------------------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------------------
def test_stacked_fixtures_exist_and_stay_out_of_the_other_sets():
    lstms, models = golden_names("lstms_"), golden_names("mpgcns_")
    cases = {(int(load_golden(n)["C"]), int(load_golden(n)["L"]), load_golden(n)["x"].shape[1]) for n in lstms}
    assert {c for c, _, _ in cases} == set(WIDTHS) and {l for _, l, _ in cases} == {2, 3} and {t for _, _, t in cases} == {1, 7}
    assert all(load_golden(n)["x"].shape[0] % 64 for n in lstms)
    assert {int(load_golden(n)["hidden"]) for n in models} == set(WIDTHS)
    for prefix in ("lstm_", "lstmw_", "mpgcn_", "mpgcnw_"):
        assert not set(lstms + models) & set(golden_names(prefix))


@pytest.mark.parametrize("name", golden_names("lstms_"))
def test_oracle_matches_reference_stacked_lstm(name):
    g = load_golden(name)
    L = int(g["L"])
    layers = _layers(_fixture_params(g), L)
    x = g["x"].astype(np.float64)
    _rel_check(sorc.lstm_stack_forward(x, layers), g["hT"], FIXTURE_TOL, f"{name}: hT")
    dx, grads = sorc.lstm_stack_backward(x, layers, g["d_hT"].astype(np.float64))
    _rel_check(dx, g["dx"], FIXTURE_TOL, f"{name}: dx")
    for l in range(L):
        for k, a in zip(KEYS, grads[l]):
            _check_fixture_grad(a, g, f"d{k}_l{l}", FIXTURE_TOL, name)


@pytest.mark.parametrize("name", golden_names("mpgcns_"))
def test_oracle_matches_reference_stacked_model(name):
    g = load_golden(name)
    y, grads = sorc.mpgcn_forward_backward(_model_params(g), g["x_seq"], [g["G_static"], (g["G_o"], g["G_d"])], M=2, gcn_num_layers=3,
                                           L=int(g["lstm_num_layers"]), d_y=g["d_y"])
    _rel_check(y, g["y"], FIXTURE_TOL, f"{name}: y")
    _check_model_grads(grads, g, FIXTURE_TOL, name)


def test_stack_support_query_and_sizes():
    lib = _lib.load()
    fp16, fp32 = _lib.PREC_FP16_TC, _lib.PREC_FP32
    for C in WIDTHS:
        for L in (2, 3, 8):
            assert lib.mpgcn_lstm_stack_supported(1, C, L, fp16) == 1 and lib.mpgcn_lstm_stack_supported(256, C, L, fp16) == 1
            assert lib.mpgcn_lstm_stack_supported(257, C, L, fp16) == 0 and lib.mpgcn_lstm_stack_supported(0, C, L, fp16) == 0
            assert lib.mpgcn_lstm_stack_supported(12, C, L, fp32) == 0
            B, T, NN = 3, 5, 1000
            assert lib.mpgcn_lstm_stack_saved_bytes(B, T, NN, C, L, fp16) == L * lib.mpgcn_lstm_saved_bytes(B, T, NN, C, fp16)
            assert lib.mpgcn_lstm_stack_fwd_workspace_bytes(B, T, NN, C, L, fp16) >= (1 if L == 2 else 2) * B * T * NN * C * 2
            assert lib.mpgcn_lstm_stack_bwd_workspace_bytes(B, T, NN, C, L, fp16) >= B * T * NN * C * (8 + 4)
    for C in (16, 64, 128, 160):
        assert lib.mpgcn_lstm_stack_supported(12, C, 2, fp16) == 0
        assert lib.mpgcn_lstm_stack_saved_bytes(2, 12, 100, C, 2, fp16) == 0
    for T, C, p in ((12, 32, fp16), (12, 64, fp32), (300, 128, fp16), (16, 64, fp32)):      # L = 1: the single-layer query
        assert lib.mpgcn_lstm_stack_supported(T, C, 1, p) == lib.mpgcn_lstm_precision_supported(T, C, p)


@pytest.mark.parametrize("hid,L,T,prec,dropout,training,engine", [
    (32, 2, 12, None, 0.0, True, True), (96, 3, 256, "auto", 0.0, True, True), (32, 2, 12, "fp16", 0.0, True, True),
    (128, 2, 12, None, 0.0, True, False), (64, 2, 12, "fp16", 0.0, True, False), (16, 2, 12, None, 0.0, True, False),
    (32, 2, 300, None, 0.0, True, False), (32, 2, 12, "fp32", 0.0, True, False), (96, 2, 12, None, 0.5, True, False),
    (96, 2, 12, None, 0.5, False, True), (32, 1, 12, None, 0.0, True, True), (64, 1, 16, "auto", 0.0, True, False)])
def test_engine_or_nn_lstm_is_one_rule(hid, L, T, prec, dropout, training, engine, monkeypatch):
    """ops.lstm_runs_on_engine, which the model and the sharded model both ask: stacks on the engine at hidden 32 / 96, T <= 256,
    tensor-core precision, no dropout in training; the single-layer rule unchanged."""
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    lstm = nn.LSTM(1, hid, L, batch_first=True, dropout=dropout)
    lstm.train(training)
    assert ops.lstm_runs_on_engine(lstm, T, prec) == engine
    assert not ops.lstm_runs_on_engine(nn.LSTM(2, hid, L, batch_first=True), T, prec)
    for kw in (dict(bias=False), dict(bidirectional=True), dict(proj_size=hid // 2), dict(batch_first=False)):
        assert not ops.lstm_runs_on_engine(nn.LSTM(1, hid, L, **{"batch_first": True, **kw}), T, prec), kw


@pytest.mark.parametrize("H", WIDTHS)
def test_dseq_decoder_inverts_the_kernel_layout(H):
    """decode_dseq against a buffer filled by the formula of dseq_off: (((tile T + t) NW + warp) 512 + lane 16 + slot) holds
    cell tile CELLS + 16 cg + g + 8 h2, unit 32 js + 8 jn + 2 q + e, with warp = cg CH + js, lane = 4 g + q, slot = 8 h2 + 2 jn + e."""
    CH, CG, CELLS = emu.dims(H)
    cells, T = CELLS + 5, 3
    nt = emu.tiles(cells, H)
    buf = np.zeros(nt * T * CELLS * H, np.float32)
    want = np.zeros((cells, T, H))
    for tile in range(nt):
        for t in range(T):
            for w in range(CG * CH):
                for lane in range(32):
                    for slot in range(16):
                        cell = tile * CELLS + 16 * (w // CH) + lane // 4 + 8 * (slot // 8)
                        unit = 32 * (w % CH) + 8 * ((slot % 8) // 2) + 2 * (lane % 4) + slot % 2
                        v = 1 + cell * 1000 + t * 10 ** 6 + unit * 1e-3
                        buf[(((tile * T + t) * CG * CH + w) * 512) + lane * 16 + slot] = v
                        if cell < cells:
                            want[cell, t, unit] = np.float32(v)
    assert np.array_equal(sorc.decode_dseq(buf, cells, T, H), want)
    assert np.array_equal(sorc.decode_dseq(sorc.encode_dseq(want, H), cells, T, H), want)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: the LSTM alone
# ------------------------------------------------------------------------------------------------------------------------------
def _t(a, dev, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev).requires_grad_(grad)


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("lstms_"))
def test_stack_matches_reference_fixture(name, cuda_device):
    g = load_golden(name)
    L = int(g["L"])
    p = _fixture_params(g)
    S, T, _ = g["x"].shape
    x = _t(np.ascontiguousarray(g["x"][:, :, 0].T)[None], cuda_device, grad=True)        # [1,T,S]
    ws = [_t(p[f"{k}_l{l}"], cuda_device, grad=True) for l in range(L) for k in KEYS]
    hT = ops.lstm_stack(x.view(1, T, S, 1, 1), ws)
    hT.backward(_t(g["d_hT"], cuda_device))
    torch.cuda.synchronize()
    _rel_check(hT, g["hT"], H_TOL, f"{name}/hT")
    for i, w in enumerate(ws):
        _check_fixture_grad(w.grad, g, f"d{KEYS[i % 4]}_l{i // 4}", G_TOL, name)
    _rel_check(x.grad[0].T, g["dx"][:, :, 0], G_TOL, f"{name}/dx")


def _random_stack(C, L, seed):
    torch.manual_seed(seed)
    lstm = nn.LSTM(1, C, L, batch_first=True)
    return [getattr(lstm, f"{k}_l{l}").detach().clone() for l in range(L) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]


@pytest.mark.gpu
@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("L", (2, 3))
@pytest.mark.parametrize("S,T,gmag,xmag", [(300, 7, 1.0, 8.0), (129, 1, 1.0, 8.0), (130, 256, 1.0, 8.0), (200, 5, 1e-7, 8.0),
                                            (200, 5, 1e4, 8.0), (200, 6, 1.0, 3000.0)])
def test_stack_matches_float64(C, L, S, T, gmag, xmag, cuda_device):
    """Ragged tile counts (2 S cells, not whole 128- or 64-cell tiles), T = 1, 7 and 256, d_hT at 1e-7 and 1e4, and saturated
    gates (|x| ~ 3000): every output of the stack against the float64 oracle."""
    ws0 = _random_stack(C, L, S + T + C + L)
    x0 = torch.rand(2, T, S, 1, 1) * xmag
    d_h = torch.randn(2 * S, C) * gmag
    ws = [w.to(cuda_device).requires_grad_(True) for w in ws0]
    x = x0.to(cuda_device).requires_grad_(True)
    h = ops.lstm_stack(x, ws)
    h.backward(d_h.to(cuda_device))
    torch.cuda.synchronize()
    xs = x0[:, :, :, 0, 0].permute(0, 2, 1).reshape(2 * S, T, 1).double().numpy()
    layers = [tuple(w.double().numpy() for w in ws0[4 * l:4 * l + 4]) for l in range(L)]
    tag = f"C={C} L={L} S={S} T={T} |dh|={gmag:g} |x|={xmag:g}"
    _rel_check(h, sorc.lstm_stack_forward(xs, layers), H_TOL, f"{tag} hT")
    dx, grads = sorc.lstm_stack_backward(xs, layers, d_h.double().numpy())
    for i, w in enumerate(ws):
        _rel_check(w.grad, grads[i // 4][i % 4], G_TOL, f"{tag} {KEYS[i % 4]}_l{i // 4}")
    _rel_check(x.grad[:, :, :, 0, 0].permute(0, 2, 1).reshape(2 * S, T, 1), dx, G_TOL, f"{tag} dx")


@pytest.mark.gpu
@pytest.mark.parametrize("C", WIDTHS)
def test_stack_row_slab_is_bitwise_the_whole_and_inference_equals_training(C, cuda_device):
    """The sharded model runs the stack on its origin rows: those rows of h_T are bitwise the whole run's.  The inference forward
    (h sequences only) gives the training forward's bits."""
    B, T, N, L = 2, 6, 37, 3
    ws = [w.to(cuda_device) for w in _random_stack(C, L, 11)]
    x = torch.rand(B, T, N, N, 1, device=cuda_device) * 8
    with torch.no_grad():
        whole = ops.lstm_stack(x, ws).view(B, N, N, C)
        for r0, r1 in ((0, 1), (5, 29), (30, 37)):
            part = ops.lstm_stack(x[:, :, r0:r1].contiguous(), ws).view(B, r1 - r0, N, C)
            assert torch.equal(part, whole[:, r0:r1]), (r0, r1)
    train = ops.lstm_stack(x, [w.requires_grad_(True) for w in ws]).view(B, N, N, C)
    assert torch.equal(train.detach(), whole)


@pytest.mark.gpu
def test_stack_refuses_small_buffers_and_unsupported_shapes(cuda_device):
    lib = _lib.load()
    B, T, S, C, L, prec = 2, 4, 100, 32, 2, _lib.PREC_FP16_TC
    st = torch.cuda.current_stream().cuda_stream
    ws = [w.to(cuda_device).contiguous() for w in _random_stack(C, L, 3)]
    arr = lambda ts: ops._ptr_array(ts)  # noqa: E731
    P = [arr(ws[k::4]) for k in range(4)]
    x = torch.rand(B, T, S, device=cuda_device)
    hT = torch.empty(B * S, C, device=cuda_device)
    nsave = lib.mpgcn_lstm_stack_saved_bytes(B, T, S, C, L, prec)
    saved = torch.empty(nsave, dtype=torch.uint8, device=cuda_device)
    rc = lib.mpgcn_lstm_stack_forward(x.data_ptr(), L, *P, hT.data_ptr(), saved.data_ptr(), nsave - 1, None, 0, B, T, S, C, prec, st)
    assert rc != 0 and b"saved buffer too small" in lib.mpgcn_last_error()
    nfw = lib.mpgcn_lstm_stack_fwd_workspace_bytes(B, T, S, C, L, prec)
    wsb = torch.empty(nfw, dtype=torch.uint8, device=cuda_device)
    rc = lib.mpgcn_lstm_stack_forward(x.data_ptr(), L, *P, hT.data_ptr(), None, 0, wsb.data_ptr(), nfw - 1, B, T, S, C, prec, st)
    assert rc != 0 and b"workspace too small" in lib.mpgcn_last_error()
    _lib.check(lib.mpgcn_lstm_stack_forward(x.data_ptr(), L, *P, hT.data_ptr(), saved.data_ptr(), nsave, None, 0, B, T, S, C, prec, st), "fwd")
    g = [torch.empty_like(w) for w in ws]
    G = [arr(g[k::4]) for k in range(4)]
    d_h = torch.randn(B * S, C, device=cuda_device)
    nbw = lib.mpgcn_lstm_stack_bwd_workspace_bytes(B, T, S, C, L, prec)
    wsb = torch.empty(nbw, dtype=torch.uint8, device=cuda_device)
    rc = lib.mpgcn_lstm_stack_backward(x.data_ptr(), L, *P, d_h.data_ptr(), *G, None, saved.data_ptr(), nsave, wsb.data_ptr(), nbw - 1,
                                       B, T, S, C, prec, None, st)
    assert rc != 0 and b"workspace too small" in lib.mpgcn_last_error()
    rc = lib.mpgcn_lstm_stack_backward(x.data_ptr(), L, *P, d_h.data_ptr(), *G, None, saved.data_ptr(), nsave - 1, wsb.data_ptr(), nbw,
                                       B, T, S, C, prec, None, st)
    assert rc != 0 and b"saved buffer too small" in lib.mpgcn_last_error()
    with pytest.raises(ValueError):
        ops.lstm_stack(x.view(B, T, S, 1, 1), [w.t() if i == 1 else w for i, w in enumerate(ws)] + ws[4:])   # a transposed W_hh
    with pytest.raises(ValueError):
        ops.lstm_stack(x.view(B, T, S, 1, 1), ws[:4] + [ws[0]] + ws[5:])                                   # layer 1 given W_ih_l0
    for T_, C_, L_ in ((257, 32, 2), (4, 128, 2), (4, 64, 2), (4, 32, 1)):
        rc = lib.mpgcn_lstm_stack_forward(x.data_ptr(), L_, *P, hT.data_ptr(), None, 0, wsb.data_ptr(), nbw, B, T_, S, C_, prec, st)
        assert rc != 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: the model
# ------------------------------------------------------------------------------------------------------------------------------
def _set_precision(model, prec):
    model.lstm_precision = prec
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = prec


def _count_nn_lstm(model):
    calls = []
    for branch in model.branch_models:
        branch['temporal'].register_forward_hook(lambda *a: calls.append(1))
    return calls


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("mpgcns_"))
def test_stacked_model_matches_reference_fixture(name, cuda_device):
    """(a) LSTM "fp16", BDGCN layers fp32: y within 1e-3 of the reference, gradients within 5e-3 of the oracle's on the engine's
    ReLU masks; (b) the whole model "fp16": y within FP16_MODEL_FWD_TOL of the reference.  No nn.LSTM forward runs."""
    g = load_golden(name)
    params = _model_params(g)
    K, hid, L, N = int(g["K"]), int(g["hidden"]), int(g["lstm_num_layers"]), g["x_seq"].shape[2]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)  # noqa: E731
    for layer_prec, ytol in (("fp32", H_TOL), ("fp16", FP16_MODEL_FWD_TOL)):
        model = _model(N, K, hid, 0, "cpu", L)
        model.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
        model = model.to(cuda_device)
        _set_precision(model, layer_prec)
        model.lstm_precision = "fp16"
        calls = _count_nn_lstm(model)
        caps = {m: {"layers": [], "fc": None} for m in range(2)}
        hooks = [layer.register_forward_hook(lambda mod, inp, out, m=m: caps[m]["layers"].append(out.detach().cpu().numpy()))
                 for m in range(2) for layer in model.branch_models[m]['spatial']]
        y = model(x_seq=t(g["x_seq"]), G_list=[t(g["G_static"]), (t(g["G_o"]), t(g["G_d"]))])
        y.backward(t(g["d_y"]))
        torch.cuda.synchronize()
        for h in hooks:
            h.remove()
        assert not calls, "nn.LSTM ran instead of the engine"
        _rel_check(y, g["y"], ytol, f"{name}/lstm fp16, layers {layer_prec}/y", l2_only=True)
        for m in range(2):
            fc = model.branch_models[m]['fc'][0]
            caps[m]["fc"] = orc.fc_relu_forward(caps[m]["layers"][-1], fc.weight.detach().cpu().numpy(), fc.bias.detach().cpu().numpy())
        _, grads_m = sorc.mpgcn_forward_backward(params, g["x_seq"], [g["G_static"], (g["G_o"], g["G_d"])], M=2, gcn_num_layers=3, L=L,
                                                 d_y=g["d_y"], masks=caps)
        for k, p in model.named_parameters():
            _rel_check(p.grad, grads_m[k], MODEL_GRAD_TOL, f"{name}/layers {layer_prec}/grad:{k} (engine masks)", l2_only=True)


@pytest.mark.gpu
@pytest.mark.parametrize("hid", WIDTHS)
def test_stacked_model_runs_no_nn_lstm_keeps_no_stash_under_no_grad_and_graph_rollout_equals_eager(hid, cuda_device):
    from mpgcn_b200 import rollout
    dev = cuda_device
    N, K, B, T, P = 23, 3, 2, 5, 3
    model = _model(N, K, hid, 3, dev, L=2)
    _set_precision(model, "auto")
    calls = _count_nn_lstm(model)
    G = torch.rand(K, N, N, device=dev) / N
    dyn = (torch.rand(B, K, N, N, device=dev) / N, torch.rand(B, K, N, N, device=dev) / N)
    x = torch.rand(B, T, N, N, 1, device=dev) * 8
    ops.STASH_BYTES.clear()
    with torch.no_grad():
        y0 = model(x_seq=x, G_list=[G, dyn])
    assert sum(ops.STASH_BYTES.values()) == 0, dict(ops.STASH_BYTES)
    y1 = model(x_seq=x, G_list=[G, dyn])
    assert ops.STASH_BYTES["lstm"] > 0 and torch.equal(y0, y1.detach())
    y1.sum().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())
    eager = rollout.forecast(model, x, [G, dyn], P, use_cuda_graph=False)
    graphed = rollout.forecast(model, x, [G, dyn], P, use_cuda_graph=True)
    assert tuple(graphed.shape) == (B, P, N, N, 1)
    assert torch.equal(eager, graphed)
    assert not calls, "nn.LSTM ran instead of the engine"


@pytest.mark.gpu
@pytest.mark.parametrize("hid,T,prec,dropout", [(128, 4, None, 0.0), (64, 4, None, 0.0), (16, 4, None, 0.0), (32, 300, None, 0.0),
                                                (32, 4, "fp32", 0.0), (96, 4, "auto", 0.3)])
def test_stacked_model_keeps_nn_lstm_where_the_engine_has_no_kernel(hid, T, prec, dropout, cuda_device, monkeypatch):
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    N = 5
    model = _model(N, 2, hid, 5, cuda_device, L=2, dropout=dropout)
    model.lstm_precision = prec
    calls = _count_nn_lstm(model)
    x = torch.rand(2, T, N, N, 1, device=cuda_device) * 4
    y = model(x_seq=x, G_list=[torch.rand(2, N, N, device=cuda_device) / N,
                               (torch.rand(2, 2, N, N, device=cuda_device) / N, torch.rand(2, 2, N, N, device=cuda_device) / N)])
    y.sum().backward()
    assert len(calls) == 2


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: the sharded model
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("world", (1, 2))
def test_sharded_model_with_stacked_lstm_matches_the_whole_model(world, tmp_path):
    """shard.sharded_forward with lstm_num_layers = 2 (row shard, NCCL) against the whole model on one GPU at the bars of
    test_gpu_shard.py; the sharded model runs the model's own dispatch, so hidden 64 at T = 16 falls back to nn.LSTM there too."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    # (hidden, T, LSTM precision, forward / gradient bars): the tensor-core stacks at 32 and 96, and hidden 64 at T = 16, which the
    # model runs on nn.LSTM (the fp32 kernels' backward does not hold 16 steps at 64); the layers on the fp32 engine
    models = [dict(N=40, T=T, hidden=hid, gcn_hidden=32, lstm_layers=2, seed=hid, yardstick="same", cases=[(prec, "fp32", tol_f, tol_g)])
              for hid, T, prec, tol_f, tol_g in ((32, 5, "fp16", 1e-3, 8e-2), (96, 4, "fp16", 1e-3, 8e-2), (64, 16, "auto", 1e-5, 2e-3))]
    rows = nccl_worker.run(world, tmp_path, models)["rows"]
    assert {row["hid"] for row in rows} == {32, 96, 64}
    for row in rows:
        record_parity(row["what"], row["linf"], row["l2"], row["tol"])
        assert row["err"] <= row["tol"], row


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: every stage of every layer against the rounding emulation (the bounds of test_gpu_lstm_stages.py)
# ------------------------------------------------------------------------------------------------------------------------------
def _run_stack_stages(x, ws, d_hT, C, L, dev):
    """Training forward + backward through the C ABI into NaN-prefilled buffers, with a workspace that keeps every layer's da
    records -> per layer the decoded saved c / h, da records and gradients; the final d_seq; h_T; dx; the gradient scale."""
    from test_gpu_lstm_stages import _garbage
    lib = _lib.load()
    B, T, NN = x.shape
    cells, prec = B * NN, _lib.PREC_FP16_TC
    st = torch.cuda.current_stream().cuda_stream
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    xt, wt, dh = t(x), [t(w) for w in ws], t(d_hT)
    P = [ops._ptr_array(wt[k::4]) for k in range(4)]
    hT = torch.full((cells, C), float("nan"), device=dev)
    nsave = lib.mpgcn_lstm_stack_saved_bytes(B, T, NN, C, L, prec)
    saved = _garbage(nsave, dev)
    _lib.check(lib.mpgcn_lstm_stack_forward(xt.data_ptr(), L, *P, hT.data_ptr(), saved.data_ptr(), nsave, None, 0, B, T, NN, C, prec, st),
               "stack_forward")
    nt, tile = emu.tiles(cells, C), emu.dims(C)[2]
    dseq_bytes = -(-nt * tile * T * C * 4 // 256) * 256
    da_bytes = nt * tile * T * 4 * C * 2
    da_region = -(-da_bytes // 256) * 256
    nws = lib.mpgcn_lstm_stack_bwd_workspace_bytes(B, T, NN, C, L, prec)
    assert nws == emu.GRAD_SCALE_BYTES + dseq_bytes + da_region
    wsb = _garbage(nws + (L - 1) * da_region, dev)
    g = [torch.full_like(w, float("nan")) for w in wt]
    G = [ops._ptr_array(g[k::4]) for k in range(4)]
    dx = torch.full_like(xt, float("nan"))
    _lib.check(lib.mpgcn_lstm_stack_backward(xt.data_ptr(), L, *P, dh.data_ptr(), *G, dx.data_ptr(), saved.data_ptr(), nsave,
                                             wsb.data_ptr(), wsb.numel(), B, T, NN, C, prec, None, st), "stack_backward")
    torch.cuda.synchronize()
    per = nsave // L
    state = saved.view(torch.float16).cpu().numpy()
    f64 = lambda a: a.detach().cpu().numpy().astype(np.float64)  # noqa: E731
    r = dict(hT=f64(hT), scale2=f64(wsb[:8].view(torch.float32)), dx=f64(dx).transpose(0, 2, 1).reshape(cells, T), layers=[])
    o = emu.GRAD_SCALE_BYTES
    r["d_seq"] = sorc.decode_dseq(wsb[o:o + dseq_bytes].view(torch.float32).cpu().numpy(), cells, T, C)
    for l in range(L):
        c, h = emu.decode_saved(state[l * per // 2:(l + 1) * per // 2], cells, T, C)
        ro = o + dseq_bytes + l * da_region
        da = emu.decode_da_records(wsb[ro:ro + da_bytes].view(torch.float16).cpu().numpy(), cells, T, C)
        gl = [f64(a) for a in g[4 * l:4 * l + 4]]
        r["layers"].append(dict(c=c, h=h, da=da, dw_ih=gl[0][:, 0] if l == 0 else gl[0], dw_hh=gl[1], db=gl[2], db_hh=gl[3]))
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("L", (2, 3))
@pytest.mark.parametrize("T", (1, 7))
def test_stack_every_stage_matches_the_emulation(C, L, T, cuda_device):
    """Each layer's saved c_t / h_t (upper layers driven by the kernel's saved h of the layer below), h_T, the da records of every
    layer, the d(h^{l-1}_t) sequence handed down, every weight gradient and dx, against the emulation of the kernels' roundings
    (tests/lstm_stack_oracle.py) at the stage bounds of test_gpu_lstm_stages.py.  Cells: two batches of half a tile + 3."""
    from test_gpu_lstm_stages import _assert_and_record, dw_coef, store_coef
    B, NN = 2, emu.dims(C)[2] // 2 + 3
    cells = B * NN
    rng = np.random.default_rng(C + 10 * L + T)
    ws = [w.numpy() for w in _random_stack(C, L, C + L + T)]
    x = (rng.random((B, T, NN)) * 8).astype(np.float32)
    x_cells = np.ascontiguousarray(x.transpose(0, 2, 1)).reshape(cells, T)
    d_hT = rng.standard_normal((cells, C)).astype(np.float32)
    r = _run_stack_stages(x, ws, d_hT, C, L, cuda_device)
    tag = f"stack C={C} L={L} T={T}"
    lay = r["layers"]
    assert np.array_equal(lay[-1]["h"][:, -1], emu.f16(r["hT"])), f"{tag}: decoded saved h_(T-1) of the top != fp16(h_T)"
    S, invS = emu.expected_scale(float(np.abs(d_hT).max()))
    assert tuple(r["scale2"]) == (S, invS), f"{tag}: gradient scale {tuple(r['scale2'])}"
    res, l2 = {}, {}
    for l, k in enumerate(lay):
        assert not np.isnan(k["c"]).any() and not np.isnan(k["h"]).any(), f"{tag}: layer {l} saved state has unwritten halves"
        assert np.array_equal(k["db"], k["db_hh"]), f"{tag}: layer {l} d_b_hh != d_b_ih"
        assert not k["da"][cells:].any(), f"{tag}: layer {l} da records of the padded cells are not zero"
        w = ws[4 * l:4 * l + 4]
        fwd = emu.forward(x_cells, *w, h_saved=k["h"]) if l == 0 else sorc.forward_up(lay[l - 1]["h"], *w, h_saved=k["h"])
        e_c, e_h = emu.forward_error_scale(fwd)
        res[f"L{l} fwd c_t"] = store_coef(k["c"], fwd["c"], e_c, True)
        res[f"L{l} fwd h_t"] = store_coef(k["h"], fwd["h"], e_h, True)
        if l == L - 1:
            res[f"L{l} fwd h_T"] = store_coef(r["hT"], fwd["h"][:, -1], e_h[:, -1], False)
    # the walks top-down: the top seeded by d_hT; a middle layer by the d_in its upper neighbour's emulated walk forms from the
    # kernel's records (the kernel's own sequence of it is overwritten in place); the bottom by the kernel's final d_seq
    d_in_above = None
    for l in reversed(range(L)):
        k, w = lay[l], ws[4 * l:4 * l + 4]
        dh_in = None if l == L - 1 else (r["d_seq"] if l == 0 else d_in_above)
        bw = sorc.walk(*w, k["c"], k["h"], S, k["da"][:cells], x=x_cells if l == 0 else None, h_in=lay[l - 1]["h"] if l else None,
                       d_hT=d_hT if l == L - 1 else None, dh_in=dh_in)
        res[f"L{l} bwd da records"] = store_coef(k["da"][:cells], bw["da"], bw["da_mag"], True)
        for g in ("dw_hh", "dw_ih", "db"):
            res[f"L{l} bwd {g}"] = dw_coef(k[g], bw[g], bw[g + "_mag"], bw[g + "_sub"], cells * T)
        if l == 1:                       # the sequence left in the workspace: layer 1's d(h^0_t)
            res["L1 bwd d_in"] = dw_coef(r["d_seq"], bw["d_in"], bw["d_in_mag"], 0.0, 4 * C)
        if l:
            d_in_above = bw["d_in"]
        else:
            l2["dx"] = orc.rel_errors(r["dx"], bw["dx"])[1]
    _assert_and_record(res, l2, tag)
