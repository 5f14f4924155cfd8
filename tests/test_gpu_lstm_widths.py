"""The tensor-core LSTM (precision 1) at hidden sizes 96 and 128.

Hidden 32 has its own kernels (lstm_tc.cu, test_gpu_parity.py); 96 and 128 run the width-generic ones (a warp per 16 cells x
32-unit slice of all four gates, h exchanged through shared memory; the backward writes fp16 gate gradients that a separate
tensor-core pass reduces to the weight gradients).  Hidden 64 stays on the fp32 kernels.

  * CPU: the float64 oracle against fixtures of the unmodified reference (`tests/golden/lstmw_*`, `mpgcnw_*`,
    tools/gen_golden_wide_lstm.py); the support matrix and the saved-state sizes.
  * GPU: the LSTM against the fixtures and against float64 (ragged cell counts, T = 1 .. 256, tiny / huge gradients, saturated
    gates); the two backward flavours; the whole model at hidden 128; an LSTM row slab as the sharded model runs it.

Bounds are those of the hidden-32 path (test_gpu_parity.py): h_T 1e-3, gradients 2e-3.
"""
import numpy as np
import pytest
import torch
from torch import nn

import _shard_nccl_worker as nccl_worker
from conftest import golden_names, load_golden, record_parity
from oracle import mpgcn_oracle as orc

import MPGCN as shim
from mpgcn_b200 import _lib, ops
from tools.gen_golden_wide import params_checksum, wide_model_params
from tools.gen_golden_wide_lstm import lstm_params

FIXTURE_TOL = 2e-5
H_TOL, G_TOL = 1e-3, 2e-3
# whole model in fp16 at hidden 128 against the reference, forward rel_L2: the fp16 BDGCN layers at C = H = 128 reach 2.18e-3 on
# the 8-node fixture by themselves (with the reference's nn.LSTM); the tensor-core LSTM adds < 1e-4 (fp32 layers: 8.1e-5).  The
# BDGCN engine is not changed here; the bound is that layer error plus the LSTM's own 1e-3, rounded up (DESIGN.md section 3).
FP16_MODEL_FWD_TOL = 3.5e-3
MODEL_GRAD_TOL = 5e-3           # whole model, against the oracle on the engine's ReLU masks (as test_gpu_channel_widths.py)
WIDTHS = (96, 128)


def _rel_check(a, ref, tol, what, l2_only=False):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    ref = ref.detach().cpu().numpy() if isinstance(ref, torch.Tensor) else ref
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    assert np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol), f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"
    return linf, l2


def _lstm_fixture_params(g):
    params = lstm_params(int(g["seed"]), int(g["C"]))
    assert abs(float(params_checksum(params)) - float(g["params_checksum"])) < 1e-6, "numpy RNG stream changed: regenerate the fixture"
    return params


def _check_lstm_fixture_grad(a, g, k, tol, what):
    """One LSTM gradient against an `lstmw_` fixture: dw_hh on its stored rows and in norm, the others in full."""
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    if k != "dw_hh":
        return _rel_check(a, g[k], tol, f"{what}/{k}")
    _rel_check(a[g["dw_hh_row_ids"]], g["dw_hh_rows"], tol, f"{what}/dw_hh rows")
    ref = float(g["dw_hh_norm"])
    assert abs(float(np.linalg.norm(a.astype(np.float64))) - ref) <= tol * ref, f"{what}/dw_hh: norm of the whole tensor"


def _model(N, K, hid, seed, dev):
    torch.manual_seed(seed)
    return shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3, num_nodes=N,
                      user_bias=True, activation=nn.ReLU).to(dev)


def _model_params(g):
    hid, K, N = int(g["hidden"]), int(g["K"]), g["x_seq"].shape[2]
    shapes = {k: v.shape for k, v in _model(N, K, hid, 0, "cpu").state_dict().items()}
    params = wide_model_params(int(g["seed"]), shapes)
    assert abs(float(params_checksum(params)) - float(g["params_checksum"])) < 1e-6, "numpy RNG stream changed: regenerate the fixture"
    return params


def _check_model_grads(grads, g, tol, what, l2_only=False):
    """Every gradient of the model fixture: the row-sampled ones on their rows and in norm, the others in full."""
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
def test_wide_lstm_fixtures_exist_and_stay_out_of_the_other_sets():
    lstms, models = golden_names("lstmw_"), golden_names("mpgcnw_")
    assert len(lstms) == 4 and len(models) == 1
    cases = {(int(load_golden(n)["C"]), load_golden(n)["x"].shape[1]) for n in lstms}
    assert cases == {(96, 1), (96, 7), (128, 1), (128, 7)}
    assert all(load_golden(n)["x"].shape[0] % 128 for n in lstms)
    assert int(load_golden(models[0])["hidden"]) == 128
    for prefix in ("lstm_", "mpgcn_", "wide_mpgcn_", "wide_bdgcn_"):
        assert not set(lstms + models) & set(golden_names(prefix))


@pytest.mark.parametrize("name", golden_names("lstmw_"))
def test_oracle_matches_reference_lstm_at_wide_hidden(name):
    g = load_golden(name)
    p = {k: v.astype(np.float64) for k, v in _lstm_fixture_params(g).items()}
    x = g["x"].astype(np.float64)
    hT = orc.lstm_last_forward(x, p["w_ih"], p["w_hh"], p["b_ih"], p["b_hh"])
    _rel_check(hT, g["hT"], FIXTURE_TOL, f"{name}: hT")
    grads = orc.lstm_last_backward(x, p["w_ih"], p["w_hh"], p["b_ih"], p["b_hh"], g["d_hT"].astype(np.float64))
    for a, k in zip(grads, ("dx", "dw_ih", "dw_hh", "db_ih", "db_hh")):
        _check_lstm_fixture_grad(a, g, k, FIXTURE_TOL, name)


@pytest.mark.parametrize("name", golden_names("mpgcnw_"))
def test_oracle_matches_reference_model_at_hidden_128(name):
    g = load_golden(name)
    y, grads = orc.mpgcn_forward_backward(_model_params(g), g["x_seq"], [g["G_static"], (g["G_o"], g["G_d"])], M=2, gcn_num_layers=3,
                                          d_y=g["d_y"])
    _rel_check(y, g["y"], FIXTURE_TOL, f"{name}: y")
    _check_model_grads(grads, g, FIXTURE_TOL, name)


def test_lstm_support_matrix():
    lib = _lib.load()
    for C in (32, 96, 128):
        assert lib.mpgcn_lstm_precision_supported(5, C, 1) == 1
        assert lib.mpgcn_lstm_precision_supported(1, C, 1) == 1 and lib.mpgcn_lstm_precision_supported(256, C, 1) == 1
        assert lib.mpgcn_lstm_precision_supported(0, C, 1) == 0 and lib.mpgcn_lstm_precision_supported(257, C, 1) == 0
    for C in (16, 48, 64, 160, 256):
        assert lib.mpgcn_lstm_precision_supported(5, C, 1) == 0
    # precision 0 (fp32 CUDA-core kernels) is unchanged: any hidden up to 64
    for C, want in ((1, 1), (8, 1), (32, 1), (48, 1), (64, 1), (65, 0), (96, 0), (128, 0)):
        assert lib.mpgcn_lstm_precision_supported(5, C, 0) == want
    assert lib.mpgcn_lstm_precision_supported(0, 32, 0) == 0


def test_lstm_saved_and_workspace_bytes_at_wide_hidden():
    lib = _lib.load()
    B, T, NN = 3, 7, 1000
    for C, tile in ((96, 64), (128, 48)):
        cells = -(-B * NN // tile) * tile
        saved = lib.mpgcn_lstm_saved_bytes(B, T, NN, C, 1)
        assert saved == cells * T * 2 * C * 2                   # c_t | h_t in fp16
        da = cells * T * 4 * C * 2                              # fp16 gate gradients of the reverse walk
        align = lambda n: -(-n // 256) * 256
        assert lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, 1) == 1024 + align(da) + align(saved)
    # hidden 32 keeps its sizes
    assert lib.mpgcn_lstm_saved_bytes(B, T, NN, 32, 1) == -(-B * NN // 128) * T * 128 * 128
    assert lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, 32, 1) == 1024 + lib.mpgcn_lstm_saved_bytes(B, T, NN, 32, 1)


def test_lstm_precision_resolution_at_wide_hidden_and_fp32_length_limit():
    """Which kernel each precision name resolves to above and at hidden 64, and where "auto" leaves the LSTM to nn.LSTM: the
    tensor-core kernels stop at T = 256, the fp32 kernels at the longest sequence their backward's shared-memory stash holds."""
    for C in WIDTHS:
        assert ops.resolve_lstm_precision("fp16", 12, C) == _lib.PREC_FP16_TC
        assert ops.resolve_lstm_precision("auto", 12, C) == _lib.PREC_FP16_TC
        assert ops.lstm_engine_supports("fp16", 12, C) and not ops.lstm_engine_supports("fp32", 12, C)
        with pytest.raises(RuntimeError, match="hidden 32, 96 or 128"):
            ops.resolve_lstm_precision("fp32", 12, C)
    # hidden 64 stays on the fp32 kernels
    assert ops.resolve_lstm_precision("auto", 12, 64) == _lib.PREC_FP32
    with pytest.raises(RuntimeError, match="hidden 32, 96 or 128"):
        ops.resolve_lstm_precision("fp16", 12, 64)
    assert not ops.lstm_engine_supports("fp16", 300, 128)
    # "auto" (the model's default) runs the engine only where a kernel applies: tensor cores at 32 / 96 / 128 with T <= 256, the
    # fp32 kernels up to hidden 64 as long as their backward's shared-memory stash holds T steps (15 at hidden 64, 95 at 48, 224
    # at 32); everywhere else the model keeps nn.LSTM
    for T, C, want in ((12, 32, True), (12, 48, True), (12, 64, True), (12, 96, True), (12, 128, True), (256, 128, True),
                       (300, 128, False), (300, 96, False), (300, 64, False), (15, 64, True), (16, 64, False), (95, 48, True),
                       (96, 48, False), (256, 32, True), (300, 32, False), (12, 80, False), (12, 160, False), (12, 256, False)):
        assert ops.lstm_engine_supports("auto", T, C) == want, (T, C)
        assert ops.lstm_engine_supports(None, T, C) == want or ops.default_precision() != "auto", (T, C)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: the LSTM alone
# ------------------------------------------------------------------------------------------------------------------------------
def _t(a, dev, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev).requires_grad_(grad)


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("lstmw_"))
def test_lstm_matches_reference_fixture_at_wide_hidden(name, cuda_device):
    g = load_golden(name)
    p = _lstm_fixture_params(g)
    S, T, _ = g["x"].shape
    x = _t(np.ascontiguousarray(g["x"][:, :, 0].T)[None], cuda_device, grad=True)        # [1,T,S]
    ws = [_t(p[k], cuda_device, grad=True) for k in ("w_ih", "w_hh", "b_ih", "b_hh")]
    hT = ops.lstm_last(x.view(1, T, S, 1, 1), *ws, precision="fp16")
    hT.backward(_t(g["d_hT"], cuda_device))
    torch.cuda.synchronize()
    _rel_check(hT, g["hT"], H_TOL, f"{name}/fp16/hT")
    for t, k in zip(ws, ("dw_ih", "dw_hh", "db_ih", "db_hh")):
        _check_lstm_fixture_grad(t.grad, g, k, G_TOL, f"{name}/fp16")
    _rel_check(x.grad[0].T, g["dx"][:, :, 0], G_TOL, f"{name}/fp16/dx")


@pytest.mark.gpu
@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("S,T,gmag,xmag", [(1000, 12, 1.0, 8.0), (300, 7, 1e-7, 8.0), (129, 1, 1.0, 8.0), (4097, 3, 1e3, 8.0),
                                            (500, 6, 1.0, 3000.0), (256, 4, 1.0, 0.01), (129, 256, 1.0, 8.0)])
def test_lstm_tensor_path_matches_float64_at_wide_hidden(C, S, T, gmag, xmag, cuda_device):
    """Ragged tile counts, T = 1 and 256, tiny / huge gradient magnitudes, un-normalised (|x| ~ 3000, saturated gates) and tiny
    inputs: the tensor-core LSTM against the float64 oracle."""
    torch.manual_seed(S + T + C)
    lstm = nn.LSTM(1, C, 1, batch_first=True)
    ws0 = [w.detach().clone() for w in (lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0)]
    x0 = torch.rand(2, T, S, 1, 1) * xmag
    d_h = torch.randn(2 * S, C) * gmag
    ws = [w.to(cuda_device).requires_grad_(True) for w in ws0]
    x = x0.to(cuda_device).requires_grad_(True)
    h = ops.lstm_last(x, *ws, precision="fp16")
    h.backward(d_h.to(cuda_device))
    torch.cuda.synchronize()
    # oracle cells: cell (b, s) is row b S + s; sequences [2S, T, 1]
    xs = x0[:, :, :, 0, 0].permute(0, 2, 1).reshape(2 * S, T, 1).double().numpy()
    w64 = [w.double().numpy() for w in ws0]
    hT = orc.lstm_last_forward(xs, *w64)
    dx, dw_ih, dw_hh, db_ih, db_hh = orc.lstm_last_backward(xs, *w64, d_h.double().numpy())
    tag = f"C={C} S={S} T={T} |dh|={gmag:g} |x|={xmag:g}"
    _rel_check(h, hT, H_TOL, f"{tag} hT")
    for a, r, n in zip([w.grad for w in ws], (dw_ih, dw_hh, db_ih, db_hh), ("dw_ih", "dw_hh", "db_ih", "db_hh")):
        _rel_check(a, r, G_TOL, f"{tag} {n}")
    _rel_check(x.grad[:, :, :, 0, 0].permute(0, 2, 1).reshape(2 * S, T, 1), dx, G_TOL, f"{tag} dx")


@pytest.mark.gpu
@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("S,T", [(700, 12), (130, 2), (64, 1)])
def test_lstm_saved_state_backward_agrees_with_rebuild_first_backward_at_wide_hidden(C, S, T, cuda_device):
    """The two C-ABI backward flavours: (a) forward_train keeps c_t/h_t and backward_saved walks them, (b) plain forward +
    backward_ex, which rebuilds that state in its workspace first.  Same hT bits, gradients to 2e-3 (the weight-gradient pass
    flushes with atomics).  A too-small saved buffer or workspace is refused."""
    lib = _lib.load()
    torch.manual_seed(7 * S + T + C)
    B, prec = 2, _lib.PREC_FP16_TC
    lstm = nn.LSTM(1, C, 1, batch_first=True).to(cuda_device)
    ws = [w.detach().contiguous() for w in (lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0)]
    x = (torch.rand(B, T, S, device=cuda_device) * 6).contiguous()
    d_h = torch.randn(B * S, C, device=cuda_device)
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: None if t is None else t.data_ptr()
    h_a, h_b = torch.empty(B * S, C, device=cuda_device), torch.empty(B * S, C, device=cuda_device)
    nsave = lib.mpgcn_lstm_saved_bytes(B, T, S, C, prec)
    saved = torch.empty(nsave, dtype=torch.uint8, device=cuda_device)
    _lib.check(lib.mpgcn_lstm_last_forward_train(p(x), *[p(w) for w in ws], p(h_a), p(saved), nsave, B, T, S, C, prec, st), "fwd_train")
    _lib.check(lib.mpgcn_lstm_last_forward(p(x), *[p(w) for w in ws], p(h_b), B, T, S, C, prec, st), "fwd")
    torch.cuda.synchronize()
    assert torch.equal(h_a, h_b)
    nws = lib.mpgcn_lstm_bwd_workspace_bytes(B, T, S, C, prec)
    outs = []
    for flavour in ("saved", "rebuild"):
        g = [torch.empty_like(w) for w in ws]
        dx = torch.empty_like(x)
        if flavour == "saved":
            wsb = torch.empty(nws - nsave, dtype=torch.uint8, device=cuda_device)
            _lib.check(lib.mpgcn_lstm_last_backward_saved(p(x), *[p(w) for w in ws], p(d_h), *[p(t) for t in g], p(dx), p(saved), nsave,
                                                          p(wsb), wsb.numel(), B, T, S, C, prec, None, st), "bwd_saved")
        else:
            wsb = torch.empty(nws, dtype=torch.uint8, device=cuda_device)
            _lib.check(lib.mpgcn_lstm_last_backward_ex(p(x), *[p(w) for w in ws], p(d_h), *[p(t) for t in g], p(dx), p(wsb), wsb.numel(),
                                                       B, T, S, C, prec, None, st), "bwd_rebuild")
        torch.cuda.synchronize()
        outs.append(g + [dx])
    for a, r, n in zip(outs[0], outs[1], ("dw_ih", "dw_hh", "db_ih", "db_hh", "dx")):
        _rel_check(a, r, G_TOL, f"C={C} S={S} T={T} saved-vs-rebuild {n}")
    rc = lib.mpgcn_lstm_last_forward_train(p(x), *[p(w) for w in ws], p(h_a), p(saved), nsave - 1, B, T, S, C, prec, st)
    assert rc != 0 and b"saved buffer too small" in lib.mpgcn_last_error()
    g = [torch.empty_like(w) for w in ws]
    wsb = torch.empty(1024, dtype=torch.uint8, device=cuda_device)
    rc = lib.mpgcn_lstm_last_backward_saved(p(x), *[p(w) for w in ws], p(d_h), *[p(t) for t in g], None, p(saved), nsave, p(wsb), 1024,
                                            B, T, S, C, prec, None, st)
    assert rc != 0 and b"workspace too small" in lib.mpgcn_last_error()


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: the whole model at hidden 128
# ------------------------------------------------------------------------------------------------------------------------------
def _set_precision(model, prec):
    model.lstm_precision = prec
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = prec


def _forbid_nn_lstm(model):
    """Make any call of the branches' nn.LSTM modules (the fallback) an error: the engine LSTM must run."""
    def boom(*a, **k):
        raise AssertionError("nn.LSTM ran instead of the engine LSTM")
    for branch in model.branch_models:
        branch['temporal'].forward = boom


def _run_fixture_model(g, params, lstm_prec, layer_prec, dev, engine_lstm=True):
    """The fixture's model at the given precisions -> (y, {name: grad}, the oracle's gradients on the engine's ReLU masks)."""
    K, hid = int(g["K"]), int(g["hidden"])
    N = g["x_seq"].shape[2]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    model = _model(N, K, hid, 0, "cpu")
    model.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    model = model.to(dev)
    model.lstm_precision = lstm_prec
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = layer_prec
    if engine_lstm:
        _forbid_nn_lstm(model)
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
    _, grads_m = orc.mpgcn_forward_backward(params, g["x_seq"], [g["G_static"], (g["G_o"], g["G_d"])], M=2, gcn_num_layers=3,
                                            d_y=g["d_y"], masks=caps)
    return y.detach(), {k: p.grad.detach() for k, p in model.named_parameters()}, grads_m


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden_names("mpgcnw_"))
def test_model_at_hidden_128_fp16_matches_reference_fixture(name, cuda_device):
    """The whole model at hidden 128 with the tensor-core LSTM.

    (a) LSTM "fp16", BDGCN layers fp32: the forward within 1e-3 in rel_L2 of the reference (rel_Linf recorded) -- the LSTM's
        own error reaches y undiluted here.
    (b) precision "fp16" on the whole model (no nn.LSTM anywhere): gradients within 5e-3 in rel_L2 of the oracle's on the
        engine's ReLU masks.  Its forward differs from the reference by what the fp16 BDGCN layers alone give at C = H = 128
        on this 8-node fixture: rel_L2 2.18e-3 with the reference's nn.LSTM in front of them (H100), which is recorded.  The
        whole-fp16 forward is held to the fixed FP16_MODEL_FWD_TOL = 3.5e-3 (DESIGN.md section 3), so that a regression of
        the layers or the LSTM cannot hide in a bound that follows a measurement."""
    g = load_golden(name)
    params = _model_params(g)
    y, grads, grads_m = _run_fixture_model(g, params, "fp16", "fp32", cuda_device)
    _rel_check(y, g["y"], H_TOL, f"{name}/lstm fp16, layers fp32/y", l2_only=True)
    for k, v in grads.items():
        _rel_check(v, grads_m[k], MODEL_GRAD_TOL, f"{name}/lstm fp16, layers fp32/grad:{k} (engine masks)", l2_only=True)

    y16, grads16, grads16_m = _run_fixture_model(g, params, "fp16", "fp16", cuda_device)
    for k, v in grads16.items():
        _rel_check(v, grads16_m[k], MODEL_GRAD_TOL, f"{name}/fp16/grad:{k} (engine masks)", l2_only=True)
    y_ref_lstm, _, _ = _run_fixture_model(g, params, "fp32", "fp16", cuda_device, engine_lstm=False)   # nn.LSTM + fp16 layers
    layers_linf, layers_l2 = orc.rel_errors(y_ref_lstm.cpu().numpy(), g["y"])
    record_parity(f"{name}/nn.LSTM, layers fp16/y", layers_linf, layers_l2, None)
    _rel_check(y16, g["y"], FP16_MODEL_FWD_TOL, f"{name}/fp16/y", l2_only=True)


@pytest.mark.gpu
def test_model_at_hidden_128_no_grad_allocates_no_stash_and_graph_rollout_equals_eager(cuda_device):
    """precision "auto" picks the tensor-core LSTM at hidden 128; under torch.no_grad() the model keeps no training state; the
    CUDA-graph rollout equals the eager loop bitwise."""
    from mpgcn_b200 import rollout
    dev = cuda_device
    N, K, B, T, P = 23, 3, 2, 5, 3
    model = _model(N, K, 128, 3, dev)
    _set_precision(model, "auto")
    _forbid_nn_lstm(model)
    G = torch.rand(K, N, N, device=dev) / N
    dyn = (torch.rand(B, K, N, N, device=dev) / N, torch.rand(B, K, N, N, device=dev) / N)
    x = torch.rand(B, T, N, N, 1, device=dev) * 8
    ops.STASH_BYTES.clear()
    with torch.no_grad():
        y0 = model(x_seq=x, G_list=[G, dyn])
    assert sum(ops.STASH_BYTES.values()) == 0, dict(ops.STASH_BYTES)
    y1 = model(x_seq=x, G_list=[G, dyn])
    assert ops.STASH_BYTES["lstm"] > 0 and torch.equal(y0, y1.detach())
    eager = rollout.forecast(model, x, [G, dyn], P, use_cuda_graph=False)
    graphed = rollout.forecast(model, x, [G, dyn], P, use_cuda_graph=True)
    assert tuple(graphed.shape) == (B, P, N, N, 1)
    assert torch.equal(eager, graphed)


@pytest.mark.gpu
@pytest.mark.parametrize("hid,T,prec,engine", [(96, 4, "fp32", False), (160, 4, None, False), (256, 4, "auto", False),
                                              (128, 300, None, False), (128, 300, "auto", False), (128, 4, None, True),
                                              (96, 256, "auto", True), (64, 16, "auto", False), (64, 15, "auto", True)])
def test_model_lstm_dispatch_above_hidden_64(hid, T, prec, engine, cuda_device, monkeypatch):
    """Above hidden 64 the model runs the engine LSTM only where a kernel applies (tensor cores at 96 / 128, T <= 256) and keeps
    nn.LSTM everywhere else -- lstm_precision "fp32", other widths, longer sequences -- including under the default precision.
    At hidden 64 "auto" keeps nn.LSTM past the 15 steps the fp32 backward can hold."""
    monkeypatch.delenv("MPGCN_B200_PRECISION", raising=False)
    N = 5
    model = _model(N, 2, hid, 5, cuda_device)
    model.lstm_precision = prec
    calls = []
    for branch in model.branch_models:
        branch['temporal'].register_forward_hook(lambda *a: calls.append(1))
    x = torch.rand(2, T, N, N, 1, device=cuda_device) * 8
    G = torch.rand(2, N, N, device=cuda_device) / N
    y = model(x_seq=x, G_list=[G, (G[None].expand(2, -1, -1, -1).contiguous(),) * 2])
    torch.cuda.synchronize()
    assert bool(calls) == (not engine) and torch.isfinite(y).all()


@pytest.mark.gpu
@pytest.mark.parametrize("C", WIDTHS)
def test_lstm_row_slab_equals_the_whole_model_rows(C, cuda_device):
    """The sharded model runs the engine LSTM on its rank's origin rows (shard.sharded_forward, x_seq[:, :, lo:hi]): at the wide
    widths that slab gives the same bits as the same rows of the whole LSTM."""
    torch.manual_seed(C)
    B, T, N, lo, hi = 2, 5, 37, 11, 30
    lstm = nn.LSTM(1, C, 1, batch_first=True).to(cuda_device)
    ws = (lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0)
    x = torch.rand(B, T, N, N, 1, device=cuda_device) * 8
    whole = ops.lstm_last(x, *ws, precision="fp16").reshape(B, N, N, C)
    slab = ops.lstm_last(x[:, :, lo:hi].contiguous(), *ws, precision="fp16").reshape(B, hi - lo, N, C)
    assert torch.equal(slab, whole[:, lo:hi])


@pytest.mark.gpu
@pytest.mark.parametrize("hid,world", [(128, 1), (96, 1), (128, 2)])
def test_row_sharded_model_at_wide_hidden(hid, world, tmp_path):
    """shard.sharded_forward (row shard, NCCL, one rank per GPU) at hidden 96 / 128, whose LSTM is the engine's tensor-core kernel
    on the rank's origin rows, against the whole model at the same precisions: fp32 layers <= 1e-5 forward (2e-3 rel_L2
    gradients), fp16 layers <= 1e-3 forward (8e-2 gradients: another forward's ReLU masks), as tests/test_gpu_shard.py at 32.
    World 1 runs the whole sharded path (plan, slabs, collectives, gradient reduction) on one GPU; world 2 needs two."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    # the LSTM on the tensor-core kernel at both layer precisions; the whole model at the same precisions is the yardstick:
    # fp32 layers -> summation order only; fp16 layers -> the fp16 row partials against the fp16 whole layer
    res = nccl_worker.run(world, tmp_path, [dict(N=66, hidden=hid, dynamic="diffusion", yardstick="same",
                                                 cases=[("fp16", "fp32", 1e-5, 2e-3), ("fp16", "fp16", 1e-3, 8e-2)])])
    assert len(res["rows"]) == 2 * world * (1 + len(_model(5, 3, hid, 0, "cpu").state_dict()))
    for row in res["rows"]:
        record_parity(row["what"], row["linf"], row["l2"], row["tol"])
        assert row["err"] <= row["tol"], row
