"""Parity tests proper (run on an H100: `pytest -m gpu`).  Every call goes through the C ABI.

Tolerances (written here once):
  * precision "fp32" (CUDA-core kernels): rel_Linf, rel_L2 <= 5e-5 vs the reference fixtures
    (fp32 summation-order noise only);
  * precision "fp16" (tensor cores, fp16 operands / fp32 accumulation): forward <= 1e-3 -- the bound
    BASELINE.json's north_star states ("within 1e-3 relative fp32").  Gradients: <= 2e-3 against the
    oracle's gradient evaluated with the ENGINE's ReLU mask (the gradient of the function actually
    computed), and <= 8e-2 against the reference's own gradient: a reduced-precision forward flips
    the sign of the ~3e-4 fraction of pre-activations that lie within its rounding error of zero,
    and each flip moves one d_pre element by O(|d_out|), i.e. rel_L2 ~ sqrt(flipped/active) ~ 2-3 %
    for an i.i.d. d_out (measured 1.3-4.3e-2).  No implementation below fp32 can avoid that.
"""
import numpy as np
import pytest
import torch
from torch import nn

from conftest import golden_names, load_golden, record_parity
from oracle import mpgcn_oracle as orc
from oracle.gen_golden import layer_fixture

import MPGCN as shim
from mpgcn_b200 import _lib, ops

pytestmark = pytest.mark.gpu

TOL = {"fp32": (5e-5, 5e-5), "fp16": (1e-3, 2e-3)}
LOOSE_FP16_GRAD = 8e-2

import abi


def _check(a, ref, tol, what, l2_only=False):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    linf, l2 = orc.rel_errors(a, ref)
    record_parity(what, linf, l2, tol)
    ok = np.isfinite(linf) and l2 <= tol and (l2_only or linf <= tol)
    assert ok, f"{what}: rel_Linf={linf:.3e} rel_L2={l2:.3e} > {tol}"
    return linf, l2


def _t(a, dev, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev).requires_grad_(grad)


def _precisions(C, H, K):
    return ["fp32", "fp16"] if (C == 32 and H == 32 and K <= 8) else ["fp32"]


def test_library_is_the_cuda_one(cuda_device):
    lib = _lib.load()
    assert lib.mpgcn_abi_version() == _lib.ABI_VERSION == 4
    assert torch.cuda.get_device_capability(cuda_device) == (9, 0), "tests expect a Hopper (sm_90) device"


@pytest.mark.parametrize("name", golden_names("bdgcn_"))
def test_bdgcn_layer_matches_reference_fixture(name, cuda_device):
    g = layer_fixture(load_golden(name))
    K = int(g["K"])
    C, H = g["X"].shape[-1], g["W"].shape[1]
    act = nn.ReLU if str(g["act"]) == "relu" else None
    for prec in _precisions(C, H, K):
        layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=H, use_bias="b" in g, activation=act).to(cuda_device)
        layer.precision = prec
        with torch.no_grad():
            layer.W.copy_(_t(g["W"], cuda_device))
            if "b" in g:
                layer.b.copy_(_t(g["b"], cuda_device))
        X = _t(g["X"], cuda_device, grad=True)
        G = (_t(g["G_o"], cuda_device), _t(g["G_d"], cuda_device)) if int(g["dynamic"]) else _t(g["G"], cuda_device)
        out = layer(X, G)
        out.backward(_t(g["d_out"], cuda_device))
        torch.cuda.synchronize()
        tf, tb = TOL[prec]
        _check(out, g["out"], tf, f"{name}/{prec}/out")
        if prec == "fp32" or act is None:
            refs = (g["dX"], g["dW"], g.get("db"))
        else:   # gradient of the computed function: oracle backward with the engine's ReLU mask
            Gn = (g["G_o"], g["G_d"]) if int(g["dynamic"]) else g["G"]
            refs = orc.bdgcn_backward(g["X"], Gn, g["W"], g.get("b"), "relu", g["d_out"], mask_from=out.detach().cpu().numpy())
            _check(X.grad, g["dX"], LOOSE_FP16_GRAD, f"{name}/{prec}/dX vs reference", l2_only=True)   # a flipped mask element is an O(1) local change
            _check(layer.W.grad, g["dW"], LOOSE_FP16_GRAD, f"{name}/{prec}/dW vs reference", l2_only=True)
        _check(X.grad, refs[0], tb, f"{name}/{prec}/dX")
        _check(layer.W.grad, refs[1], tb, f"{name}/{prec}/dW")
        if "b" in g:
            _check(layer.b.grad, refs[2], tb, f"{name}/{prec}/db")


@pytest.mark.parametrize("name", golden_names("lstm_"))
def test_lstm_last_matches_reference_fixture(name, cuda_device):
    g = load_golden(name)
    S, T, _ = g["x"].shape
    # the kernel reads x_seq as [B,T,NN]; fixture sequences are [S,T,1] -> one batch element, NN = S
    x = _t(np.ascontiguousarray(g["x"][:, :, 0].T)[None], cuda_device, grad=True)        # [1,T,S]
    ws = [_t(g[k], cuda_device, grad=True) for k in ("w_ih", "w_hh", "b_ih", "b_hh")]
    C = g["w_hh"].shape[1]
    for prec in (["fp32", "fp16"] if C == 32 else ["fp32"]):
        for t in [x] + ws:
            t.grad = None
        hT = ops.lstm_last(x.view(1, T, S, 1, 1), *ws, precision=prec)
        hT.backward(_t(g["d_hT"], cuda_device))
        torch.cuda.synchronize()
        # fp32 kernels: SFU exp/rcp noise only.  tensor-core path: recurrent h (and the stashed gates in backward) in fp16.
        tf, tb = (1e-4, 2e-4) if prec == "fp32" else (1e-3, 2e-3)
        _check(hT, g["hT"], tf, f"{prec}/hT")
        for t, k in zip(ws, ("dw_ih", "dw_hh", "db_ih", "db_hh")):
            _check(t.grad, g[k], tb, f"{prec}/{k}")
        _check(x.grad[0].T, g["dx"][:, :, 0], tb, f"{prec}/dx")


@pytest.mark.parametrize("S,T,gmag,xmag", [(1000, 12, 1.0, 8.0), (300, 7, 1e-7, 8.0), (129, 1, 1.0, 8.0), (4097, 3, 1e3, 8.0),
                                            (500, 6, 1.0, 3000.0), (256, 4, 1.0, 0.01)])
def test_lstm_tensor_path_agrees_with_fp32_path(S, T, gmag, xmag, cuda_device):
    """Ragged tile counts, T = 1, tiny / huge gradient magnitudes, un-normalised (|x| ~ 3000, saturated gates) and tiny
    inputs (x rides in the gate MMA as an fp16 hi + lo pair): tensor-core LSTM vs the fp32 CUDA-core LSTM."""
    torch.manual_seed(S + T)
    lstm = nn.LSTM(1, 32, 1, batch_first=True).to(cuda_device)
    ws0 = [lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0]
    x0 = torch.rand(2, T, S, 1, 1, device=cuda_device) * xmag
    d_h = torch.randn(2 * S, 32, device=cuda_device) * gmag
    res = {}
    for prec in ("fp32", "fp16"):
        ws = [w.detach().clone().requires_grad_(True) for w in ws0]
        x = x0.clone().requires_grad_(True)
        h = ops.lstm_last(x, *ws, precision=prec)
        h.backward(d_h)
        res[prec] = [h.detach()] + [w.grad for w in ws] + [x.grad]
    names = ("hT", "dw_ih", "dw_hh", "db_ih", "db_hh", "dx")
    for a, r, n in zip(res["fp16"], res["fp32"], names):
        _check(a, r.cpu().numpy(), 1e-3 if n == "hT" else 2e-3, f"S={S} T={T} {n}")


@pytest.mark.parametrize("S,T", [(700, 12), (130, 2), (64, 1)])
def test_lstm_saved_state_backward_agrees_with_recompute_backward(S, T, cuda_device):
    """The two C-ABI backward flavours of the tensor-core LSTM: (a) forward_train keeps c_t/h_t and backward_saved walks them,
    (b) plain forward + backward_ex, which rebuilds that state in its workspace first.  Same hT bits, same gradients (up to
    the order of the atomic weight-gradient flush)."""
    from mpgcn_b200 import _lib
    lib = _lib.load()
    torch.manual_seed(7 * S + T)
    B, C, prec = 2, 32, _lib.PREC_FP16_TC
    lstm = nn.LSTM(1, C, 1, batch_first=True).to(cuda_device)
    ws = [w.detach().contiguous() for w in (lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0)]
    x = (torch.rand(B, T, S, device=cuda_device) * 6).contiguous()
    d_h = torch.randn(B * S, C, device=cuda_device)
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: None if t is None else t.data_ptr()
    h_a, h_b = torch.empty(B * S, C, device=cuda_device), torch.empty(B * S, C, device=cuda_device)
    nsave = lib.mpgcn_lstm_saved_bytes(B, T, S, C, prec)
    assert nsave == ((B * S + 127) // 128) * T * 128 * 128
    saved = torch.empty(nsave, dtype=torch.uint8, device=cuda_device)
    _lib.check(lib.mpgcn_lstm_last_forward_train(p(x), *[p(w) for w in ws], p(h_a), p(saved), nsave, B, T, S, C, prec, st), "fwd_train")
    _lib.check(lib.mpgcn_lstm_last_forward(p(x), *[p(w) for w in ws], p(h_b), B, T, S, C, prec, st), "fwd")
    assert torch.equal(h_a, h_b)
    outs = []
    for flavour in ("saved", "recompute"):
        g = [torch.empty_like(w) for w in ws]
        dx = torch.empty_like(x)
        if flavour == "saved":
            wsb = torch.empty(1024, dtype=torch.uint8, device=cuda_device)
            _lib.check(lib.mpgcn_lstm_last_backward_saved(p(x), *[p(w) for w in ws], p(d_h), *[p(t) for t in g], p(dx), p(saved), nsave,
                                                          p(wsb), wsb.numel(), B, T, S, C, prec, None, st), "bwd_saved")
        else:
            wsb = torch.empty(lib.mpgcn_lstm_bwd_workspace_bytes(B, T, S, C, prec), dtype=torch.uint8, device=cuda_device)
            _lib.check(lib.mpgcn_lstm_last_backward_ex(p(x), *[p(w) for w in ws], p(d_h), *[p(t) for t in g], p(dx), p(wsb), wsb.numel(),
                                                       B, T, S, C, prec, None, st), "bwd_recompute")
        torch.cuda.synchronize()
        outs.append(g + [dx])
    for a, r, n in zip(outs[0], outs[1], ("dw_ih", "dw_hh", "db_ih", "db_hh", "dx")):
        _check(a, r.cpu().numpy(), 2e-3, f"S={S} T={T} saved-vs-recompute {n}")
    # a too-small saved buffer is refused
    rc = lib.mpgcn_lstm_last_forward_train(p(x), *[p(w) for w in ws], p(h_a), p(saved), nsave - 1, B, T, S, C, prec, st)
    assert rc != 0 and b"saved buffer too small" in lib.mpgcn_last_error()


@pytest.mark.parametrize("name", golden_names("adj_"))
def test_adj_processor_matches_reference_fixture(name, cuda_device):
    """GPU support-matrix builder vs fixtures produced by the reference's Adj_Processor (fp32: summation-order noise only)."""
    import GCN as gshim
    g = load_golden(name)
    proc = gshim.Adj_Processor(str(g["kernel_type"]), int(g["K"]))
    sup = proc.process(torch.from_numpy(g["flow"]))                 # CPU tensor in, as the trainer passes it
    assert sup.is_cuda and tuple(sup.shape) == g["supports"].shape
    _check(sup, g["supports"], 2e-5, f"{name}/supports")
    _check(proc.process(torch.from_numpy(g["flow"]).to(cuda_device)), g["supports"], 2e-5, f"{name}/supports (cuda in)")


@pytest.mark.parametrize("kind,K,N,B", [("random_walk_diffusion", 2, 500, 3), ("chebyshev", 3, 257, 2), ("dual_random_walk_diffusion", 2, 130, 2)])
def test_adj_processor_at_size_vs_oracle(kind, K, N, B, cuda_device):
    import GCN as gshim
    rng = np.random.default_rng(N)
    flow = (rng.random((B, N, N)) * 5).astype(np.float32)
    sup = gshim.Adj_Processor(kind, K).process(_t(flow, cuda_device))
    _check(sup, orc.adj_process(flow.astype(np.float64), kind, K), 2e-5, f"adj {kind} N={N}")


@pytest.mark.parametrize("name", golden_names("dyn_"))
def test_dyn_graphs_match_reference_fixture(name, cuda_device):
    """GPU construct_dyn_G vs fixtures produced by the reference's DataInput.construct_dyn_G (float64, per-pair scipy calls):
    fp32 arithmetic on the device -> 5e-6 absolute; identical NaN pattern (zero vectors)."""
    from mpgcn_b200 import dyn_graph
    g = load_golden(name)
    O, D = dyn_graph.construct_dyn_G(g["od"], list(g["split_ratio"]), device=cuda_device)
    for a, ref, what in ((O, g["O_dyn_G"], "O"), (D, g["D_dyn_G"], "D")):
        assert a.shape == ref.shape and a.dtype == np.float64
        assert np.array_equal(np.isnan(a), np.isnan(ref)), f"{name}/{what}: NaN pattern"
        err = float(np.nanmax(np.abs(a - ref)))
        record_parity(f"{name}/{what} (abs)", err, err, 5e-6)
        assert err <= 5e-6, f"{name}/{what}: max abs err {err:.2e}"


def test_dyn_graphs_at_size_and_drop_in_method(cuda_device):
    """N = 300 (1.26 M scipy calls in the reference) against the float64 oracle, through the drop-in replacement of the
    reference's method (same signature: self, OD_data, perceived_period=7)."""
    from mpgcn_b200 import dyn_graph
    rng = np.random.default_rng(11)
    N, days = 300, 64
    od = rng.poisson(3.0, size=(days, N, N, 1)).astype(np.float32)
    class DataInput:                      # the reference class's relevant surface (Data_Container_OD.py:10-12,39)
        def __init__(self, params):
            self.params = params
    dyn_graph.install(DataInput)
    O, D = DataInput({"split_ratio": [6.4, 1.6, 2]}).construct_dyn_G(od)
    Oref, Dref = orc.construct_dyn_g(od.astype(np.float64), [6.4, 1.6, 2])
    assert O.shape == (N, N, 7) and D.shape == (N, N, 7)
    for a, ref, what in ((O, Oref, "O"), (D, Dref, "D")):
        err = float(np.max(np.abs(a - ref)))
        record_parity(f"dyn N={N}/{what} (abs)", err, err, 5e-6)
        assert err <= 5e-6, f"{what}: max abs err {err:.2e}"


@pytest.mark.parametrize("M,C,cells", [(2, 32, 1000), (1, 8, 77), (3, 64, 4099)])
def test_fused_head_matches_oracle(M, C, cells, cuda_device):
    """Linear(C->1)+ReLU per branch and branch mean in one kernel (reference MPGCN.py:74-76,107,110) vs the numpy oracle."""
    rng = np.random.default_rng(M * 100 + C)
    gs = [rng.standard_normal((cells, C)).astype(np.float32) for _ in range(M)]
    w = (rng.standard_normal((M, C)) / C ** 0.5).astype(np.float32)
    b = (rng.standard_normal(M) * 0.1).astype(np.float32)
    dy = rng.standard_normal((cells, 1)).astype(np.float32)
    gt = [_t(g, cuda_device, grad=True) for g in gs]
    wt, bt = _t(w, cuda_device, grad=True), _t(b, cuda_device, grad=True)
    y = ops.fc_relu_mean(gt, wt, bt)
    y.backward(_t(dy, cuda_device))
    outs = [orc.fc_relu_forward(gs[m], w[m:m + 1], b[m:m + 1]) for m in range(M)]
    _check(y, np.mean(np.stack(outs, -1), -1), 1e-5, "head y")
    for m in range(M):
        dg, dw, db = orc.fc_relu_backward(gs[m], w[m:m + 1], b[m:m + 1], dy / M)
        _check(gt[m].grad, dg, 1e-5, f"head dg{m}")
        _check(wt.grad[m:m + 1], dw, 1e-4, f"head dw{m}")
        _check(bt.grad[m:m + 1], db, 1e-4, f"head db{m}")


@pytest.mark.parametrize("name", golden_names("mpgcn_"))
def test_full_model_matches_reference_fixture(name, cuda_device):
    g = load_golden(name)
    K, hid = int(g["K"]), int(g["hidden"])
    N = g["x_seq"].shape[2]
    params = {k[6:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("param:")}
    for prec in _precisions(hid, hid, K):
        model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                           num_nodes=N, user_bias=True, activation=nn.ReLU)
        model.load_state_dict(params)                       # a reference checkpoint, loaded unchanged
        model = model.to(cuda_device)
        model.lstm_precision = prec
        for mod in model.modules():
            if isinstance(mod, shim.BDGCN):
                mod.precision = prec
        G_list = [_t(g["G_static"], cuda_device), (_t(g["G_o"], cuda_device), _t(g["G_d"], cuda_device))]
        # capture every ReLU output of the engine (3 BDGCN layers + FC head per branch) for the mask-aware oracle gradient
        caps = {m: {"layers": [], "fc": None} for m in range(2)}
        hooks = []
        for m in range(2):
            for layer in model.branch_models[m]['spatial']:
                hooks.append(layer.register_forward_hook(lambda mod, inp, out, m=m: caps[m]["layers"].append(out.detach().cpu().numpy())))
        y = model(x_seq=_t(g["x_seq"], cuda_device), G_list=G_list)     # keyword call, as Model_Trainer.py:107
        y.backward(_t(g["d_y"], cuda_device))
        torch.cuda.synchronize()
        for h in hooks:
            h.remove()
        for m in range(2):     # the fused head never materialises the per-branch FC output; rebuild its ReLU mask from the last layer
            fc = model.branch_models[m]['fc'][0]
            caps[m]["fc"] = orc.fc_relu_forward(caps[m]["layers"][-1], fc.weight.detach().cpu().numpy(), fc.bias.detach().cpu().numpy())
        tf, tb = TOL[prec]
        _check(y, g["y"], tf, f"{name}/{prec}/y")
        if prec == "fp32":
            for k, p in model.named_parameters():
                _check(p.grad, g["grad:" + k], 2e-4, f"{name}/{prec}/grad:{k}")     # summation-order noise only
        else:
            # gradient of the function actually computed: oracle backward with the engine's ReLU masks
            params_np = {k[6:]: v for k, v in g.items() if k.startswith("param:")}
            _, grads_m = orc.mpgcn_forward_backward(params_np, g["x_seq"], [g["G_static"], (g["G_o"], g["G_d"])], M=2, gcn_num_layers=3,
                                                    d_y=g["d_y"], masks=caps)
            for k, p in model.named_parameters():
                _check(p.grad, grads_m[k], 5e-3, f"{name}/{prec}/grad:{k} (engine masks)", l2_only=True)


@pytest.mark.parametrize("N,K,B,dyn,gmag", [(200, 3, 2, False, 1.0), (130, 6, 1, True, 1e-7), (257, 2, 1, False, 3e4)])
def test_tensor_path_agrees_with_fp32_path_at_size(N, K, B, dyn, gmag, cuda_device):
    """Sizes the CPU oracle cannot finish in seconds: the fp16 tensor-core path against our exact fp32 path."""
    torch.manual_seed(N + K)
    X = torch.tanh(torch.randn(B, N, N, 32, device=cuda_device))
    if dyn:
        G = (torch.randn(B, K, N, N, device=cuda_device) / N ** 0.5, torch.randn(B, K, N, N, device=cuda_device) / N ** 0.5)
    else:
        G = torch.randn(K, N, N, device=cuda_device) / N ** 0.5
    W = torch.randn(K * K * 32, 32, device=cuda_device) * (2.0 / (K * K * 32 + 32)) ** 0.5
    b = torch.randn(32, device=cuda_device) * 0.1
    d_out = torch.randn(B, N, N, 32, device=cuda_device) * gmag     # realistic (tiny) and huge gradient magnitudes: fp16 range
    Go, Gd = (G if dyn else (G, G))
    out16, saved16 = abi.forward(X, Go, Gd, W, b, True, "fp16")
    out32, saved32 = abi.forward(X, Go, Gd, W, b, True, "fp32")
    _check(out16, out32.cpu().numpy(), 1e-3, f"N={N} K={K} out")
    g16 = abi.backward(d_out, out16, Go, Gd, W, True, saved16, "fp16")
    g32 = abi.backward(d_out, out16, Go, Gd, W, True, saved32, "fp32")      # same ReLU mask (out16) on both paths
    for a, r, what in zip(g16, g32, ("dX", "dW", "db")):
        _check(a, r.cpu().numpy(), 2e-3, f"N={N} K={K} {what}")
    flipped = float(((out16 > 0) != (out32 > 0)).float().mean())
    assert flipped < 2e-3, f"ReLU mask flips {flipped:.2e}"


@pytest.mark.parametrize("N,K,B,dyn", [(500, 3, 2, True), (1000, 6, 1, False), (2000, 3, 1, False)])
def test_baseline_config_sizes_forward_and_backward(N, K, B, dyn, cuda_device):
    """BASELINE.json configs[2..4] shapes (N=500/K=3, N=1000/K=6, N=2000/K=3; batch reduced to keep the fp32 cross-check
    short): fp16 tensor-core path (ragged 128-row tiles) vs our exact fp32 path, forward and backward."""
    torch.manual_seed(N)
    X = torch.tanh(torch.randn(B, N, N, 32, device=cuda_device))
    if dyn:
        Go = torch.randn(B, K, N, N, device=cuda_device) / N ** 0.5
        Gd = torch.randn(B, K, N, N, device=cuda_device) / N ** 0.5
    else:
        Go = Gd = torch.randn(K, N, N, device=cuda_device) / N ** 0.5
    W = torch.randn(K * K * 32, 32, device=cuda_device) * (2.0 / (K * K * 32 + 32)) ** 0.5
    b = torch.randn(32, device=cuda_device) * 0.1
    d_out = torch.randn(B, N, N, 32, device=cuda_device) * 1e-6
    out16, saved16 = abi.forward(X, Go, Gd, W, b, True, "fp16")
    out32, saved32 = abi.forward(X, Go, Gd, W, b, True, "fp32")
    _check(out16, out32.cpu().numpy(), 1e-3, f"cfg N={N} K={K} out")
    g16 = abi.backward(d_out, out16, Go, Gd, W, True, saved16, "fp16")
    del saved16
    g32 = abi.backward(d_out, out16, Go, Gd, W, True, saved32, "fp32")
    for a, r, what in zip(g16, g32, ("dX", "dW", "db")):
        _check(a, r.cpu().numpy(), 2e-3, f"cfg N={N} K={K} {what}")


@pytest.mark.parametrize("N,K,T,B", [(200, 3, 8, 4), (500, 3, 12, 1)])
def test_full_model_at_baseline_config_shapes(N, K, T, B, cuda_device):
    """BASELINE.json configs[1] / [2] model shapes (N=200,K=3,T=8 and N=500,K=3,T=12; batch reduced): the whole MPGCN forward +
    backward (LSTM -> 3 x BDGCN -> fused head, two branches, static + dynamic supports) on the tensor-core kernels against
    the same model on the exact fp32 kernels.  Forward within 1e-3; parameter gradients see the ReLU-mask flips of a
    reduced-precision forward (DESIGN.md section 3), hence the rel_L2 bound."""
    torch.manual_seed(N + T)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=32, lstm_num_layers=1, gcn_hidden_dim=32, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    x = torch.rand(B, T, N, N, 1, device=cuda_device) * 4
    G = torch.randn(K, N, N, device=cuda_device) / N ** 0.5
    dyn = (torch.randn(B, K, N, N, device=cuda_device) / N ** 0.5, torch.randn(B, K, N, N, device=cuda_device) / N ** 0.5)
    res = {}
    for prec in ("fp32", "fp16"):
        model.lstm_precision = prec
        for mod in model.modules():
            if isinstance(mod, shim.BDGCN):
                mod.precision = prec
        model.zero_grad(set_to_none=True)
        y = model(x_seq=x, G_list=[G, dyn])
        # the trainer's loss (nn.MSELoss, Model_Trainer.py:64,108) against a zero target: a coherent d_y.  (An i.i.d. random d_y
        # makes every parameter gradient a noise-dominated sum of random-sign terms, in which the ~3e-4 ReLU-mask flips of the
        # reduced-precision forward show up as 10 % relative differences.)
        loss = (y ** 2).mean()
        loss.backward()
        torch.cuda.synchronize()
        res[prec] = (y.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters()})
    _check(res["fp16"][0], res["fp32"][0].cpu().numpy(), 1e-3, f"model N={N} K={K} T={T} y")
    for k, gref in res["fp32"][1].items():
        _check(res["fp16"][1][k], gref.cpu().numpy(), 8e-2, f"model N={N} grad:{k}", l2_only=True)


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_size_independent_properties(prec, cuda_device):
    """Linearity in X (no activation), identity supports, static == broadcast dynamic; N = 300."""
    N, K, B = 300, 3, 2
    torch.manual_seed(5)
    layer = shim.BDGCN(K=K, input_dim=32, hidden_dim=32, use_bias=False, activation=None).to(cuda_device)
    layer.precision = prec
    G = torch.randn(K, N, N, device=cuda_device) / N ** 0.5
    X1 = torch.tanh(torch.randn(B, N, N, 32, device=cuda_device))
    X2 = torch.tanh(torch.randn(B, N, N, 32, device=cuda_device))
    tol = 5e-5 if prec == "fp32" else 1.5e-3
    with torch.no_grad():
        lhs = layer(2.0 * X1 - 0.5 * X2, G)
        rhs = 2.0 * layer(X1, G) - 0.5 * layer(X2, G)
        _check(lhs, rhs.cpu().numpy(), tol, "linearity")
        eye = torch.eye(N, device=cuda_device).expand(K, N, N).contiguous()
        W_sum = layer.W.view(K, K, 32, 32).sum(dim=(0, 1))
        _check(layer(X1, eye), (X1 @ W_sum).cpu().numpy(), tol, "identity supports")
        Gb = G.expand(B, K, N, N).contiguous()
        _check(layer(X1, (Gb, Gb)), layer(X1, G).cpu().numpy(), 1e-6, "static == dynamic broadcast")


def test_inference_mode_needs_no_stash_and_trainer_call_pattern(cuda_device):
    """Mimics Model_Trainer.train/test call patterns (Model_Trainer.py:98-115,159-164): train step with Adam,
    eval under no_grad with an autoregressive roll, state_dict round trip."""
    torch.manual_seed(1)
    N, K, B, T = 20, 3, 2, 5
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=32, lstm_num_layers=1, gcn_hidden_dim=32, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    crit = nn.MSELoss()
    # supports exactly as the trainer builds them (Model_Trainer.py:38-42,82-84,106): static graph once, dynamic O/D graphs per
    # step from CPU tensors, through the drop-in GCN.Adj_Processor
    import GCN as gshim
    adj_pre = gshim.Adj_Processor("random_walk_diffusion", K - 1)
    G = adj_pre.process(torch.rand(1, N, N)).squeeze(dim=0).to(cuda_device)
    dyn = (adj_pre.process(torch.rand(B, N, N)).to(cuda_device), adj_pre.process(torch.rand(B, N, N)).to(cuda_device))
    assert tuple(G.shape) == (K, N, N) and tuple(dyn[0].shape) == (B, K, N, N)
    x = torch.rand(B, T, N, N, 1, device=cuda_device) * 8
    y_true = torch.rand(B, 1, N, N, 1, device=cuda_device)
    losses = []
    model.train()
    for _ in range(5):
        with torch.set_grad_enabled(True):
            loss = crit(model(x_seq=x, G_list=[G, dyn]), y_true)
            opt.zero_grad()
            loss.backward()
            opt.step()
        losses.append(float(loss.detach()))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]
    model.eval()
    with torch.no_grad():
        cur = x
        for _ in range(3):
            step = model(x_seq=cur, G_list=[G, dyn])
            assert tuple(step.shape) == (B, 1, N, N, 1)
            cur = torch.cat([cur[:, 1:], step], dim=1)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    model2 = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=32, lstm_num_layers=1, gcn_hidden_dim=32, gcn_num_layers=3,
                        num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    model2.load_state_dict(sd)
    with torch.no_grad():
        assert torch.equal(model2(x_seq=x, G_list=[G, dyn]), model(x_seq=x, G_list=[G, dyn]))


def test_layer_extras_prepared_supports_and_f16_copies(cuda_device):
    """mpgcn_bdgcn_forward_x / _backward_x: supports prepared once, an fp16 copy of X handed in, an fp16 copy of `out` handed
    out and used for the ReLU mask -- same results as the plain entry points (bit-identical forward)."""
    import ctypes
    lib = _lib.load()
    torch.manual_seed(21)
    B, N, K = 2, 70, 3
    X = torch.tanh(torch.randn(B, N, N, 32, device=cuda_device))
    Go = torch.randn(B, K, N, N, device=cuda_device) / N ** 0.5
    Gd = torch.randn(B, K, N, N, device=cuda_device) / N ** 0.5
    Gd[:, 1] += 3 * torch.eye(N, device=cuda_device)          # a diagonally dominant support: the remainder correction is active
    W = torch.randn(K * K * 32, 32, device=cuda_device) * 0.05
    b = torch.randn(32, device=cuda_device) * 0.1
    d_out = torch.randn(B, N, N, 32, device=cuda_device) * 1e-4
    out_ref, saved_ref = abi.forward(X, Go, Gd, W, b, True, "fp16")
    g_ref = abi.backward(d_out, out_ref, Go, Gd, W, True, saved_ref, "fp16")
    st = torch.cuda.current_stream().cuda_stream
    prec = _lib.PREC_FP16_TC
    preps = []
    for G in (Go, Gd):
        nb = lib.mpgcn_bdgcn_supports_prepared_bytes(B * K, N)
        blob = torch.empty(nb, dtype=torch.uint8, device=cuda_device)
        _lib.check(lib.mpgcn_bdgcn_prepare_supports(G.data_ptr(), blob.data_ptr(), nb, B * K, N, st), "prepare")
        preps.append(blob)
    x16 = X.half()
    out = torch.empty_like(out_ref)
    out16 = torch.empty(out.shape, dtype=torch.float16, device=cuda_device)
    saved = torch.empty(lib.mpgcn_bdgcn_saved_bytes(B, N, K, 32, 32, prec), dtype=torch.uint8, device=cuda_device)
    ws = torch.empty(lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, 32, 32, 1, prec), dtype=torch.uint8, device=cuda_device)
    ex = _lib.BdgcnExtras()
    ex.go_prepared, ex.gd_prepared, ex.x_f16, ex.out_f16 = preps[0].data_ptr(), preps[1].data_ptr(), x16.data_ptr(), out16.data_ptr()
    _lib.check(lib.mpgcn_bdgcn_forward_x(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), 1, W.data_ptr(), b.data_ptr(), 1, out.data_ptr(),
                                         saved.data_ptr(), ws.data_ptr(), ws.numel(), B, N, K, 32, 32, prec, ctypes.addressof(ex), st), "fwd_x")
    torch.cuda.synchronize()
    assert torch.equal(out, out_ref)
    assert torch.equal(out16, out_ref.half())
    dX, dW, db = torch.empty_like(X), torch.empty_like(W), torch.empty(32, device=cuda_device)
    wsb = torch.empty(lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, 32, 32, 1, prec), dtype=torch.uint8, device=cuda_device)
    amax = torch.zeros(1, device=cuda_device)
    ex.x_f16, ex.dX_absmax = None, amax.data_ptr()
    _lib.check(lib.mpgcn_bdgcn_backward_x(d_out.data_ptr(), None, Go.data_ptr(), Gd.data_ptr(), 1, W.data_ptr(), 1, saved.data_ptr(),
                                          dX.data_ptr(), dW.data_ptr(), db.data_ptr(), wsb.data_ptr(), wsb.numel(), B, N, K, 32, 32, prec,
                                          ctypes.addressof(ex), st), "bwd_x")
    torch.cuda.synchronize()
    for a, r, what in zip((dX, dW, db), g_ref, ("dX", "dW", "db")):
        _check(a, r.cpu().numpy(), 1e-5, f"extras {what}", l2_only=True)
    assert abs(float(amax) - float(dX.abs().max())) <= 1e-6 * float(dX.abs().max())
    # a misaligned output (the epilogues use 256-bit stores), a too-small prepared buffer and a missing ReLU-mask source are refused
    big = torch.empty(out.numel() + 8, device=cuda_device)
    assert lib.mpgcn_bdgcn_forward(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), 1, W.data_ptr(), b.data_ptr(), 1, big.data_ptr() + 16,
                                   saved.data_ptr(), ws.data_ptr(), ws.numel(), B, N, K, 32, 32, prec, st) != 0
    assert b"32-byte aligned" in lib.mpgcn_last_error()
    assert lib.mpgcn_bdgcn_prepare_supports(Go.data_ptr(), preps[0].data_ptr(), 16, B * K, N, st) != 0
    ex.out_f16 = None
    assert lib.mpgcn_bdgcn_backward_x(d_out.data_ptr(), None, Go.data_ptr(), Gd.data_ptr(), 1, W.data_ptr(), 1, saved.data_ptr(),
                                      dX.data_ptr(), dW.data_ptr(), db.data_ptr(), wsb.data_ptr(), wsb.numel(), B, N, K, 32, 32, prec,
                                      ctypes.addressof(ex), st) != 0


def test_support_cache_tracks_the_support_tensor(cuda_device):
    """ops caches the fp16 staging of a support per tensor object: an in-place update (version bump) or a new tensor must be
    re-staged."""
    torch.manual_seed(8)
    N, K, B = 48, 2, 2
    l1 = shim.BDGCN(K=K, input_dim=32, hidden_dim=32, use_bias=True, activation=nn.ReLU).to(cuda_device)
    l2 = shim.BDGCN(K=K, input_dim=32, hidden_dim=32, use_bias=True, activation=nn.ReLU).to(cuda_device)
    X = torch.tanh(torch.randn(B, N, N, 32, device=cuda_device)).requires_grad_(True)
    G = torch.randn(K, N, N, device=cuda_device) / N ** 0.5
    y1 = l2(l1(X, G), G)
    G.mul_(2.0)                                    # same object, same address, new contents
    y2 = l2(l1(X, G), G)
    y2_fresh = l2(l1(X, G.clone()), G.clone())     # never cached
    assert not torch.allclose(y1, y2)
    assert torch.equal(y2, y2_fresh)
    y2.sum().backward()
    assert torch.isfinite(X.grad).all() and float(X.grad.abs().max()) > 0


def test_gradient_magnitude_hints_follow_the_autograd_graph(cuda_device, monkeypatch):
    """max|grad| hand-over (ops._put_hint / _take_hint): in the model every fp16 backward receives its scale from the kernel
    that wrote its incoming gradient (8 hand-overs: head -> layer 3 -> 2 -> 1 -> LSTM on two branches), results are
    the same with and without the hand-over, and a gradient that is not the producer's own buffer (here: a second
    consumer of the LSTM output, so autograd accumulates) is not trusted."""
    torch.manual_seed(3)
    N, K, B, T = 40, 2, 2, 3
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=32, lstm_num_layers=1, gcn_hidden_dim=32, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    x = torch.rand(B, T, N, N, 1, device=cuda_device) * 4
    G = torch.randn(K, N, N, device=cuda_device) / N ** 0.5
    lib = _lib.load()

    def run():
        model.zero_grad(set_to_none=True)
        lib.mpgcn_profile_reset()
        (model(x_seq=x, G_list=[G, G]) ** 2).mean().backward()
        torch.cuda.synchronize()
        return _lib.profile_read()["ELEMENTWISE"]["launches"], [p.grad.clone() for p in model.parameters()]

    run()                                     # stages the supports once (ops._prepared_supports), outside the counts below
    n_with, g_with = run()
    monkeypatch.setattr(ops, "_put_hint", lambda *a: None)
    n_without, g_without = run()
    monkeypatch.undo()
    assert n_without - n_with == 8, (n_with, n_without)          # one absmax pass saved per hand-over
    for a, b in zip(g_with, g_without):      # same scales either way; only the atomic summation order differs run to run
        _check(a, b.cpu().numpy(), 1e-5, "gradients with vs without the hand-over", l2_only=True)
    # second consumer of h_T: the LSTM node receives an accumulated gradient -> its hint must be rejected, result still right
    lstm = model.branch_models[0]['temporal']
    layer = model.branch_models[0]['spatial'][0]
    ws = [lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0]
    def two_consumers(scale_side):
        for w in ws:
            w.grad = None
        h = ops.lstm_last(x, *ws, precision="fp16")
        out = layer(h.reshape(B, N, N, 32), G)
        (out.sum() * 1e-3 + scale_side * (h ** 2).sum()).backward()
        torch.cuda.synchronize()
        return [w.grad.clone() for w in ws]
    ref = two_consumers(0.0)
    big = two_consumers(50.0)         # the side branch dominates max|grad|: a stale scale would saturate fp16
    assert all(torch.isfinite(g).all() for g in big)
    assert not torch.allclose(big[1], ref[1])
    for w in ws:
        w.grad = None
    h = ops.lstm_last(x, *ws, precision="fp32")
    out = layer(h.reshape(B, N, N, 32), G)
    (out.sum() * 1e-3 + 50.0 * (h ** 2).sum()).backward()
    for a, w in zip(big, ws):
        _check(a, w.grad.cpu().numpy(), 5e-3, "two consumers of h_T: accumulated gradient", l2_only=True)


def test_cuda_graph_rollout_equals_eager_loop(cuda_device):
    """Model_Trainer.test's autoregressive loop (Model_Trainer.py:157-165): CUDA-graph replay vs the eager loop, N = 47."""
    from mpgcn_b200 import rollout
    torch.manual_seed(3)
    N, K, B, T, P = 47, 3, 2, 7, 5
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=32, lstm_num_layers=1, gcn_hidden_dim=32, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU).to(cuda_device)
    G = torch.rand(K, N, N, device=cuda_device) / N
    dyn = (torch.rand(B, K, N, N, device=cuda_device) / N, torch.rand(B, K, N, N, device=cuda_device) / N)
    x = torch.rand(B, T, N, N, 1, device=cuda_device) * 8
    eager = rollout.forecast(model, x, [G, dyn], P, use_cuda_graph=False)
    graphed = rollout.forecast(model, x, [G, dyn], P, use_cuda_graph=True)
    assert tuple(graphed.shape) == (B, P, N, N, 1)
    assert torch.equal(eager, graphed)
