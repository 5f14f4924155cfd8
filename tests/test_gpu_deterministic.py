"""torch.use_deterministic_algorithms(True) on the GPU: every call that sums across CTAs gives the same bits when repeated with
identical inputs and garbage-filled outputs / workspace, stays close to the default (atomic) path, does not depend on concurrent
work, and a whole training run reproduces bit for bit (DESIGN.md section 11)."""
import ctypes
import contextlib
import warnings

import numpy as np
import pytest
import torch
from torch import nn

from mpgcn_b200 import _lib

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def deterministic(on=True, warn_only=False):
    prev, prev_w = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_w)


def garbage(t, k):
    """k = 0: NaN bytes, else random bytes"""
    b = t.view(torch.uint8)
    if k == 0:
        b.fill_(0xFF)
    else:
        b.copy_(torch.randint(0, 256, b.shape, dtype=torch.uint8, device=b.device, generator=torch.Generator(b.device).manual_seed(k)))


def ws(nbytes, dev):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=dev)


def repeat3(run, outs):
    """run(k) fills `outs` (after they and the workspace were set to garbage k); -> the three runs' outputs as host tensors"""
    res = []
    for k in range(3):
        for o in outs:
            garbage(o, k)
        run(k)
        torch.cuda.synchronize()
        res.append([o.cpu().clone() for o in outs])
    return res


def assert_bitwise(res, what):
    for r in res[1:]:
        for i, (a, b) in enumerate(zip(res[0], r)):
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b), \
                f"{what}: output {i} differs between runs"


def assert_close(a, b, what, rel=2e-4):
    """the deterministic result against the default (atomic) one: the same sums in another order"""
    a, b = a.double(), b.double()
    err = (a - b).norm() / max(b.norm().item(), 1e-30)
    assert err < rel, f"{what}: rel L2 {err:.2e}"


# ------------------------------------------------------------------------------------------------------------------------------
# LSTM: one layer at hidden 32 / 48 (fp32) / 96 / 128, stacks L = 2 at 32 / 96; about 2e5 cells, T = 12
# ------------------------------------------------------------------------------------------------------------------------------
def lstm_case(C, L, dev, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + C + L)
    B, T, NN = 2, 12, 316 * 316
    x = (torch.rand((B, T, NN), generator=g) * 4).to(dev)
    params = []
    for l in range(L):
        params.append([(torch.randn(s, generator=g) * 0.3).to(dev) for s in ((4 * C, 1 if l == 0 else C), (4 * C, C), (4 * C,), (4 * C,))])
    d_hT = (torch.randn((B * NN, C), generator=g) * 1e-3).to(dev)
    return x, params, d_hT, (B, T, NN)


def lstm_backward_runner(C, L, prec, dev):
    """-> (outs, run): run(k) = forward (training state) + backward with its workspace prefilled with garbage k"""
    lib = _lib.load()
    x, params, d_hT, (B, T, NN) = lstm_case(C, L, dev)
    st = torch.cuda.current_stream().cuda_stream
    grads = [[torch.empty_like(p) for p in layer] for layer in params]
    d_x = torch.empty_like(x)
    flat = [o for layer in grads for o in layer] + [d_x]
    if L == 1:
        nsave = lib.mpgcn_lstm_saved_bytes(B, T, NN, C, prec)
        saved = ws(nsave, dev)
        w, gr = params[0], grads[0]

        def run(k):
            lib.mpgcn_set_deterministic(int(torch.are_deterministic_algorithms_enabled()))
            work = ws(lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, prec) - nsave, dev)
            garbage(work, k)
            hT = torch.empty((B * NN, C), device=dev)
            _lib.check(lib.mpgcn_lstm_last_forward_train(x.data_ptr(), *[p.data_ptr() for p in w], hT.data_ptr(),
                                                         saved.data_ptr() if nsave else None, nsave, B, T, NN, C, prec, st), "fwd")
            _lib.check(lib.mpgcn_lstm_last_backward_saved(x.data_ptr(), *[p.data_ptr() for p in w], d_hT.data_ptr(),
                                                          *[o.data_ptr() for o in gr], d_x.data_ptr(), saved.data_ptr() if nsave else None,
                                                          nsave, work.data_ptr(), work.numel(), B, T, NN, C, prec, None, st), "bwd")
        return flat, run
    nsave = lib.mpgcn_lstm_stack_saved_bytes(B, T, NN, C, L, 1)
    saved = ws(nsave, dev)

    def arr(k, src):
        return (ctypes.c_void_p * L)(*[src[l][k].data_ptr() for l in range(L)])

    def run(k):
        lib.mpgcn_set_deterministic(int(torch.are_deterministic_algorithms_enabled()))
        work = ws(lib.mpgcn_lstm_stack_bwd_workspace_bytes(B, T, NN, C, L, 1), dev)
        garbage(work, k)
        hT = torch.empty((B * NN, C), device=dev)
        _lib.check(lib.mpgcn_lstm_stack_forward(x.data_ptr(), L, *[arr(i, params) for i in range(4)], hT.data_ptr(), saved.data_ptr(), nsave,
                                                None, 0, B, T, NN, C, 1, st), "stack fwd")
        _lib.check(lib.mpgcn_lstm_stack_backward(x.data_ptr(), L, *[arr(i, params) for i in range(4)], d_hT.data_ptr(),
                                                 *[arr(i, grads) for i in range(4)], d_x.data_ptr(), saved.data_ptr(), nsave, work.data_ptr(),
                                                 work.numel(), B, T, NN, C, 1, None, st), "stack bwd")
    return flat, run


LSTM_CASES = [(32, 1, 1), (48, 1, 0), (96, 1, 1), (128, 1, 1), (32, 2, 1), (96, 2, 1)]


@pytest.mark.parametrize("C,L,prec", LSTM_CASES)
def test_lstm_backward_repeats_bitwise(C, L, prec, cuda_device):
    outs, run = lstm_backward_runner(C, L, prec, cuda_device)
    with deterministic():
        res = repeat3(run, outs)
    assert_bitwise(res, f"lstm C={C} L={L}")
    ref = repeat3(run, outs)[0]          # the default (atomic) path: the same sums in another order
    for i, (a, b) in enumerate(zip(res[0], ref)):
        assert_close(a, b, f"lstm C={C} L={L} output {i}")
    _lib.load().mpgcn_set_deterministic(0)


# ------------------------------------------------------------------------------------------------------------------------------
# fused head: M = 2, 8; C = 32, 256; 1e6 cells
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,C", [(2, 32), (8, 32), (2, 256), (8, 256)])
def test_head_backward_repeats_bitwise(M, C, cuda_device):
    lib = _lib.load()
    dev = cuda_device
    cells = 10 ** 6 if C == 32 else 250_000
    g = torch.Generator(device="cpu").manual_seed(M * C)
    gs = [torch.randn((cells, C), generator=g).to(dev) for _ in range(M)]
    w = (torch.randn((M, C), generator=g) * 0.2).to(dev)
    b = (torch.randn(M, generator=g) * 0.1).to(dev)
    dy = (torch.randn(cells, generator=g) * 1e-3).to(dev)
    pre = torch.empty((M, cells), device=dev)
    y = torch.empty(cells, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    ptrs = (ctypes.c_void_p * M)(*[t.data_ptr() for t in gs])
    _lib.check(lib.mpgcn_head_forward(ptrs, w.data_ptr(), b.data_ptr(), y.data_ptr(), pre.data_ptr(), cells, C, M, st), "head fwd")
    dgs = [torch.empty_like(t) for t in gs]
    dw, db, amax = torch.empty_like(w), torch.empty_like(b), torch.empty(M, device=dev)
    dptrs = (ctypes.c_void_p * M)(*[t.data_ptr() for t in dgs])

    def run(k):
        lib.mpgcn_set_deterministic(int(torch.are_deterministic_algorithms_enabled()))
        work = ws(lib.mpgcn_head_backward_workspace_bytes(cells, C, M), dev)
        garbage(work, k)
        _lib.check(lib.mpgcn_head_backward_ex(ptrs, w.data_ptr(), pre.data_ptr(), dy.data_ptr(), dptrs, dw.data_ptr(), db.data_ptr(),
                                              amax.data_ptr(), cells, C, M, work.data_ptr(), work.numel(), st), "head bwd")
    outs = [dw, db, amax] + dgs
    with deterministic():
        res = repeat3(run, outs)
    assert_bitwise(res, f"head M={M} C={C}")
    ref = repeat3(run, outs)[0]
    for i, (a, c) in enumerate(zip(res[0], ref)):
        assert_close(a, c, f"head output {i}", rel=1e-5)
    # against float64 (the stage tests' quantities): dw = sum_cell d_pre g, db = sum_cell d_pre
    d = torch.where(pre > 0, dy.unsqueeze(0) / M, torch.zeros_like(pre)).double()
    dw64 = torch.stack([(d[m].unsqueeze(1) * gs[m].double()).sum(0) for m in range(M)])
    assert_close(res[0][0], dw64.cpu(), "head dw vs float64", rel=1e-5)
    assert_close(res[0][1], d.sum(1).cpu(), "head db vs float64", rel=1e-5)
    lib.mpgcn_set_deterministic(0)


# ------------------------------------------------------------------------------------------------------------------------------
# BDGCN backward with bias, fp16 / fp32, static / dynamic, N = 200
# ------------------------------------------------------------------------------------------------------------------------------
def bdgcn_runner(prec, dyn, dev, B=2, N=200, K=3, C=32, H=32):
    lib = _lib.load()
    g = torch.Generator(device="cpu").manual_seed(7 + prec + 2 * dyn)
    X = torch.randn((B, N, N, C), generator=g).to(dev)
    shape = (B, K, N, N) if dyn else (K, N, N)
    Go = (torch.randn(shape, generator=g) / N ** 0.5).to(dev)
    Gd = (torch.randn(shape, generator=g) / N ** 0.5).to(dev) if dyn else Go
    W = (torch.randn((K * K * C, H), generator=g) / (K * C) ** 0.5).to(dev)
    bias = (torch.randn(H, generator=g) * 0.1).to(dev)
    out = torch.empty((B, N, N, H), device=dev)
    saved = ws(lib.mpgcn_bdgcn_saved_bytes(B, N, K, C, H, prec), dev)
    st = torch.cuda.current_stream().cuda_stream
    fws = ws(lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, C, H, dyn, prec), dev)
    _lib.check(lib.mpgcn_bdgcn_forward(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), dyn, W.data_ptr(), bias.data_ptr(), 1, out.data_ptr(),
                                       saved.data_ptr(), fws.data_ptr(), fws.numel(), B, N, K, C, H, prec, st), "bdgcn fwd")
    d_out = (torch.randn((B, N, N, H), generator=g) * 1e-4).to(dev)
    dX, dW, db = torch.empty_like(X), torch.empty_like(W), torch.empty_like(bias)

    def run(k, stream=None):
        lib.mpgcn_set_deterministic(int(torch.are_deterministic_algorithms_enabled()))
        work = ws(lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, dyn, prec), dev)
        garbage(work, k)
        _lib.check(lib.mpgcn_bdgcn_backward(d_out.data_ptr(), out.data_ptr(), Go.data_ptr(), Gd.data_ptr(), dyn, W.data_ptr(), 1,
                                            saved.data_ptr(), dX.data_ptr(), dW.data_ptr(), db.data_ptr(), work.data_ptr(), work.numel(),
                                            B, N, K, C, H, prec, torch.cuda.current_stream().cuda_stream), "bdgcn bwd")
    return [dX, dW, db], run, (d_out, out)


@pytest.mark.parametrize("prec,dyn", [(1, 0), (1, 1), (0, 0), (0, 1)])
def test_bdgcn_backward_repeats_bitwise(prec, dyn, cuda_device):
    outs, run, (d_out, out) = bdgcn_runner(prec, dyn, cuda_device)
    with deterministic():
        res = repeat3(run, outs)
    assert_bitwise(res, f"bdgcn prec={prec} dyn={dyn}")
    ref = repeat3(run, outs)[0]
    for i, (a, b) in enumerate(zip(res[0], ref)):
        assert_close(a, b, f"bdgcn output {i}", rel=1e-5)
    db64 = torch.where(out > 0, d_out, torch.zeros_like(d_out)).double().sum((0, 1, 2)).cpu()
    assert_close(res[0][2], db64, "bdgcn db vs float64", rel=1e-6)
    _lib.load().mpgcn_set_deterministic(0)


def test_construct_dyn_G_repeats_bitwise(cuda_device):
    from mpgcn_b200.dyn_graph import construct_dyn_G
    rng = np.random.default_rng(3)
    od = (rng.random((70, 500, 500, 1)) * 10).astype(np.float32)
    with deterministic():
        res = [construct_dyn_G(od, [6.4, 1.6, 2], device=cuda_device) for _ in range(3)]
    for r in res[1:]:
        assert np.array_equal(r[0], res[0][0]) and np.array_equal(r[1], res[0][1])
    ref = construct_dyn_G(od, [6.4, 1.6, 2], device=cuda_device)
    assert np.abs(ref[1] - res[0][1]).max() < 1e-5 and np.abs(ref[0] - res[0][0]).max() < 1e-5


def test_lstm_independent_of_concurrent_work(cuda_device):
    """An LSTM backward beside a large fp32 BDGCN backward on another stream gives the bits of an isolated run."""
    outs, run = lstm_backward_runner(32, 1, 1, cuda_device)
    b_outs, b_run, _ = bdgcn_runner(0, 0, cuda_device, B=4)
    side = torch.cuda.Stream(cuda_device)
    with deterministic():
        alone = repeat3(run, outs)[0]
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            b_run(1)
        run(2)
        torch.cuda.synchronize()
        together = [o.cpu() for o in outs]
    for a, b in zip(alone, together):
        assert torch.equal(a, b)
    _lib.load().mpgcn_set_deterministic(0)


# ------------------------------------------------------------------------------------------------------------------------------
# whole model: 3 Adam steps, twice from the same state
# ------------------------------------------------------------------------------------------------------------------------------
def _model(hid, layers, prec, N, K, dev, learn_adj=False):
    import MPGCN as shim
    torch.manual_seed(11)
    m = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=layers, gcn_hidden_dim=hid, gcn_num_layers=3,
                   num_nodes=N, user_bias=True, activation=nn.ReLU).to(dev)
    m.lstm_precision = prec
    for mod in m.modules():
        if isinstance(mod, shim.BDGCN):
            mod.precision = prec
            mod.support_grad = learn_adj
        if isinstance(mod, nn.Linear):          # a live head (ReLU of a positive pre-activation), so that every gradient is non-zero
            nn.init.constant_(mod.bias, 0.5)
    return m


def _train(hid, layers, prec, dev, learn_adj=False, branch_streams=None, graphed=False, N=60, K=3, T=7, B=2):
    from mpgcn_b200.GCN import Adj_Processor
    g = torch.Generator(device="cpu").manual_seed(5)
    x = (torch.rand((B, T, N, N, 1), generator=g) * 5).to(dev)
    y = (torch.rand((B, 1, N, N, 1), generator=g) * 5).to(dev)
    flow = torch.rand((N, N), generator=g).to(dev)
    go = torch.rand((B, K, N, N), generator=g).to(dev) / N
    gd = torch.rand((B, K, N, N), generator=g).to(dev) / N
    model = _model(hid, layers, prec, N, K, dev, learn_adj)
    model.branch_streams = branch_streams
    adj = Adj_Processor("random_walk_diffusion", K - 1)
    flow_p = nn.Parameter(flow.clone()) if learn_adj else None
    params = list(model.parameters()) + ([flow_p] if learn_adj else [])
    opt = torch.optim.Adam(params, lr=1e-3, capturable=True)      # eager and graphed runs take the same Adam arithmetic
    crit = nn.MSELoss()
    G = adj.process(flow.unsqueeze(0))[0] if not learn_adj else None
    losses = []
    if graphed:
        from mpgcn_b200.graph_step import GraphedTrainStep
        state = {k: v.clone() for k, v in model.state_dict().items()}
        step = GraphedTrainStep(model, crit, opt, example=(x, y, G, (go, gd)), warmup=2, branch_streams=branch_streams)
        with torch.no_grad():
            for k, v in model.state_dict().items():
                v.copy_(state[k])
            for s in opt.state.values():
                for v in s.values():
                    if torch.is_tensor(v):
                        v.zero_()
        for _ in range(3):
            losses.append(step(x, y, go, gd).detach().clone())
    else:
        for _ in range(3):
            Gs = adj.process(flow_p.unsqueeze(0))[0] if learn_adj else G
            loss = crit(model(x_seq=x, G_list=[Gs, (go, gd)]), y)
            opt.zero_grad(set_to_none=False)
            loss.backward()
            opt.step()
            losses.append(loss.detach().clone())
    torch.cuda.synchronize()
    return [l.cpu() for l in losses], [p.detach().cpu().clone() for p in params]


def _same(a, b, what):
    for i, (u, v) in enumerate(zip(a[0] + a[1], b[0] + b[1])):
        assert torch.equal(u, v), f"{what}: tensor {i} differs"


@pytest.mark.parametrize("hid,layers,prec", [(32, 1, "fp16"), (96, 1, "fp16"), (32, 2, "fp16"), (96, 2, "fp16"), (32, 1, "fp32")])
def test_training_reproduces_bitwise(hid, layers, prec, cuda_device):
    with deterministic():
        a = _train(hid, layers, prec, cuda_device)
        b = _train(hid, layers, prec, cuda_device)
    _same(a, b, f"hidden {hid} L={layers} {prec}")
    assert float(a[0][-1]) != float(a[0][0]), "the steps trained"



def test_training_with_learnable_adjacency_reproduces_bitwise(cuda_device):
    with deterministic():
        a = _train(32, 1, "fp16", cuda_device, learn_adj=True)
        b = _train(32, 1, "fp16", cuda_device, learn_adj=True)
    _same(a, b, "learnable adjacency")


def test_branch_streams_and_graph_replay_match_eager_bitwise(cuda_device):
    with deterministic():
        eager = _train(32, 1, "fp16", cuda_device, branch_streams=False)
        par = _train(32, 1, "fp16", cuda_device, branch_streams=True)
        graphed = _train(32, 1, "fp16", cuda_device, graphed=True, branch_streams=False)
    _same(eager, par, "branch_streams on against off")
    _same(eager, graphed, "GraphedTrainStep replay against eager")


def test_flag_off_restores_every_query_and_the_shard_refuses(cuda_device):
    lib = _lib.load()
    B, T, NN, C = 2, 12, 10000, 32
    before = (lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, 1), lib.mpgcn_head_backward_workspace_bytes(10 ** 5, 32, 2),
              lib.mpgcn_bdgcn_bwd_workspace_bytes(2, 60, 3, 32, 32, 0, 0))
    with deterministic():
        _train(32, 1, "fp16", cuda_device)
    _train(32, 1, "fp16", cuda_device)      # the backward threads sync back to the flag's value
    after = (lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, 1), lib.mpgcn_head_backward_workspace_bytes(10 ** 5, 32, 2),
             lib.mpgcn_bdgcn_bwd_workspace_bytes(2, 60, 3, 32, 32, 0, 0))
    assert lib.mpgcn_get_deterministic() == 0 and before == after
    from mpgcn_b200 import shard
    with deterministic():
        with pytest.raises(RuntimeError, match="relu_backward"):
            shard._ENGINE.relu_backward(torch.zeros((1, 4, 4, 32), device=cuda_device), torch.zeros((1, 4, 4, 32), device=cuda_device), 1, True)
    with deterministic(warn_only=True):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            d_pre, db = shard._ENGINE.relu_backward(torch.ones((1, 4, 4, 32), device=cuda_device),
                                                    torch.ones((1, 4, 4, 32), device=cuda_device), 1, True)
        assert any("no deterministic implementation" in str(x.message) for x in w)
        assert float(db.sum()) == 16 * 32
    _lib.set_deterministic(False)
