"""world_size-2 gloo tests (CPU) of the model-parallel shards (mpgcn_b200/shard.py): the exchange logic -- reduce-scatter of the
partial pre-activation / all-gather of dPre (origin-row shard), all-reduce of pre and dX + row-sharded LSTM (K shard), the
plan-aware gradient reduction -- with the CUDA engine replaced by a torch stand-in (tests/shard_standin.py), against the numpy
oracle of the WHOLE model (reference MPGCN.py:89-112).  One-rank runs check that a sharded layer, and the whole sharded model in
both kinds, refuse supports that require grad (the part kernels have no support gradient)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch import nn

from oracle import mpgcn_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))


def test_shard_plan_partitions():
    from mpgcn_b200 import shard
    for world in (1, 2, 4, 8):
        rows = [shard.ShardPlan("row", r, world, 1000, 3) for r in range(world)]
        assert rows[0].row_lo == 0 and rows[-1].row_hi == 1000 and all(p.rows == 1000 // world for p in rows)
        ks = [shard.ShardPlan("k", r, world, 1000, 6) for r in range(world)]
        assert sum(p.Kd for p in ks) == 6 and ks[0].d_lo == 0 and ks[-1].d_hi == 6
    with pytest.raises(ValueError):
        shard.ShardPlan("row", 0, 3, 1000, 3)


@pytest.mark.parametrize("kind", ["row", "k", "rowhyb"])
def test_sharded_model_world2_matches_whole_model_oracle(kind, tmp_path):
    """row / k: world 2.  rowhyb: world 4 = 2 batch groups x 2 row ranks (the exchange stays inside a group; gradients are summed
    over all ranks and averaged over the groups)."""
    _run_and_check(kind, tmp_path, 8, 8)


@pytest.mark.parametrize("kind", ["row", "k"])
def test_sharded_model_with_lstm_hidden_unlike_gcn_hidden_matches_whole_model_oracle(kind, tmp_path):
    """lstm_hidden_dim 8, gcn_hidden_dim 12: the first BDGCN layer of each branch has C != H, so the K shard's weight slice
    W.view(K, K, C, H)[:, d_lo:d_hi] and the row shard's exchanges of H-channel tensors fed by C-channel slabs are checked."""
    _run_and_check(kind, tmp_path, 8, 12)


def _run_workers(nproc, tmp_path, kind, *args):
    """tests/_shard_worker.py on `nproc` gloo ranks -> what each rank saved"""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    worker = os.path.join(HERE, "_shard_worker.py")
    procs = []
    for r in range(nproc):
        env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(r), WORLD_SIZE=str(nproc))
        procs.append(subprocess.Popen([sys.executable, worker, kind, str(tmp_path / f"r{r}.pt"), *map(str, args)], env=env))
    for p in procs:
        assert p.wait(timeout=300) == 0
    return [torch.load(tmp_path / f"r{r}.pt") for r in range(nproc)]


def _run_and_check(kind, tmp_path, lstm_hid, gcn_hid):
    nproc = 4 if kind == "rowhyb" else 2
    res = _run_workers(nproc, tmp_path, kind, lstm_hid, gcn_hid)
    # the same model / inputs as the worker builds, evaluated whole by the oracle
    sys.path.insert(0, os.path.dirname(HERE))
    import MPGCN as shim
    N, K, T, B = 8, 3, 3, 2
    torch.manual_seed(0)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=lstm_hid, lstm_num_layers=1, gcn_hidden_dim=gcn_hid, gcn_num_layers=3,
                       num_nodes=N, user_bias=True, activation=nn.ReLU)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.05)
    rng = np.random.default_rng(1)
    x = (rng.random((B, T, N, N, 1)) * 4).astype(np.float32)
    y = rng.random((B, 1, N, N, 1)).astype(np.float32)
    G = (rng.random((K, N, N)) / N).astype(np.float32)
    go = (rng.random((B, K, N, N)) / N).astype(np.float32)
    gd = (rng.random((B, K, N, N)) / N).astype(np.float32)
    params = {k: v.detach().numpy().astype(np.float64) for k, v in model.state_dict().items()}
    GL = [G.astype(np.float64), (go.astype(np.float64), gd.astype(np.float64))]
    y_o = orc.mpgcn_forward(params, x.astype(np.float64), GL, M=2, gcn_num_layers=3)
    d_y = 2.0 * (y_o - y) / y.size
    _, grads_o = orc.mpgcn_forward_backward(params, x.astype(np.float64), GL, M=2, gcn_num_layers=3, d_y=d_y)
    loss_o = float(((y_o - y) ** 2).mean())
    if kind == "row":
        pred = np.concatenate([r["pred"].numpy() for r in sorted(res, key=lambda r: r["rank"])], axis=2)
    elif kind == "rowhyb":     # ranks (0,1) hold sample 0's row slabs, ranks (2,3) sample 1's
        by = sorted(res, key=lambda r: r["rank"])
        pred = np.concatenate([np.concatenate([by[2 * gi]["pred"].numpy(), by[2 * gi + 1]["pred"].numpy()], axis=2) for gi in range(2)], axis=0)
    else:
        pred = res[0]["pred"].numpy()
        assert np.array_equal(pred, res[1]["pred"].numpy()), "K shard: the prediction is replicated"
    assert max(orc.rel_errors(pred, y_o)) <= 1e-5
    for r in res:
        assert abs(r["loss"] - loss_o) <= 1e-5 * loss_o
        assert set(r["grads"]) == set(grads_o)
        for k, g in r["grads"].items():
            assert max(orc.rel_errors(g.numpy(), grads_o[k])) <= 2e-5, (kind, k)


def test_k_sharded_layer_on_a_static_stack_world2_matches_the_whole_layer(tmp_path):
    """sharded_bdgcn on a K shard over 2 ranks with a static [K,N,N] stack: each rank contracts the destination side over its own
    supports only.  The replicated output, dX and the rank-summed W / b gradients against a float64 evaluation of the whole layer."""
    res = _run_workers(2, tmp_path, "k-layer")
    r = res[0]
    f64 = lambda t: t.numpy().astype(np.float64)  # noqa: E731
    X, G, W, b, d_out = (f64(r[k]) for k in ("X", "G", "W", "b", "d_out"))
    out_o = orc.bdgcn_forward(X, G, W, b, "relu")
    dX_o, dW_o, db_o = orc.bdgcn_backward(X, G, W, b, "relu", d_out)
    for r in res:
        assert max(orc.rel_errors(r["out"].numpy(), out_o)) <= 1e-5
        for k, want in (("dX", dX_o), ("dW", dW_o), ("db", db_o)):
            assert max(orc.rel_errors(r[k].numpy(), want)) <= 2e-5, k


@pytest.fixture
def world1(monkeypatch):
    """A one-rank gloo group in this process and the torch stand-in engine: a sharded layer runs end to end on the CPU."""
    import torch.distributed as dist
    from mpgcn_b200 import shard
    from shard_standin import TorchEngine
    assert not dist.is_initialized()
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    monkeypatch.setattr(shard, "_ENGINE", TorchEngine())
    try:
        yield shard
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("kind", ["row", "k"])
@pytest.mark.parametrize("support_grad", [False, True])
def test_sharded_layer_refuses_a_support_that_requires_grad(kind, support_grad, world1):
    """The part kernels have no dG stages, so a sharded layer given a support that requires grad raises instead of leaving
    G.grad None, whether or not the layer opted into support gradients; without grad mode, or with G detached, it runs."""
    import MPGCN as shim
    shard = world1
    B, N, K, C = 2, 6, 3, 4
    torch.manual_seed(0)
    layer = shim.BDGCN(K=K, input_dim=C, hidden_dim=C, use_bias=True, activation=nn.ReLU)
    layer.support_grad = support_grad
    plan = shard.ShardPlan(kind, 0, 1, N, K)
    X = torch.rand(B, N, N, C)
    G = (torch.rand(K, N, N) / N).requires_grad_(True)
    dyn = lambda: torch.rand(B, K, N, N) / N
    learnable_o = (dyn().requires_grad_(True), dyn())
    learnable_d = (dyn(), dyn().requires_grad_(True))
    for g in (G, learnable_o, learnable_d):
        with pytest.raises(NotImplementedError, match="whole layers only"):
            shard.sharded_bdgcn(layer, X, g, plan).sum().backward()
    with torch.no_grad():
        assert shard.sharded_bdgcn(layer, X, G, plan).shape == (B, N, N, C)
    out = shard.sharded_bdgcn(layer, X, G.detach(), plan)
    out.sum().backward()
    assert G.grad is None and layer.W.grad is not None and float(layer.W.grad.abs().max()) > 0


@pytest.mark.parametrize("kind", ["row", "k"])
@pytest.mark.parametrize("learnable", ["static", "dynamic"])
def test_sharded_model_refuses_learnable_supports(kind, learnable, world1):
    """The whole sharded model (the trainer's M = 2 layout) with a learnable static stack or a learnable dynamic pair: every branch
    refuses it, including the K shard's static branch, whose layers take the whole stack as G_o and the rank's slice as G_d."""
    import MPGCN as shim
    shard = world1
    B, T, N, K, hid = 2, 3, 6, 3, 4
    torch.manual_seed(0)
    model = shim.MPGCN(M=2, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3, num_nodes=N,
                       user_bias=True, activation=nn.ReLU)
    for mod in model.modules():
        if isinstance(mod, shim.BDGCN):
            mod.support_grad = True
    plan = shard.ShardPlan(kind, 0, 1, N, K)
    x, y = torch.rand(B, T, N, N, 1), torch.rand(B, 1, N, N, 1)
    G = torch.rand(K, N, N) / N
    go, gd = torch.rand(B, K, N, N) / N, torch.rand(B, K, N, N) / N
    xs, ys, gos, gds = shard.shard_host_inputs(plan, x, y, go, gd)
    if learnable == "static":
        G = G.requires_grad_(True)
    else:
        gos, gds = gos.requires_grad_(True), gds.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="whole layers only"):
        shard.sharded_mse_loss(plan, shard.sharded_forward(model, plan, xs, G, (gos, gds)), ys).backward()
    with torch.no_grad():
        shard.sharded_forward(model, plan, xs, G, (gos, gds))
    detached = shard.sharded_forward(model, plan, xs, G.detach(), (gos.detach(), gds.detach()))
    shard.sharded_mse_loss(plan, detached, ys).backward()
    assert all(p.grad is not None for p in model.parameters())


@pytest.mark.parametrize("kind", ["row", "k"])
def test_sharded_model_with_two_input_features_matches_whole_model_oracle(kind, world1):
    """input_dim = 2: each branch's fc is Linear(C -> 2), which the fused head (one output per branch) cannot compute, so the
    sharded model must take the per-branch modules, as the whole model does.  The prediction [B,1,N,N,2], the loss and every
    gradient against the float64 oracle of the whole model."""
    import MPGCN as shim
    shard = world1
    B, T, N, K, I, hid = 2, 3, 6, 3, 2, 8
    torch.manual_seed(0)
    model = shim.MPGCN(M=2, K=K, input_dim=I, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=2, num_nodes=N,
                       user_bias=True, activation=nn.ReLU)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.05)
    rng = np.random.default_rng(3)
    x = (rng.random((B, T, N, N, I)) * 4).astype(np.float32)
    y = rng.random((B, 1, N, N, I)).astype(np.float32)
    G = (rng.random((K, N, N)) / N).astype(np.float32)
    go = (rng.random((B, K, N, N)) / N).astype(np.float32)
    gd = (rng.random((B, K, N, N)) / N).astype(np.float32)
    plan = shard.ShardPlan(kind, 0, 1, N, K)
    xs, ys, gos, gds = shard.shard_host_inputs(plan, *(torch.from_numpy(a) for a in (x, y, go, gd)))
    pred = shard.sharded_forward(model, plan, xs, torch.from_numpy(G), (gos, gds))
    assert tuple(pred.shape) == (B, 1, N, N, I)
    loss = shard.sharded_mse_loss(plan, pred, ys)
    loss.backward()
    params = {k: v.detach().numpy().astype(np.float64) for k, v in model.state_dict().items()}
    GL = [G.astype(np.float64), (go.astype(np.float64), gd.astype(np.float64))]
    y_o = orc.mpgcn_forward(params, x.astype(np.float64), GL, M=2, gcn_num_layers=2)
    _, grads_o = orc.mpgcn_forward_backward(params, x.astype(np.float64), GL, M=2, gcn_num_layers=2, d_y=2.0 * (y_o - y) / y.size)
    assert max(orc.rel_errors(pred.detach().numpy(), y_o)) <= 1e-5
    loss_o = float(((y_o - y) ** 2).mean())
    assert abs(float(loss.detach()) - loss_o) <= 1e-5 * loss_o
    named = dict(model.named_parameters())
    assert set(named) == set(grads_o)
    for k, p in named.items():
        assert max(orc.rel_errors(p.grad.numpy(), grads_o[k])) <= 2e-5, (kind, k)


@pytest.mark.parametrize("kind", ["row", "k"])
def test_sharded_model_refuses_what_the_whole_model_refuses(kind, world1):
    """Inputs whose node count is not the model's num_nodes, and a model whose branch count does not match the supports given
    (the sharded model always passes the trainer's two): the sharded model raises the whole model's AssertionError."""
    import MPGCN as shim
    shard = world1
    B, T, N, K, hid = 2, 3, 6, 3, 4

    def model(M, num_nodes):
        return shim.MPGCN(M=M, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=2,
                          num_nodes=num_nodes, user_bias=True, activation=nn.ReLU)

    x, y = torch.rand(B, T, N, N, 1), torch.rand(B, 1, N, N, 1)
    G = torch.rand(K, N, N) / N
    go, gd = torch.rand(B, K, N, N) / N, torch.rand(B, K, N, N) / N
    plan = shard.ShardPlan(kind, 0, 1, N, K)
    xs, _, gos, gds = shard.shard_host_inputs(plan, x, y, go, gd)
    for wrong in (model(2, N + 1), model(3, N)):
        with pytest.raises(AssertionError):
            wrong(x_seq=x, G_list=[G, (go, gd)])
        with pytest.raises(AssertionError):
            shard.sharded_forward(wrong, plan, xs, G, (gos, gds))
