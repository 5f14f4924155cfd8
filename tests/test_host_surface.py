"""CPU-only checks of the drop-in boundary: module surface, state_dict contract, error conventions,
and that libmpgcn_b200.so loads and exports every symbol include/mpgcn_b200.h declares."""
import os
import re

import numpy as np
import pytest
import torch
from torch import nn

from conftest import ROOT, load_golden

import MPGCN as shim
from mpgcn_b200 import _lib


def _model(N=6, K=3, hid=8, M=2):
    return shim.MPGCN(M=M, K=K, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=1, gcn_hidden_dim=hid, gcn_num_layers=3,
                      num_nodes=N, user_bias=True, activation=nn.ReLU)


def test_header_symbols_are_exported():
    hdr = open(os.path.join(ROOT, "include", "mpgcn_b200.h")).read()
    declared = set(re.findall(r"MPGCN_API\s+[\w\s\*]+?\b(mpgcn_\w+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/mpgcn_b200.h but not exported"
    assert declared == set(_lib.EXPORTED_SYMBOLS)
    m = re.search(r"#define MPGCN_B200_ABI_VERSION\s+(\d+)", hdr)
    assert m and lib.mpgcn_abi_version() == int(m.group(1)) == _lib.ABI_VERSION


def test_workspace_queries_are_pure_host_functions():
    lib = _lib.load()
    assert lib.mpgcn_bdgcn_precision_supported(2, 50, 3, 32, 32, 1) == 1
    assert lib.mpgcn_bdgcn_precision_supported(2, 50, 3, 16, 32, 1) == 0
    assert lib.mpgcn_bdgcn_precision_supported(2, 50, 3, 16, 7, 0) == 1
    assert lib.mpgcn_bdgcn_saved_bytes(2, 50, 3, 32, 32, 1) == 2 * 3 * 2500 * 32 * 2
    assert lib.mpgcn_bdgcn_saved_bytes(2, 50, 3, 32, 32, 0) == 2 * 3 * 2500 * 32 * 4
    assert lib.mpgcn_bdgcn_fwd_workspace_bytes(2, 50, 3, 32, 32, 0, 1) > 0


def test_null_pointer_is_an_error_not_a_crash():
    lib = _lib.load()
    rc = lib.mpgcn_bdgcn_forward(None, None, None, 0, None, None, 1, None, None, None, 0, 1, 4, 1, 32, 32, 0, None)
    assert rc != 0 and b"null" in lib.mpgcn_last_error()
    rc = lib.mpgcn_bdgcn_forward(None, None, None, 0, None, None, 1, None, None, None, 0, 1, 4, 1, 16, 32, 1, None)
    assert rc != 0 and b"C == H == 32" in lib.mpgcn_last_error()


def test_state_dict_contract_matches_reference_checkpoint():
    g = load_golden("mpgcn_n6_k3")
    ref_params = {k[6:]: v for k, v in g.items() if k.startswith("param:")}
    m = _model()
    sd = m.state_dict()
    assert list(sd.keys()) == list(ref_params.keys())
    for k, v in sd.items():
        assert tuple(v.shape) == ref_params[k].shape, k
    m.load_state_dict({k: torch.from_numpy(v) for k, v in ref_params.items()})     # reference checkpoint loads
    np.testing.assert_array_equal(m.branch_models[1]['spatial'][2].W.detach().numpy(), ref_params["branch_models.1.spatial.2.W"])


def test_constructor_attributes_and_init():
    torch.manual_seed(0)
    layer = shim.BDGCN(K=3, input_dim=4, hidden_dim=5, use_bias=True, activation=nn.ReLU)
    assert (layer.K, layer.input_dim, layer.hidden_dim, layer.use_bias) == (3, 4, 5, True)
    assert isinstance(layer.activation, nn.ReLU)
    assert tuple(layer.W.shape) == (36, 5) and tuple(layer.b.shape) == (5,)
    assert float(layer.b.abs().sum()) == 0.0
    std = float(layer.W.std())
    assert abs(std - (2.0 / (36 + 5)) ** 0.5) < 0.05       # xavier_normal_
    assert not hasattr(shim.BDGCN(K=1, input_dim=2, hidden_dim=2, use_bias=False), "b")
    m = _model()
    assert (m.M, m.K, m.num_nodes, m.lstm_hidden_dim, m.lstm_num_layers, m.gcn_num_layers) == (2, 3, 6, 8, 1, 3)
    h = m.init_hidden_list(2)
    assert len(h) == 2 and tuple(h[0][0].shape) == (1, 2 * 36, 8) and float(h[1][1].abs().sum()) == 0.0


def test_error_conventions():
    layer = shim.BDGCN(K=3, input_dim=4, hidden_dim=5)
    X = torch.zeros(2, 6, 6, 4)
    with pytest.raises(AssertionError):
        layer(X, torch.zeros(2, 6, 6))                       # K mismatch (reference MPGCN.py:27)
    with pytest.raises(AssertionError):
        layer(X, (torch.zeros(2, 2, 6, 6), torch.zeros(2, 3, 6, 6)))   # reference MPGCN.py:35
    with pytest.raises(NotImplementedError):
        layer(X, [torch.zeros(3, 6, 6)])                     # neither Tensor nor tuple (reference MPGCN.py:41-42)
    m = _model()
    with pytest.raises(AssertionError):
        m(torch.zeros(2, 3, 6, 6), [torch.zeros(3, 6, 6)] * 2)          # not 5-D (reference MPGCN.py:95)
    with pytest.raises(AssertionError):
        m(torch.zeros(2, 3, 5, 5, 1), [torch.zeros(3, 5, 5)] * 2)       # N mismatch
    with pytest.raises(AssertionError):
        m(torch.zeros(2, 3, 6, 6, 1), [torch.zeros(3, 6, 6)])           # len(G_list) != M (reference MPGCN.py:96)


def test_cpu_tensors_fail_loudly_no_fallback():
    layer = shim.BDGCN(K=1, input_dim=32, hidden_dim=32)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        layer(torch.zeros(1, 4, 4, 32), torch.zeros(1, 4, 4))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "mpgcn_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("test oracle", ""), f"{f} references the oracle"


def test_adj_processor_surface_and_errors():
    import GCN as gshim
    p = gshim.Adj_Processor("localpool", 5)
    assert (p.kernel_type, p.K) == ("localpool", 1)                 # reference GCN.py:53
    assert gshim.Adj_Processor("random_walk_diffusion", 2).num_supports() == 3          # Model_Trainer.py:30
    assert gshim.Adj_Processor("dual_random_walk_diffusion", 2).num_supports() == 5     # Model_Trainer.py:32
    assert gshim.Adj_Processor("chebyshev", 3).num_supports() == 4
    with pytest.raises(ValueError, match="Invalid kernel_type"):
        gshim.Adj_Processor("bogus", 2).process(torch.zeros(1, 4, 4))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA"):
            gshim.Adj_Processor("localpool", 1).process(torch.ones(1, 4, 4))
    # static helpers behave like the reference's on plain tensors
    A = torch.tensor([[0., 2.], [0., 0.]])
    P = gshim.Adj_Processor.random_walk_normalize(A)
    assert torch.equal(P, torch.tensor([[0., 1.], [0., 0.]]))     # 1/0 -> 0 guard (reference GCN.py:105)


def test_gradient_hint_routing_is_graph_based():
    """ops._producer_node / _put_hint / _take_hint (host logic only): the hand-over walks pure view nodes back to one of our
    autograd nodes, and a hint is honoured only for the very buffer it was written for, unmodified."""
    import torch
    from mpgcn_b200 import ops

    class _LSTMLastFn(torch.autograd.Function):            # stands in for ops._LSTMLastFn: only the node's class name matters
        @staticmethod
        def forward(ctx, x):
            return x * 2

        @staticmethod
        def backward(ctx, g):
            return g * 2

    x = torch.randn(4, 6, requires_grad=True)
    h = _LSTMLastFn.apply(x)
    node = h.grad_fn
    assert ops._producer_node(h) is node
    assert ops._producer_node(h.view(2, 2, 6).reshape(4, 6).view(2, 12)) is node       # views only: same memory
    assert ops._producer_node(h * 1.0) is None                                           # a real op in between
    assert ops._producer_node(x) is None and ops._producer_node(torch.zeros(3)) is None
    g = torch.randn(4, 6)
    scalar = torch.tensor([1.0])
    ops._put_hint(node, g, scalar)
    assert ops._take_hint(node, g) is scalar
    assert ops._take_hint(node, g) is None                                               # consumed
    ops._put_hint(node, g, scalar)
    assert ops._take_hint(node, g.clone()) is None                                       # another buffer (e.g. accumulated gradient)
    ops._put_hint(node, g, scalar)
    g.add_(1.0)                                                                          # modified in place: version bump
    assert ops._take_hint(node, g) is None
    ops._put_hint(None, g, scalar)                                                       # no producer: nothing happens



def test_c_abi_rejects_bad_arguments_without_a_gpu():
    """Argument validation happens before any CUDA call: empty / malformed shapes, unknown precisions, bad layer parts and bad
    exchange slabs come back as error codes with a message (`mpgcn_last_error`), never as a crash -- also on a box without a GPU."""
    import ctypes
    from mpgcn_b200 import _lib
    lib = _lib.load()
    one = ctypes.c_void_p(256)          # any non-null, 256-byte "aligned" pointer: never dereferenced on these paths

    def err():
        return lib.mpgcn_last_error().decode()
    # empty batch / zero nodes (the reference would return empty tensors; the engine refuses them loudly)
    assert lib.mpgcn_bdgcn_forward(one, one, one, 0, one, None, 1, one, None, one, 1 << 20, 0, 8, 3, 32, 32, 0, None) != 0 and "bad BDGCN shape" in err()
    assert lib.mpgcn_bdgcn_forward(one, one, one, 0, one, None, 1, one, None, one, 1 << 20, 2, 0, 3, 32, 32, 0, None) != 0
    assert lib.mpgcn_bdgcn_forward(one, one, one, 0, one, None, 1, one, None, one, 1 << 20, 2, 8, 3, 32, 32, 7, None) != 0 and "unknown precision" in err()
    assert lib.mpgcn_bdgcn_forward(one, one, one, 0, one, None, 2, one, None, one, 1 << 20, 2, 8, 3, 32, 32, 0, None) != 0 and "activation" in err()
    assert lib.mpgcn_bdgcn_forward(one, one, one, 0, one, None, 1, one, None, one, 1 << 20, 2, 8, 3, 16, 32, 1, None) != 0 and "C == H == 32" in err()
    # layer parts
    part = _lib.BdgcnPart(4, 8, 3, 3)                      # rows [4, 12) of N = 8
    assert lib.mpgcn_bdgcn_forward_part(one, one, one, 0, one, one, None, one, 1 << 20, 2, 8, 32, 32, 0, ctypes.addressof(part), None, None) != 0
    assert "bad layer part" in err()
    assert lib.mpgcn_bdgcn_forward_part(one, one, one, 0, one, one, None, one, 1 << 20, 2, 8, 32, 32, 0, None, None, None) != 0 and "part descriptor" in err()
    part = _lib.BdgcnPart(0, 4, 3, 3)
    for prec in (0, 1):                                    # a valid part with no pre_partial buffer
        assert lib.mpgcn_bdgcn_forward_part(one, one, one, 0, one, None, None, one, 1 << 20, 2, 8, 32, 32, prec, ctypes.addressof(part), None, None) != 0
        assert "null pointer" in err()
    # exchange kernels
    arr = (ctypes.c_void_p * 9)(*[256] * 9)
    assert lib.mpgcn_rows_reduce_bias_act(one, arr, 9, None, 1, 1, 8, 0, 4, 32, None) != 0 and "ranks unsupported" in err()
    assert lib.mpgcn_rows_reduce_bias_act(one, arr, 2, None, 1, 1, 8, 6, 4, 32, None) != 0 and "bad slab" in err()
    assert lib.mpgcn_relu_backward_scatter(one, one, 1, arr, 2, None, 1, 8, 6, 4, 32, None) != 0 and "bad slab" in err()
    # LSTM
    assert lib.mpgcn_lstm_last_forward(one, one, one, one, one, one, 0, 4, 16, 32, 0, None) != 0 and "empty input" in err()
    assert lib.mpgcn_lstm_last_forward(one, one, one, one, one, one, 1, 4, 16, 48, 1, None) != 0 and "does not support" in err()
    # sizing queries are pure host functions
    assert lib.mpgcn_bdgcn_part_saved_bytes(2, 8, 32, 32, 1, ctypes.addressof(_lib.BdgcnPart(0, 4, 3, 2))) == 2 * 2 * 4 * 8 * 32 * 2
    assert lib.mpgcn_bdgcn_part_saved_bytes(2, 8, 32, 32, 0, ctypes.addressof(_lib.BdgcnPart(0, 4, 3, 2))) == 2 * 2 * 4 * 8 * 32 * 4
