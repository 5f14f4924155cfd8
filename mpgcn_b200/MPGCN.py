"""Drop-in module surface of the reference's `MPGCN.py`, backed by the H100 engine.

`Model_Trainer.py:5` does `import GCN, MPGCN` by bare name and builds
`MPGCN.MPGCN(M=..., K=..., ..., user_bias=..., activation=nn.ReLU)` (Model_Trainer.py:47-56); put this
repository ahead of the reference on `sys.path` (the root-level `MPGCN.py` re-exports this module)
and the trainer runs unchanged on our kernels.  What is kept identical to the reference:

  * class names, constructor signatures (including the `user_bias` spelling) and attributes;
  * parameter names / shapes / init: `W [K*K*C_in, H]` Xavier-normal with row order (o, d, l),
    `b [H]` zeros (reference MPGCN.py:16-22); `state_dict` keys `branch_models.{m}.temporal.*`,
    `branch_models.{m}.spatial.{n}.{W,b}`, `branch_models.{m}.fc.0.{weight,bias}` -- checkpoints are
    interchangeable in both directions;
  * call conventions and error behaviour: `forward(X, G)` with G a `[K,N,N]` tensor or a 2-tuple of
    `[B,K,N,N]` tensors, AssertionError on K / shape mismatches, NotImplementedError for any other G
    (reference MPGCN.py:26-42, 95-96).

What differs: the arithmetic.  No einsum / cat / cuDNN -- `BDGCN.forward` is one call of
`ops.bdgcn` (factored 2K-contraction engine; a static G may be a sparse COO tensor, DESIGN.md section 12) and the per-cell LSTM is `ops.lstm_module_last`, which reads
`x_seq` in place, assumes the zero initial state the reference always passes (MPGCN.py:80-87,98) and
never materialises the `[B*N*N, T, C]` output sequence.
"""
from __future__ import annotations

import contextlib
from typing import Callable, NamedTuple

import torch
from torch import nn

from . import ops


class BDGCN(nn.Module):
    """2-D (origin x destination) multi-graph convolution.  Reference: MPGCN.py:6-50."""

    def __init__(self, K: int, input_dim: int, hidden_dim: int, use_bias=True, activation=None):
        super().__init__()
        self.K = K
        self.input_dim = input_dim
        self.hidden_dim = hidden_dim
        self.use_bias = use_bias
        self.activation = activation() if activation is not None else None     # a class, as in the reference (MPGCN.py:13)
        self.precision = None          # None -> ops.default_precision(); or "auto" / "fp16" / "bf16x3" / "fp32"
        self.support_grad = False      # True: a G that requires grad gets dL/dG (opt-in: it doubles the layer's N^3 backward work)
        self.init_params()

    def init_params(self, b_init=0.0):
        self.W = nn.Parameter(torch.empty(self.input_dim * (self.K ** 2), self.hidden_dim), requires_grad=True)
        nn.init.xavier_normal_(self.W)
        if self.use_bias:
            self.b = nn.Parameter(torch.empty(self.hidden_dim), requires_grad=True)
            nn.init.constant_(self.b, val=b_init)

    def extra_repr(self) -> str:
        return f"K={self.K}, {self.input_dim} -> {self.hidden_dim}, bias={self.use_bias}"

    def fused_act(self):
        """The activation the layer kernels fuse into their epilogue: 1 ReLU, 0 none.  None for any other activation, which
        forward() applies after the kernel and the sharded layers (mpgcn_b200.shard.sharded_bdgcn) refuse."""
        if self.activation is None:
            return 0
        return 1 if isinstance(self.activation, nn.ReLU) else None

    def forward(self, X: torch.Tensor, G):
        if isinstance(G, torch.Tensor):                     # static supports (K, N, N)
            assert self.K == G.shape[-3]
            assert G.dim() == 3, "static graph input must be (K, N, N)"
        elif isinstance(G, tuple):                          # dynamic supports ((B,K,N,N), (B,K,N,N))
            assert (len(G) == 2) & (self.K == G[0].shape[-3] == G[1].shape[-3])
            assert G[0].dim() == 4 and G[1].dim() == 4 and G[0].shape[0] == X.shape[0] == G[1].shape[0]
        else:
            raise NotImplementedError
        N = (G if isinstance(G, torch.Tensor) else G[0]).shape[-1]      # (no select on a sparse stack)
        assert X.dim() == 4 and X.shape[1] == X.shape[2] == N and X.shape[3] == self.input_dim
        act = self.fused_act()
        out = ops.bdgcn(X, G, self.W, self.b if self.use_bias else None, relu=act == 1, precision=self.precision,
                        support_grad=self.support_grad)
        if act is None:                                     # any other activation: unfused epilogue
            out = self.activation(out)
        return out


class BranchRunner(NamedTuple):
    """How MPGCN._forward evaluates a branch: with the whole model's own parts (MPGCN.forward) or a shard's
    (mpgcn_b200.shard.sharded_forward)."""
    temporal: Callable      # (nn.LSTM, x_seq [B,T,rows,N,I]) -> the LSTM's last hidden state [B, rows, N, C] (the K shard: all N rows)
    layer: Callable         # (BDGCN, X, G, branch index) -> the layer's output
    head: Callable          # the fused head of fc_head: (feats, w [M, C], b [M]) -> [..., 1]
    streams: bool           # evaluate the branches on one CUDA stream each


class MPGCN(nn.Module):
    """Multi-perspective model: per branch LSTM -> L x BDGCN -> Linear+ReLU, mean over branches.
    Reference: MPGCN.py:54-112."""

    def __init__(self, M: int, K: int, input_dim: int, lstm_hidden_dim: int, lstm_num_layers: int, gcn_hidden_dim: int,
                 gcn_num_layers: int, num_nodes: int, user_bias: bool, activation=None):
        super().__init__()
        self.M = M
        self.K = K
        self.num_nodes = num_nodes
        self.lstm_hidden_dim = lstm_hidden_dim
        self.lstm_num_layers = lstm_num_layers
        self.gcn_num_layers = gcn_num_layers
        self.lstm_precision = None      # None -> ops.default_precision(); or "auto" / "fp16" / "fp32" ("bf16x3" reads as "auto")
        # True (or a number of cells per chunk): the tensor-core LSTM keeps no training state in the forward and its backward
        # rebuilds it a chunk at a time (ops.lstm_last), for models whose state does not fit; None -> off
        self.lstm_recompute = None
        # True: evaluate the M branches on M CUDA streams (they are independent until the head, reference MPGCN.py:101-110), so that
        # the HBM-bound elementwise kernels of one branch run beside the tensor-bound contractions of the other; None -> off
        self.branch_streams = None
        self._streams = None
        self.branch_models = nn.ModuleList()
        for _ in range(self.M):
            branch = nn.ModuleDict()
            # nn.LSTM is kept as the parameter container so state_dict keys / default init match
            branch['temporal'] = nn.LSTM(input_size=input_dim, hidden_size=lstm_hidden_dim, num_layers=lstm_num_layers, batch_first=True)
            branch['spatial'] = nn.ModuleList(
                BDGCN(K=K, input_dim=lstm_hidden_dim if n == 0 else gcn_hidden_dim, hidden_dim=gcn_hidden_dim,
                      use_bias=user_bias, activation=activation) for n in range(gcn_num_layers))
            branch['fc'] = nn.Sequential(nn.Linear(in_features=gcn_hidden_dim, out_features=input_dim, bias=True), nn.ReLU())
            self.branch_models.append(branch)

    def init_hidden_list(self, batch_size: int):
        """Kept for API compatibility (reference MPGCN.py:80-87); forward() does not need it."""
        weight = next(self.parameters()).data
        shape = (self.lstm_num_layers, batch_size * (self.num_nodes ** 2), self.lstm_hidden_dim)
        return [(weight.new_zeros(shape), weight.new_zeros(shape)) for _ in range(self.M)]

    def _temporal(self, lstm: nn.LSTM, x_seq: torch.Tensor) -> torch.Tensor:
        B, _, rows, N, _ = x_seq.shape
        return ops.lstm_module_last(lstm, x_seq, self.lstm_precision, self.lstm_recompute).reshape(B, rows, N, self.lstm_hidden_dim)

    def forward(self, x_seq: torch.Tensor, G_list: list):
        """x_seq (B, T, N, N, 1); G_list: per branch a static (K,N,N) tensor or a dynamic tuple.  -> (B, 1, N, N, 1)"""
        run = BranchRunner(self._temporal, lambda layer, X, G, m: layer(X, G), ops.fc_relu_mean, bool(self.branch_streams))
        return self._forward(x_seq, G_list, self.num_nodes, run)

    def _forward(self, x_seq: torch.Tensor, G_list: list, rows: int, run: BranchRunner):
        """The branches and the head on x_seq [B, T, rows, N, I]: every origin row (rows = N), or a shard's slab of them."""
        assert (len(x_seq.shape) == 5) & (rows == x_seq.shape[2]) & (self.num_nodes == x_seq.shape[3])
        assert len(G_list) == self.M
        use_streams = run.streams and x_seq.is_cuda and self.M > 1
        capturing = use_streams and torch.cuda.is_current_stream_capturing()
        cur = torch.cuda.current_stream() if use_streams else None
        if use_streams and (self._streams is None or self._streams[0].device != x_seq.device):
            self._streams = [torch.cuda.Stream(device=x_seq.device) for _ in range(self.M)]
        feats = []
        for m in range(self.M):
            branch = self.branch_models[m]
            if use_streams:
                self._streams[m].wait_stream(cur)
            with (torch.cuda.stream(self._streams[m]) if use_streams else contextlib.nullcontext()):
                gcn_in = run.temporal(branch['temporal'], x_seq)
                for layer in branch['spatial']:
                    gcn_in = run.layer(layer, gcn_in, G_list[m], m)
            feats.append(gcn_in)
        if use_streams:
            for m in range(self.M):
                cur.wait_stream(self._streams[m])
                if not capturing:       # under CUDA-graph capture the join above is a graph dependency: later frees / re-uses are ordered by it
                    feats[m].record_stream(cur)
        ensemble_out = fc_head([self.branch_models[m]['fc'] for m in range(self.M)], feats, run.head)
        return ensemble_out.unsqueeze(dim=1)


def fc_head(fcs, feats, fused):
    """The FC head of every branch and the mean over branches (reference MPGCN.py:107,110): fcs[m] is branch m's
    Sequential(Linear(C -> input_dim), ReLU), feats[m] its last BDGCN output [..., C] -> [..., input_dim].
    Where the fused kernel applies (input_dim 1, C a multiple of 4, at most 8 branches) it computes all of it in one pass:
    `fused(feats, w [M, C], b [M])`; otherwise each branch runs its own modules."""
    lins = [fc[0] for fc in fcs]
    if all(lin.out_features == 1 for lin in lins) and feats[0].shape[-1] % 4 == 0 and len(fcs) <= 8:
        w = torch.cat([lin.weight for lin in lins], dim=0)             # [M, C]
        b = torch.cat([lin.bias for lin in lins], dim=0)               # [M]
        return fused(feats, w, b)                                      # [..., 1]
    return torch.mean(torch.stack([fc(f) for fc, f in zip(fcs, feats)], dim=-1), dim=-1)
