"""Drop-in surface of the reference's `GCN.py` as far as the trainer uses it: `Adj_Processor`.

`Model_Trainer.py:39-42,84` builds `GCN.Adj_Processor(kernel_type, cheby_order)` once and calls `.process(flow)` on the static
adjacency (`[1,N,N]`) and, twice per training step, on the dynamic origin / destination graphs (`[B,N,N]`, CPU tensors from the
DataLoader), then moves the result to the GPU.  The reference loops over the batch in Python on the CPU; here one call of
`mpgcn_adj_process` builds all B*Ks supports on the device (SURVEY.md section 8(f) rank 1).

Differences, all deliberate: the result lives on the CUDA device (the trainer's `.to(params['GPU'])` becomes a no-op); the
Chebyshev kernel always rescales with lambda_max = 2 -- the branch the reference takes on every torch >= 2 because `torch.eig`
no longer exists and its bare `except` swallows the error (reference GCN.py:117-126).  The reference's unused 1-D `GCN` layer
(GCN.py:6-45, never imported by name) is not provided.

Gradients.  `process` is differentiable with respect to `flow`, as the reference's tensor algebra is: a flow that requires grad
(a learnable adjacency, an `nn.Parameter` OD matrix) gets `dL/dflow` through the supports, from the adjoint of the builder on the
GPU (`mpgcn_adj_process_backward`).  A CPU or float64 flow gets its `.grad` in its own place and type.  At K = 0 the chebyshev
and random-walk kernels return the identity alone, which carries no gradient (as in the reference).  One deliberate difference:
where the random-walk normalisation masks 1/sum to 0 (an empty row, or a column in the dual kernel's backward series; also a
sum so small that its fp32 inverse overflows), that row's or column's contribution to `dL/dflow` is exactly 0.  The reference
returns NaN there (its `pow(s, -1)` backward multiplies 0 by inf), so a learnable OD matrix with an empty station would turn NaN
after one optimiser step.  The symmetric kernels have no such mask: a zero-sum row makes their forward non-finite, and their
gradient then contains NaN, as the reference's does.
"""
from __future__ import annotations

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from .ops import _f32c, _ptr, _scratch, _stream

_KERNELS = {"localpool": 0, "chebyshev": 1, "random_walk_diffusion": 2, "dual_random_walk_diffusion": 3}
_INVALID = "Invalid kernel_type. Must be one of [chebyshev, localpool, random_walk_diffusion, dual_random_walk_diffusion]."


def _adj_process(f: torch.Tensor, kt: int, K: int) -> torch.Tensor:
    """f: float32, contiguous, on the CUDA device -> supports [B, Ks, N, N]."""
    lib = _lib.load()
    B, N = f.shape[0], f.shape[1]
    Ks = lib.mpgcn_adj_num_supports(kt, K)
    out = torch.empty((B, Ks, N, N), dtype=torch.float32, device=f.device)
    ws = _scratch(lib.mpgcn_adj_workspace_bytes(B, N, kt, K), f.device)
    with torch.cuda.device(f.device):
        _lib.check(lib.mpgcn_adj_process(_ptr(f), _ptr(out), B, N, kt, K, _ptr(ws), ws.numel(), _stream()), "adj_process")
    return out


class _AdjProcessFn(torch.autograd.Function):
    """supports = process(flow); the backward reads the saved flow and supports (the T_{k-1} of the recursion's adjoint)."""
    @staticmethod
    @_lib.engine_buffers()
    def forward(ctx, f, kt: int, K: int, grad_mode: bool):
        out = _adj_process(_f32c(f), kt, K)
        if grad_mode and ctx.needs_input_grad[0]:
            ctx.save_for_backward(f, out)
            ctx.kt, ctx.K = kt, K
        return out

    @staticmethod
    @once_differentiable
    @_lib.engine_buffers()
    def backward(ctx, d_out):
        f, out = ctx.saved_tensors
        lib = _lib.load()
        _lib.sync_deterministic()        # already fixed-order; set like every backward so the thread's mode is never stale
        B, N = f.shape[0], f.shape[1]
        g = _f32c(d_out)
        d_flow = torch.empty_like(f)
        ws = _scratch(lib.mpgcn_adj_backward_workspace_bytes(B, N, ctx.kt, ctx.K), f.device)
        with torch.cuda.device(f.device):
            _lib.check(lib.mpgcn_adj_process_backward(_ptr(f), _ptr(out), _ptr(g), _ptr(d_flow), B, N, ctx.kt, ctx.K, _ptr(ws), ws.numel(),
                                                      _stream()), "adj_process_backward")
        return d_flow, None, None, None


class Adj_Processor():
    # Where CPU inputs are staged.  The trainer hands `process` CPU tensors (static adjacency, DataLoader batches) and moves the
    # result `.to(params['GPU'])` afterwards (Model_Trainer.py:41-42,84), so the processor cannot see the target device:
    # it uses, in this order, the `device` given here (class attribute = process-wide default, or per instance), the device of
    # the first CUDA tensor this instance has seen, `torch.cuda.current_device()` -- call `torch.cuda.set_device(params['GPU'])`
    # (INTEGRATION.md) or set `GCN.Adj_Processor.device` when the model does not live on cuda:0.
    device = None

    def __init__(self, kernel_type: str, K: int, device=None):
        self.kernel_type = kernel_type
        self.K = K if self.kernel_type != 'localpool' else 1
        if device is not None:
            self.device = torch.device(device)
        self._seen_device = None

    def _staging_device(self) -> torch.device:
        if self.device is not None:
            return torch.device(self.device)
        if self._seen_device is not None:
            return self._seen_device
        return torch.device("cuda", torch.cuda.current_device())

    def num_supports(self) -> int:
        if self.kernel_type not in _KERNELS:
            raise ValueError(_INVALID)
        return _lib.load().mpgcn_adj_num_supports(_KERNELS[self.kernel_type], self.K)

    def process(self, flow: torch.Tensor) -> torch.Tensor:
        """flow (batch, Origin, Destination) -> supports (batch, K_supports, O, D), on the CUDA device."""
        if self.kernel_type not in _KERNELS:
            raise ValueError(_INVALID)          # the reference raises the same error from inside process() (GCN.py:93-94)
        assert flow.dim() == 3 and flow.shape[1] == flow.shape[2], "flow must be (batch, N, N)"
        if not flow.is_cuda:
            if not torch.cuda.is_available():
                raise RuntimeError("mpgcn_b200.GCN.Adj_Processor needs a CUDA device; the engine has no CPU path")
            flow = flow.to(self._staging_device(), non_blocking=True)
        elif self._seen_device is None:
            self._seen_device = flow.device
        kt = _KERNELS[self.kernel_type]
        f = flow.to(dtype=torch.float32).contiguous()       # autograd ops: a float64 flow gets a float64 .grad
        if kt != _KERNELS["localpool"] and self.K == 0:
            return _adj_process(f.detach(), kt, 0)            # the identity alone: no gradient, as in the reference
        return _AdjProcessFn.apply(f, kt, self.K, torch.is_grad_enabled())

    # ---- the reference's static helpers, kept for API compatibility (plain tensor algebra on the caller's device) ----
    @staticmethod
    def random_walk_normalize(A):
        d_inv = 1.0 / A.sum(dim=1)
        d_inv = torch.where(torch.isinf(d_inv), torch.zeros_like(d_inv), d_inv)
        return d_inv.unsqueeze(1) * A

    @staticmethod
    def symmetric_normalize(A):
        d = A.sum(dim=1).pow(-0.5)
        return (d.unsqueeze(1) * A) * d.unsqueeze(0)

    @staticmethod
    def rescale_laplacian(L):
        eye = torch.eye(L.shape[0], dtype=L.dtype, device=L.device)
        return (2 / 2) * L - eye                 # lambda_max = 2 (see module docstring)

    def compute_chebyshev_polynomials(self, x, T_k):
        eye = torch.eye(x.shape[0], dtype=x.dtype, device=x.device)
        for k in range(self.K + 1):
            T_k.append(eye if k == 0 else x if k == 1 else 2 * torch.mm(x, T_k[k - 1]) - T_k[k - 2])
        return T_k
