"""Model-parallel shards of the hot path over the GPUs of one node (SURVEY.md section 8(e) rows 1-2), one process per GPU.

The reference has no distributed code (SURVEY.md section 2.1); this is the engine's own addition behind the same math
(`BDGCN.forward`, reference MPGCN.py:24-50; model glue MPGCN.py:89-112).  Both shards split ONE sample's work, so they
scale a fixed batch ("strong" scaling) -- the batch shard of `mpgcn_b200.dist` scales the number of samples instead.

origin-row shard (`kind="row"`, 8(e) row 1).  Rank j owns the origin rows n in slab_j of every activation: the LSTM, the
    destination contraction Z = X x_2 G_d, the channel mix and the FC head are row-local.  The origin contraction sums over n,
    so rank j produces the PARTIAL pre-activation sum_o G_o[slab_j, :]^T U_o[slab_j] for every output row m and the ranks
    exchange it with ONE reduce-scatter over m per layer (sample by sample, so that the slabs stay in the reference's
    [B, rows, N, C] layout); bias + ReLU (MPGCN.py:47-49) run after the exchange on the rank's own rows.  Backward: the masked
    dPre of the rank's rows is all-gathered (same size), everything after that is local; the parameter gradients are partial
    sums over the rank's cells and are summed once per step with the LSTM / head gradients (< 200 KB).
K shard (`kind="k"`, 8(e) row 2, the partition north_star names).  Rank j owns the destination supports d in D_j: it
    evaluates Z_d and U_o^(j) = sum_{d in D_j} Z_d W[o,d] for all o and the origin contraction of that partial U; ONE all-reduce
    of the pre-activation per layer forward and of dX per layer backward.  The origin contraction (and V = G_o x_1 dPre) is
    replicated, which bounds the speed-up by 2K / (K/g + K) < 2 (SURVEY.md section 8(e)); the LSTM is row-sharded (its cells are
    independent) with an all-gather of h_T, the head is replicated.

All arithmetic is in libmpgcn_b200.so (`mpgcn_bdgcn_forward_part` / `_backward_part`, `mpgcn_bias_act`,
`mpgcn_relu_backward`); torch.distributed (NCCL over NVLink / NVSwitch) moves the partial sums.  `_ENGINE` is the compute
back end; tests swap in a CPU stand-in to run the exchange logic under gloo (tests/test_shard_gloo.py).
"""
from __future__ import annotations

import ctypes
import warnings

import torch
import torch.distributed as dist

from . import _lib, ops
from .MPGCN import BranchRunner
from .dist import shard_range


class ShardPlan:
    """Who owns what.  kind "row": origin rows [row_lo, row_hi) (N must divide evenly: the reduce-scatter needs equal slabs);
    kind "k": destination supports [d_lo, d_hi) (may be empty when world > K) plus the same row slab for the LSTM."""

    def __init__(self, kind: str, rank: int, world: int, N: int, K: int, group=None):
        if kind not in ("row", "k"):
            raise ValueError(f"unknown shard kind {kind!r}")
        if N % world != 0:
            raise ValueError(f"the {kind} shard needs N ({N}) to be a multiple of the number of ranks ({world})")
        self.kind, self.rank, self.world, self.N, self.K, self.group = kind, rank, world, N, K, group
        self.row_lo, self.row_hi = shard_range(N, rank, world)
        self.rows = self.row_hi - self.row_lo
        self.d_lo, self.d_hi = shard_range(K, rank, world) if kind == "k" else (0, K)
        self.Kd = self.d_hi - self.d_lo
        self.peer = None          # PeerExchange once enable_peer_exchange() succeeded (row shard over NVLink peer memory)

    def describe(self) -> dict:
        d = {"kind": self.kind, "world": self.world, "rows_per_rank": self.rows,
             "exchange": ("peer memory: P2P loads / stores inside mpgcn_rows_reduce_bias_act / mpgcn_relu_backward_scatter" if self.peer is not None
                          else "NCCL collectives"),
             "collective_per_layer": ("reduce-scatter of pre [B,N,N,H] fp32 forward, all-gather of dPre backward" if self.kind == "row"
                                      else "all-reduce of pre [B,N,N,H] fp32 forward, all-reduce of dX backward; all-gather of h_T once per branch")}
        if self.kind == "k":
            d["supports_per_rank"] = [shard_range(self.K, r, self.world)[1] - shard_range(self.K, r, self.world)[0] for r in range(self.world)]
        return d


# ------------------------------------------------------------------------------------------------
# compute back end (the C ABI); tests replace it by a CPU stand-in to exercise the exchange logic under gloo
# ------------------------------------------------------------------------------------------------
def _no_deterministic(op: str) -> None:
    """The sharded layers' exchange kernels (mpgcn_relu_backward[_scatter[_f16]]) and NCCL have no fixed-order implementation.
    Under torch.use_deterministic_algorithms(True) this raises, as torch's own ops without one do; with warn_only=True it warns and
    the op runs as it does without the flag (this thread's library mode is set off for it)."""
    if not torch.are_deterministic_algorithms_enabled():
        return
    msg = (f"mpgcn_b200.shard: {op} has no deterministic implementation (its exchange steps sum with atomics and NCCL), but "
           "torch.use_deterministic_algorithms(True) is set")
    if not torch.is_deterministic_algorithms_warn_only_enabled():
        raise RuntimeError(msg)
    warnings.warn(msg)
    _lib.set_deterministic(False)


class CudaEngine:
    def _part(self, row0, rows, Ko, Kd):
        return _lib.BdgcnPart(row0, rows, Ko, Kd)

    def prepared(self, G, Gc, planes, N, prec):
        """fp16 staging of a support stack, converted once per tensor (mpgcn_b200.ops cache) and reused by every layer, forward and
        backward; None for the fp32 kernels"""
        if prec != _lib.PREC_FP16_TC:
            return None
        with torch.cuda.device(Gc.device):
            return ops._prepared_supports(_lib.load(), G, Gc, planes, N)

    def forward_part(self, X, Go, Gd, dynamic, W, N, row0, Ko, Kd, prec, keep, out=None, preps=(None, None)):
        """X [B,rows,N,C] -> (raw partial pre-activation [B,N,N,H] (written into `out` if given), Z stash or None)"""
        lib = _lib.load()
        ops._require_cuda(X, "X")
        B, rows, _, C = X.shape
        H = W.shape[1]
        part = self._part(row0, rows, Ko, Kd)
        pp = ctypes.addressof(part)
        pre = out if out is not None else torch.empty((B, N, N, H), dtype=torch.float32, device=X.device)
        saved = ops._scratch(lib.mpgcn_bdgcn_part_saved_bytes(B, N, C, H, prec, pp), X.device) if keep else None
        ws = ops._scratch(lib.mpgcn_bdgcn_part_fwd_workspace_bytes(B, N, C, H, int(dynamic), prec, pp), X.device)
        ex = _lib.BdgcnExtras()
        ex.go_prepared, ex.gd_prepared = ops._ptr(preps[0]), ops._ptr(preps[1])
        with torch.cuda.device(X.device):
            _lib.check(lib.mpgcn_bdgcn_forward_part(X.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dynamic), W.data_ptr(), ops._ptr(pre),
                                                    ops._ptr(saved), ws.data_ptr(), ws.numel(), B, N, C, H, prec, pp, ctypes.addressof(ex),
                                                    ops._stream()), "bdgcn_forward_part")
        return pre, saved

    def backward_part(self, d_pre, Go, Gd, dynamic, W, saved, N, row0, rows, Ko, Kd, C, prec, need_dx, preps=(None, None), d_pre16=None,
                      scale2=None):
        """d_pre [B,N,N,H] (every origin row, masked; fp32, or `d_pre16` + `scale2` from relu_backward_scatter_f16)
        -> (dX [B,rows,N,C] or None, dW [Ko*Kd*C, H])"""
        lib = _lib.load()
        if d_pre is None:
            d_pre = d_pre16
        B, H = d_pre.shape[0], d_pre.shape[-1]
        part = self._part(row0, rows, Ko, Kd)
        pp = ctypes.addressof(part)
        dX = torch.empty((B, rows, N, C), dtype=torch.float32, device=d_pre.device) if need_dx else None
        dW = torch.empty((Ko * Kd * C, H), dtype=torch.float32, device=d_pre.device)
        ws = ops._scratch(lib.mpgcn_bdgcn_part_bwd_workspace_bytes(B, N, C, H, int(dynamic), prec, pp), d_pre.device)
        ex = _lib.BdgcnExtras()
        ex.go_prepared, ex.gd_prepared = ops._ptr(preps[0]), ops._ptr(preps[1])
        ex.d_pre_f16, ex.d_pre_scale2 = ops._ptr(d_pre16), ops._ptr(scale2)
        with torch.cuda.device(d_pre.device):
            _lib.check(lib.mpgcn_bdgcn_backward_part(None if d_pre16 is not None else d_pre.data_ptr(), Go.data_ptr(), Gd.data_ptr(), int(dynamic),
                                                     W.data_ptr(), saved.data_ptr(), ops._ptr(dX), dW.data_ptr(), ws.data_ptr(), ws.numel(), B, N, C, H,
                                                     prec, pp, ctypes.addressof(ex), ops._stream()), "bdgcn_backward_part")
        return dX, dW

    def bias_act(self, pre, bias, act):
        """in place: pre = act(pre + bias)"""
        lib = _lib.load()
        with torch.cuda.device(pre.device):
            _lib.check(lib.mpgcn_bias_act(pre.data_ptr(), ops._ptr(bias), int(act), pre.numel(), pre.shape[-1], ops._stream()), "bias_act")
        return pre

    def relu_backward(self, d_out, out, act, want_db):
        lib = _lib.load()
        _no_deterministic("relu_backward")
        d_pre = torch.empty_like(d_out)
        db = torch.empty(d_out.shape[-1], dtype=torch.float32, device=d_out.device) if want_db else None
        with torch.cuda.device(d_out.device):
            _lib.check(lib.mpgcn_relu_backward(d_out.data_ptr(), out.data_ptr(), int(act), d_pre.data_ptr(), ops._ptr(db), d_out.numel(),
                                               d_out.shape[-1], ops._stream()), "relu_backward")
        return d_pre, db

    def rows_reduce_bias_act(self, ptrs, B, N, row0, rows, H, bias, act, device):
        """out [B,rows,N,H] = act(sum over the g buffers at `ptrs` of the rank's rows + bias); the buffers are whole [B,N,N,H]
        partials (own + peers')"""
        lib = _lib.load()
        out = torch.empty((B, rows, N, H), dtype=torch.float32, device=device)
        arr = (ctypes.c_void_p * len(ptrs))(*ptrs)
        with torch.cuda.device(device):
            _lib.check(lib.mpgcn_rows_reduce_bias_act(out.data_ptr(), arr, len(ptrs), ops._ptr(bias), int(act), B, N, row0, rows, H,
                                                      ops._stream()), "rows_reduce_bias_act")
        return out

    def relu_backward_scatter(self, d_out, out, act, ptrs, N, row0, want_db):
        """mask the rank's rows of d_out and store them into rows [row0, ..) of every buffer at `ptrs`; -> db or None"""
        lib = _lib.load()
        _no_deterministic("relu_backward_scatter")
        B, rows, _, H = d_out.shape
        db = torch.empty(H, dtype=torch.float32, device=d_out.device) if want_db else None
        arr = (ctypes.c_void_p * len(ptrs))(*ptrs)
        with torch.cuda.device(d_out.device):
            _lib.check(lib.mpgcn_relu_backward_scatter(d_out.data_ptr(), out.data_ptr(), int(act), arr, len(ptrs), ops._ptr(db), B, N, row0, rows, H,
                                                       ops._stream()), "relu_backward_scatter")
        return db

    def absmax(self, x):
        lib = _lib.load()
        out = torch.empty(1, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(lib.mpgcn_absmax(x.data_ptr(), x.numel(), out.data_ptr(), ops._stream()), "absmax")
        return out

    def relu_backward_scatter_f16(self, d_out, out, act, ptrs, N, row0, want_db, absmax):
        """fp16 flavour: -> (db or None, scale2 [S, 1/S]); every buffer at `ptrs` (fp16 [B,N,N,H]) receives fp16(S * masked d_out rows)"""
        lib = _lib.load()
        _no_deterministic("relu_backward_scatter_f16")
        B, rows, _, H = d_out.shape
        db = torch.empty(H, dtype=torch.float32, device=d_out.device) if want_db else None
        scale2 = torch.empty(2, dtype=torch.float32, device=d_out.device)
        arr = (ctypes.c_void_p * len(ptrs))(*ptrs)
        with torch.cuda.device(d_out.device):
            _lib.check(lib.mpgcn_relu_backward_scatter_f16(d_out.data_ptr(), out.data_ptr(), int(act), arr, len(ptrs), ops._ptr(db), absmax.data_ptr(),
                                                           scale2.data_ptr(), B, N, row0, rows, H, ops._stream()), "relu_backward_scatter_f16")
        return db, scale2

    def lstm_last(self, x_seq, lstm, precision, recompute=None):
        return ops.lstm_module_last(lstm, x_seq, precision, recompute)

    def head(self, feats, w, b):
        return ops.fc_relu_mean(feats, w, b)

    def resolve_precision(self, name, B, N, K, C, H):
        return ops.resolve_precision(name, B, N, K, C, H)


_ENGINE = CudaEngine()


class PeerExchange:
    """Symmetric [B,N,N,H] fp32 buffers of the row shard, mapped into every rank (torch.distributed._symmetric_memory: cuMem
    allocations exchanged once at rendezvous; `buffer_ptrs[r]` is rank r's buffer as a device pointer valid in THIS process).
    With them the two exchange steps of a layer run inside this library's own kernels -- P2P loads / stores over NVLink --
    instead of a separate NCCL collective whose kernels compete with the persistent contraction kernels for SMs:
        forward   every rank writes its partial pre-activation into ITS buffer, barrier, `mpgcn_rows_reduce_bias_act` reads the
                  rank's rows out of all g buffers (reduce-scatter + bias + ReLU in one pass);
        backward  `mpgcn_relu_backward_scatter[_f16]` masks the rank's dOut rows and stores them into ALL g buffers (all-gather
                  fused with the mask; tensor-core path: already scaled and cast to fp16, half the bytes), barrier,
                  `mpgcn_bdgcn_backward_part` reads the local copy.
    Two buffers per direction alternate from layer to layer; with ONE barrier per exchange that is enough: a rank re-uses
    buffer X two layers later, after a barrier that every rank enters only when it is done with the previous use of X."""

    def __init__(self, plan, device):
        import torch.distributed._symmetric_memory as symm_mem
        self.symm_mem, self.plan, self.device = symm_mem, plan, device
        self.group = plan.group if plan.group is not None else dist.group.WORLD
        self.bufs = {}            # (direction, parity, numel) -> (tensor, handle)
        self.count = {}

    def next(self, direction, shape, dtype=torch.float32):
        """-> (tensor [shape] in this rank's symmetric buffer, handle); alternates between two buffers per direction"""
        numel = 1
        for d in shape:
            numel *= d
        self.count.setdefault(direction, 0)
        key = (direction, self.count[direction] & 1, numel, dtype)
        self.count[direction] += 1
        if key not in self.bufs:
            t = self.symm_mem.empty(numel, dtype=dtype, device=self.device)
            hdl = self.symm_mem.rendezvous(t, self.group)            # collective: every rank allocates in the same order
            self.bufs[key] = (t, hdl)
        t, hdl = self.bufs[key]
        return t.view(shape), hdl


def enable_peer_exchange(plan, device) -> bool:
    """Try to switch the row shard of `plan` to the peer-memory exchange (NCCL backend, CUDA symmetric memory available on every
    rank).  Collective.  Returns whether it is on; on failure anywhere every rank stays on the NCCL collectives."""
    ok = 0
    if plan.kind == "row" and _backend(plan.group) == "nccl":
        try:
            px = PeerExchange(plan, device)
            ok = 1
        except Exception:
            ok = 0
    flag = torch.tensor([ok], device=device, dtype=torch.int32)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=plan.group)
    if int(flag.item()) == 1:
        try:
            px.next("probe", (4,))[1].barrier()        # smoke: one tiny rendezvous + barrier, so that a failure shows up here
            plan.peer = px
        except Exception as e:
            plan.peer = None
            flag.zero_()
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=plan.group)
        if int(flag.item()) != 1:
            plan.peer = None
    return plan.peer is not None


# ------------------------------------------------------------------------------------------------
# exchange steps
# ------------------------------------------------------------------------------------------------
def _backend(group=None) -> str:
    return dist.get_backend(group)


class _Pending:
    """An exchange in flight: `wait()` makes the current stream wait for it (NCCL: the collective runs on NCCL's own stream and
    overlaps whatever the compute stream does in between) and finishes the gloo emulation."""

    def __init__(self, work=None, finish=None):
        self.work, self.finish = work, finish

    def wait(self):
        if self.work is not None:
            self.work.wait()
        if self.finish is not None:
            self.finish()


def reduce_scatter_rows_begin(partial: torch.Tensor, out: torch.Tensor, plan: ShardPlan) -> _Pending:
    """partial [N(m), N, H] (ONE sample: this rank's partial sum for every origin row m) -> out [rows, N, H]: the sum over the
    ranks of the rows this rank owns.  Asynchronous: the next sample's contractions run while this one is exchanged."""
    if _backend(plan.group) == "nccl":
        return _Pending(dist.reduce_scatter_tensor(out, partial, group=plan.group, async_op=True))
    # gloo (CPU tests) has no reduce-scatter: all-reduce, keep the own rows
    work = dist.all_reduce(partial, group=plan.group, async_op=True)
    return _Pending(work, lambda: out.copy_(partial[plan.row_lo:plan.row_hi]))


def all_gather_rows_begin(slab: torch.Tensor, full: torch.Tensor, plan: ShardPlan) -> _Pending:
    """slab [rows, N, H] of ONE sample -> full [N, N, H] (rank r's rows at r*rows ..), asynchronously."""
    if _backend(plan.group) == "nccl":
        return _Pending(dist.all_gather_into_tensor(full, slab, group=plan.group, async_op=True))
    parts = [torch.empty_like(slab) for _ in range(plan.world)]
    work = dist.all_gather(parts, slab, group=plan.group, async_op=True)

    def finish():
        for r, p in enumerate(parts):
            full[r * plan.rows:(r + 1) * plan.rows] = p
    return _Pending(work, finish)


def all_gather_rows(slab: torch.Tensor, plan: ShardPlan) -> torch.Tensor:
    """slab [B, rows, N, H] -> [B, N, N, H]; one collective per sample keeps the [B, rows, ...] layout with no transpose pass"""
    B = slab.shape[0]
    full = slab.new_empty((B, plan.N) + tuple(slab.shape[2:]))
    slab = slab.contiguous()
    for p in [all_gather_rows_begin(slab[b], full[b], plan) for b in range(B)]:
        p.wait()
    return full


class _AllGatherRowsFn(torch.autograd.Function):
    """forward: all-gather the row slabs; backward: the incoming gradient is already complete on every rank (it comes out of an
    all-reduce), so each rank keeps the rows it owns."""

    @staticmethod
    def forward(ctx, slab, plan):
        ctx.plan = plan
        return all_gather_rows(slab, plan)

    @staticmethod
    def backward(ctx, d_full):
        p = ctx.plan
        return d_full[:, p.row_lo:p.row_hi].contiguous(), None


# ------------------------------------------------------------------------------------------------
# sharded BDGCN layers
# ------------------------------------------------------------------------------------------------
def _begin_forward(ctx, X, G_o, G_d, W, b, dynamic, act, precision, plan, grad_mode, samples):
    """The start of both sharded layer Functions' forward (inputs X, G_o, G_d, W, b, ...): resolve the precision for part calls of
    `samples` samples, make the operands fp32 and contiguous and note on ctx what backward needs.
    -> (prec, Xc, Goc, Gdc, Wc, bias, keep); keep: the forward stashes what backward reads.
    The part kernels have no dG stages: a support that requires grad would silently get none, whatever layer.support_grad says,
    so it is refused as ops.bdgcn refuses one without support_grad."""
    if grad_mode and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
        raise NotImplementedError("mpgcn_b200.shard: gradients with respect to the supports G exist for whole layers only "
                                  "(ops.bdgcn with support_grad=True); pass G.detach() to the sharded model")
    N, C = X.shape[2], X.shape[3]
    K, H = G_o.shape[-3], W.shape[1]
    prec = _ENGINE.resolve_precision(precision, samples, N, K, C, H)
    Xc, Goc, Wc = ops._f32c(X), ops._f32c(G_o), ops._f32c(W)
    Gdc = Goc if G_d is G_o else ops._f32c(G_d)
    keep = grad_mode and any(ctx.needs_input_grad)
    ctx.meta = (dynamic, act, prec, b is not None, N, K, C, H)
    ctx.keep, ctx.plan = keep, plan
    return prec, Xc, Goc, Gdc, Wc, None if b is None else ops._f32c(b), keep


def _begin_backward(ctx, d_out):
    """-> d_out as fp32 contiguous; refuses a backward through a forward that kept nothing"""
    if not ctx.keep:
        raise RuntimeError("mpgcn_b200.shard: backward called but forward ran without requires_grad inputs")
    return ops._f32c(d_out)


class _RowShardLayerFn(torch.autograd.Function):
    """Sample by sample, so that the exchange of sample b overlaps the contractions of sample b + 1 (forward: partial pre of b is
    reduce-scattered while b + 1 is computed; backward: every dPre slab is put on the wire up front and the gradient
    contractions of sample b start as soon as ITS rows have arrived)."""

    @staticmethod
    def forward(ctx, X, G_o, G_d, W, b, dynamic, act, precision, plan, branch, grad_mode):
        prec, Xc, Goc, Gdc, Wc, bias, keep = _begin_forward(ctx, X, G_o, G_d, W, b, dynamic, act, precision, plan, grad_mode, 1)
        N, K, C, H = ctx.meta[4:]
        B, rows = X.shape[:2]
        if plan.peer is not None:
            # peer-memory exchange: the whole batch in one part call, partial written straight into the symmetric buffer,
            # one barrier, then the reduce-scatter + bias + ReLU kernel reads this rank's rows from every rank's buffer
            buf, hdl = plan.peer.next(("fwd", branch), (B, N, N, H))
            ctx.branch = branch
            planes = (B if dynamic else 1) * K
            go_p = _ENGINE.prepared(G_o, Goc, planes, N, prec)
            preps = (go_p, go_p if G_d is G_o else _ENGINE.prepared(G_d, Gdc, planes, N, prec))
            ctx.preps = preps
            _, saved = _ENGINE.forward_part(Xc, Goc, Gdc, dynamic, Wc, N, plan.row_lo, K, K, prec, keep, out=buf, preps=preps)
            hdl.barrier()
            out = _ENGINE.rows_reduce_bias_act(list(hdl.buffer_ptrs), B, N, plan.row_lo, rows, H, bias, act, X.device)
            ctx.stash = [saved]
            ctx.save_for_backward(out, Goc, Gdc, Wc)
            return out
        out = torch.empty((B, rows, N, H), dtype=torch.float32, device=X.device)
        pending, stash = [], []
        for s in range(B):
            go_s, gd_s = (Goc[s:s + 1], Gdc[s:s + 1]) if dynamic else (Goc, Gdc)
            partial, saved = _ENGINE.forward_part(Xc[s:s + 1], go_s, gd_s, dynamic, Wc, N, plan.row_lo, K, K, prec, keep)
            pending.append((reduce_scatter_rows_begin(partial[0], out[s], plan), partial))      # the ONE exchange step of the layer forward
            stash.append(saved)
        for p, _ in pending:
            p.wait()
        del pending
        _ENGINE.bias_act(out, bias, act)
        ctx.stash = stash
        ctx.save_for_backward(out, Goc, Gdc, Wc)
        return out

    @staticmethod
    def backward(ctx, d_out):
        d_out = _begin_backward(ctx, d_out)
        out, Goc, Gdc, Wc = ctx.saved_tensors
        dynamic, act, prec, has_bias, N, K, C, H = ctx.meta
        plan = ctx.plan
        B = d_out.shape[0]
        if plan.peer is not None:
            if prec == _lib.PREC_FP16_TC:
                # tensor-core path: the gathered dPre travels as fp16 (what the contraction reads anyway), scaled by ONE power of two
                # derived from the global max|dOut| -- half the bytes, and no rank casts / scans the gathered tensor
                amax = _ENGINE.absmax(d_out)
                dist.all_reduce(amax, op=dist.ReduceOp.MAX, group=plan.group)
                d_pre16, hdl = plan.peer.next(("bwd16", ctx.branch), (B, N, N, H), torch.float16)
                db, scale2 = _ENGINE.relu_backward_scatter_f16(d_out, out, act, list(hdl.buffer_ptrs), N, plan.row_lo, has_bias, amax)
                hdl.barrier()
                dX, dW = _ENGINE.backward_part(None, Goc, Gdc, dynamic, Wc, ctx.stash[0], N, plan.row_lo, plan.rows, K, K, C, prec,
                                               ctx.needs_input_grad[0], preps=ctx.preps, d_pre16=d_pre16, scale2=scale2)
            else:
                d_pre, hdl = plan.peer.next(("bwd", ctx.branch), (B, N, N, H))
                db = _ENGINE.relu_backward_scatter(d_out, out, act, list(hdl.buffer_ptrs), N, plan.row_lo, has_bias)
                hdl.barrier()
                dX, dW = _ENGINE.backward_part(d_pre, Goc, Gdc, dynamic, Wc, ctx.stash[0], N, plan.row_lo, plan.rows, K, K, C, prec,
                                               ctx.needs_input_grad[0])
            ctx.stash = None
            ctx.preps = None
            return dX, None, None, dW, db, None, None, None, None, None, None
        d_pre_slab, db = _ENGINE.relu_backward(d_out, out, act, has_bias)       # mask + bias gradient of the rank's own rows
        d_pre = d_pre_slab.new_empty((B, N, N, H))
        pending = [all_gather_rows_begin(d_pre_slab[s], d_pre[s], plan) for s in range(B)]     # the ONE exchange step of the layer backward
        need_dx = ctx.needs_input_grad[0]
        dX = torch.empty((B, plan.rows, N, C), dtype=torch.float32, device=d_out.device) if need_dx else None
        dW = None
        for s in range(B):
            pending[s].wait()
            go_s, gd_s = (Goc[s:s + 1], Gdc[s:s + 1]) if dynamic else (Goc, Gdc)
            dx_s, dw_s = _ENGINE.backward_part(d_pre[s:s + 1], go_s, gd_s, dynamic, Wc, ctx.stash[s], N, plan.row_lo, plan.rows, K, K, C, prec, need_dx)
            if need_dx:
                dX[s:s + 1] = dx_s
            dW = dw_s if dW is None else dW + dw_s
        ctx.stash = None
        return dX, None, None, dW, db, None, None, None, None, None, None


class _KShardLayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X, G_o, G_d, W, b, dynamic, act, precision, plan, branch, grad_mode):
        prec, Xc, Goc, Gdc, Wc, bias, keep = _begin_forward(ctx, X, G_o, G_d, W, b, dynamic, act, precision, plan, grad_mode, X.shape[0])
        N, K, C, H = ctx.meta[4:]
        Kd = plan.Kd
        saved = Wl = None
        if Kd > 0:
            Wl = Wc.view(K, K, C, H)[:, plan.d_lo:plan.d_hi].reshape(K * Kd * C, H).contiguous()
            pre, saved = _ENGINE.forward_part(Xc, Goc, Gdc, dynamic, Wl, N, 0, K, Kd, prec, keep)
        else:               # more ranks than supports: this rank only takes part in the exchange
            pre = torch.zeros((X.shape[0], N, N, H), dtype=torch.float32, device=X.device)
        dist.all_reduce(pre, group=plan.group)                   # the ONE exchange step of the layer forward
        _ENGINE.bias_act(pre, bias, act)
        empty = torch.empty(0, device=X.device)
        ctx.save_for_backward(pre, Goc, Gdc, Wl if Wl is not None else empty, saved if saved is not None else empty)
        return pre

    @staticmethod
    def backward(ctx, d_out):
        d_out = _begin_backward(ctx, d_out)
        out, Goc, Gdc, Wl, saved = ctx.saved_tensors
        dynamic, act, prec, has_bias, N, K, C, H = ctx.meta
        plan = ctx.plan
        d_pre, db = _ENGINE.relu_backward(d_out, out, act, has_bias)            # replicated: identical on every rank
        dW = torch.zeros((K, K, C, H), dtype=torch.float32, device=d_out.device)
        need_dx = ctx.needs_input_grad[0]
        if plan.Kd > 0:
            dX, dWl = _ENGINE.backward_part(d_pre, Goc, Gdc, dynamic, Wl, saved, N, 0, N, K, plan.Kd, C, prec, need_dx)
            dW[:, plan.d_lo:plan.d_hi] = dWl.view(K, plan.Kd, C, H)
        else:
            dX = torch.zeros((d_out.shape[0], N, N, C), dtype=torch.float32, device=d_out.device) if need_dx else None
        if need_dx:
            dist.all_reduce(dX, group=plan.group)                # the ONE exchange step of the layer backward
        if db is not None:
            db = db / plan.world          # replicated quantity: the parameter-gradient exchange SUMS over the ranks
        return dX, None, None, dW.view(K * K * C, H), db, None, None, None, None, None, None


def sharded_bdgcn(layer, X, G, plan: ShardPlan, branch: int = 0):
    """One BDGCN layer (mpgcn_b200.MPGCN.BDGCN: parameters W, b; activation None or ReLU) on this rank's shard.
    row: X [B,rows,N,C] -> [B,rows,N,H];  k: X [B,N,N,C] -> [B,N,N,H] (replicated).
    G: the whole static [K,N,N] stack, or the dynamic pair (G_o [B,K,N,N], G_d) with G_d whole (row shard) or the rank's slice
    [B,Kd,N,N] (K shard, shard_host_inputs).  `branch`: the model branch, whose pair of peer-exchange buffers the row shard uses."""
    act = layer.fused_act()
    if act is None:
        raise NotImplementedError("sharded layers fuse None / ReLU only")
    _no_deterministic("sharded_bdgcn")
    if any(g.layout != torch.strided for g in ((G,) if isinstance(G, torch.Tensor) else G)):
        raise NotImplementedError("sharded layers take dense supports; a sparse stack runs on one GPU (mpgcn_b200.ops.bdgcn)")
    dynamic = not isinstance(G, torch.Tensor)
    if dynamic:
        G_o, G_d = G
    else:           # the K shard contracts the destination side over its own supports only
        G_o, G_d = G, (G[plan.d_lo:plan.d_hi] if plan.kind == "k" else G)
    fn = _RowShardLayerFn if plan.kind == "row" else _KShardLayerFn
    return fn.apply(X, G_o, G_d, layer.W, layer.b if layer.use_bias else None, dynamic, act, layer.precision, plan, branch,
                    torch.is_grad_enabled())


# ------------------------------------------------------------------------------------------------
# the model on a shard  (reference MPGCN.forward, MPGCN.py:89-112)
# ------------------------------------------------------------------------------------------------
def shard_host_inputs(plan: ShardPlan, x_seq, y_true, g_o, g_d):
    """This rank's slices of the step inputs (host side; pinned like their sources).
    x_seq [B,T,N,N,1] -> its origin rows (the LSTM is row-local in both shards); y [B,1,N,N,1] -> its rows (row shard; the K
    shard's head is replicated and keeps all of y); dynamic G_o stays whole (every rank contracts over its own rows of every
    support / over all of them); G_d [B,K,N,N] -> the rank's destination supports (K shard)."""
    def pin(t):
        t = t.contiguous()
        return t.pin_memory() if torch.cuda.is_available() else t
    lo, hi = plan.row_lo, plan.row_hi
    x = pin(x_seq[:, :, lo:hi])
    if plan.kind == "row":
        return x, pin(y_true[:, :, lo:hi]), g_o, g_d
    return x, y_true, g_o, pin(g_d[:, plan.d_lo:plan.d_hi])


def sharded_forward(model, plan: ShardPlan, x_slab, G_static, G_dyn):
    """model: mpgcn_b200.MPGCN.MPGCN, run through its own forward with the LSTM and the layers on this rank's shard.
    x_slab [B,T,rows,N,1] (shard_host_inputs).  G_static [K,N,N] (whole, on every rank);
    G_dyn = (G_o [B,K,N,N], G_d) with G_d whole (row shard) or the rank's slice [B,Kd,N,N] (K shard).
    -> row shard: y of the rank's rows [B,1,rows,N,1];  K shard: the whole y [B,1,N,N,1] on every rank."""
    assert len(model.branch_models) == 2 == model.M, "the trainer's M = 2 layout: static branch, dynamic branch"

    def temporal(lstm, x):
        B, _, rows, N, _ = x.shape
        # (the option is passed only when set, so an engine without it -- the CPU stand-ins of the tests -- is called as before)
        extra = {"recompute": model.lstm_recompute} if getattr(model, "lstm_recompute", None) else {}
        h = _ENGINE.lstm_last(x, lstm, model.lstm_precision, **extra).reshape(B, rows, N, model.lstm_hidden_dim)
        return h if plan.kind == "row" else _AllGatherRowsFn.apply(h, plan)

    # The branches are independent until the head: each runs on its own CUDA stream, so that the exchange steps of one branch
    # (NVLink-bound kernels that leave the SMs mostly idle) overlap the contractions of the other.  autograd replays every
    # backward node on the stream of its forward, so the backward overlaps the same way.  The head is row-local.
    run = BranchRunner(temporal, lambda layer, X, G, m: sharded_bdgcn(layer, X, G, plan, m), _ENGINE.head, streams=True)
    return model._forward(x_slab, [G_static, G_dyn], plan.rows, run)


def sharded_mse_loss(plan: ShardPlan, y_pred, y_true):
    """nn.MSELoss(reduction='mean') (Model_Trainer.py:64,108) of the WHOLE prediction.  Row shard: each rank holds its rows; the value
    returned is the rank's share sum((y - t)^2) / (B*N*N), whose gradients are exactly the rank's part of the global gradient
    (sum the returned values over the ranks for the loss itself).  K shard: y is replicated, plain MSE."""
    if plan.kind == "row":
        total = y_pred.shape[0] * plan.N * plan.N * y_pred.shape[-1]
        return ((y_pred - y_true) ** 2).sum() / total
    return torch.nn.functional.mse_loss(y_pred, y_true)


def allreduce_sum_gradients(params, plan: ShardPlan = None, model=None, over_world: bool = False, scale: float = 1.0) -> int:
    """ONE all-reduce (sum) of every parameter gradient on a flat buffer.  Row shard: all gradients are partial sums over the
    rank's cells.  K shard: dW slices are disjoint (zeros elsewhere), db was pre-divided, the LSTM is row-sharded; only the
    replicated head's gradients must be divided by the number of ranks first (pass `model`).
    Hybrid (row groups x batch shard): over_world=True reduces over ALL ranks and `scale` = 1 / number of groups turns the sum of
    the groups' mean-loss gradients into the gradient of the global mean."""
    params = list(params)
    if not (dist.is_available() and dist.is_initialized()) or not params:
        return 0
    group = None if over_world else (plan.group if plan is not None else None)
    world = dist.get_world_size(group)
    if world == 1:
        return 0
    if plan is not None and plan.kind == "k" and model is not None:
        for m in range(model.M):
            for p in model.branch_models[m]['fc'].parameters():
                if p.grad is not None:
                    p.grad.div_(plan.world)
    flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in params])
    dist.all_reduce(flat, group=group)
    if scale != 1.0:
        flat.mul_(scale)
    off = 0
    for p in params:
        n = p.numel()
        g = flat[off:off + n].view_as(p)
        if p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)
        off += n
    return off
