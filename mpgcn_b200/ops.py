"""Autograd-aware operators of the hot path, each a thin call into the C ABI.

    bdgcn(X, G, W, b, activation)  <->  reference BDGCN.forward           (MPGCN.py:24-50), dL/dG too with support_grad=True;
                                        a sparse COO static G runs the gathers over its nonzeros (DESIGN.md section 12)
    lstm_last(x_seq, w_ih, w_hh, b_ih, b_hh)  <->  nn.LSTM(...)[:, -1, :]  (MPGCN.py:69,100-104)
    lstm_stack(x_seq, params, precision)      <->  the same with num_layers = L >= 2
    lstm_module_last(lstm, x_seq, precision)  <->  either of them, or the module itself where the engine has no kernel
                                                  (each takes `recompute`: keep no LSTM training state, rebuild it in the backward)

PyTorch supplies device memory, the current stream and the autograd tape; all arithmetic is in
libmpgcn_b200.so.
"""
from __future__ import annotations

import collections
import os

import torch

from . import _lib

_PREC_NAMES = {"fp32": _lib.PREC_FP32, "fp16": _lib.PREC_FP16_TC, "auto": -1}

# bytes of training state (Z stash, LSTM c_t/h_t, head pre-activations) allocated by forward calls since the last .clear():
# stays at zero under torch.no_grad() (tests/test_gpu_at_size.py::test_no_grad_allocates_no_training_state)
STASH_BYTES = collections.Counter()


def default_precision() -> str:
    """'auto' (tensor cores whenever the shape allows), 'fp16' or 'fp32'.  Env: MPGCN_B200_PRECISION."""
    return os.environ.get("MPGCN_B200_PRECISION", "auto")


def resolve_precision(name, B, N, K, C, H) -> int:
    name = default_precision() if name is None else name
    if name not in _PREC_NAMES:
        raise ValueError(f"unknown precision {name!r}; expected one of {sorted(_PREC_NAMES)}")
    lib = _lib.load()
    if name == "auto":
        return _lib.PREC_FP16_TC if lib.mpgcn_bdgcn_precision_supported(B, N, K, C, H, _lib.PREC_FP16_TC) else _lib.PREC_FP32
    code = _PREC_NAMES[name]
    if not lib.mpgcn_bdgcn_precision_supported(B, N, K, C, H, code):
        raise RuntimeError(f"precision {name!r} does not support B={B} N={N} K={K} C={C} H={H} (tensor path needs C and H to be multiples of 32, from C == H == 32 up, H <= 1024)")
    return code


def _require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"mpgcn_b200: {what} must be a CUDA tensor (got device {t.device}); the engine has no CPU path")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(dtype=torch.float32).contiguous()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _scratch(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


# Gradient-magnitude hand-over between consecutive backward calls of the fp16 path: the kernel that writes a gradient tensor also
# records max|grad| in a device scalar, and the backward that receives that tensor reuses it for its power-of-two scaling
# instead of re-reading the tensor.  The hand-over follows the autograd graph, not memory addresses: at forward time a consumer
# (BDGCN layer, FC head) notes which of OUR autograd nodes produced its input (looking through pure view nodes only); at
# backward time it leaves (data_ptr, version, numel, scalar) of the gradient it wrote ON that node, and the node's backward
# accepts the hint only if the gradient it receives is that very memory, unmodified (gradient accumulation from a second
# consumer arrives in a different buffer or with a bumped version).  Purely an optimisation: a missed hint costs one pass.
_VIEW_NODES = ("ViewBackward", "UnsafeViewBackward", "ReshapeAliasBackward", "AliasBackward")
_OUR_NODES = ("_BDGCNFnBackward", "_LSTMLastFnBackward", "_LSTMStackFnBackward")


def _producer_node(t):
    node = getattr(t, "grad_fn", None)
    for _ in range(8):
        if node is None:
            return None
        name = type(node).__name__
        if name in _OUR_NODES:
            return node
        if not name.startswith(_VIEW_NODES) or len(node.next_functions) != 1:
            return None
        node = node.next_functions[0][0]
    return None


def _put_hint(node, grad, absmax_scalar):
    if node is not None and grad is not None and absmax_scalar is not None:
        node._mpgcn_hint = (grad.data_ptr(), grad._version, grad.numel(), absmax_scalar)


def _take_hint(node, grad):
    e = getattr(node, "_mpgcn_hint", None)
    if e is None:
        return None
    node._mpgcn_hint = None
    return e[3] if (e[0] == grad.data_ptr() and e[1] == grad._version and e[2] == grad.numel()) else None


# Supports staged once: the same G_o / G_d serve every layer of a branch, forward and backward (6 calls per training step),
# so their fp16 conversion (+ diagonal remainders) -- or, for a sparse stack, its CSR / CSC structure -- is cached per support
# TENSOR OBJECT.  An entry is valid only while that very object is alive (weak reference), unmodified (version counter), at the
# same address (a sparse stack: of its values) and used on the same stream.
_SUPPORT_CACHE = {}
_SPARSE_CACHE = {}
_SUPPORT_CACHE_MAX = 8


def _cached(cache, G, ptr: int, make):
    import weakref
    key = id(G)
    stream = _stream()
    e = cache.get(key)
    if e is not None:
        ref, ver, p, st, dev, val = e
        if ref() is G and ver == G._version and p == ptr and st == stream and dev == G.device:
            return val
        del cache[key]
    for k in [k for k, v in cache.items() if v[0]() is None]:      # supports that no longer exist: free their staging now
        del cache[k]
    while len(cache) >= _SUPPORT_CACHE_MAX:
        cache.pop(next(iter(cache)))
    val = make(stream)
    try:
        cache[key] = (weakref.ref(G), G._version, ptr, stream, G.device, val)
    except TypeError:        # not weak-referenceable: do not cache
        pass
    return val


def _prepared_supports(lib, G, Gc, planes: int, N: int):
    def make(stream):
        nbytes = lib.mpgcn_bdgcn_supports_prepared_bytes(planes, N)
        blob = torch.empty(nbytes, dtype=torch.uint8, device=Gc.device)
        with torch.cuda.device(Gc.device):
            _lib.check(lib.mpgcn_bdgcn_prepare_supports(_ptr(Gc), _ptr(blob), nbytes, planes, N, stream), "bdgcn_prepare_supports")
        return blob
    return _cached(_SUPPORT_CACHE, G, Gc.data_ptr(), make)


def _sparse_supports(lib, G, K: int, N: int):
    """(structure, nnz) of a sparse COO stack [K,N,N]: CSR and CSC of every support, built on the device (mpgcn_sparse_supports_build)
    from the coalesced tensor, so that duplicate entries add up as in the dense sum."""
    def make(stream):
        Gc = G.detach()
        if not Gc.is_coalesced():
            Gc = Gc.coalesce()
        idx = Gc._indices().contiguous()
        val = Gc._values().to(torch.float32).contiguous()
        nnz = val.numel()
        nbytes = lib.mpgcn_sparse_supports_bytes(K, N, nnz)
        if nbytes == 0:
            raise RuntimeError(f"mpgcn_b200.bdgcn: a sparse support stack holds {nnz} nonzeros; its int32 indices take fewer than 2^31")
        blob = torch.empty(nbytes, dtype=torch.uint8, device=G.device)
        with torch.cuda.device(G.device):
            _lib.check(lib.mpgcn_sparse_supports_build(_ptr(idx), _ptr(val), nnz, K, N, _ptr(blob), nbytes, stream), "sparse_supports_build")
        return blob, nnz
    return _cached(_SPARSE_CACHE, G, G._values().data_ptr(), make)


class _BDGCNFn(torch.autograd.Function):
    @staticmethod
    @_lib.engine_buffers()
    def forward(ctx, X, G_o, G_d, W, b, dynamic: bool, act: int, precision, grad_mode: bool, support_grad: bool):
        import ctypes
        lib = _lib.load()
        B, N, N2, C = X.shape
        K = G_o.shape[-3]
        H = W.shape[1]
        sparse = G_o.layout == torch.sparse_coo          # bdgcn() checked it: static, fp32 family, no gradient
        prec = _lib.PREC_FP32 if sparse else resolve_precision(precision, B, N, K, C, H)
        tc = prec == _lib.PREC_FP16_TC
        Xc, Wc = _f32c(X), _f32c(W)
        Goc = torch.empty(0, device=X.device) if sparse else _f32c(G_o)
        Gdc = Goc if G_d is G_o else _f32c(G_d)
        bc = None if b is None else _f32c(b)
        out = torch.empty((B, N, N, H), dtype=torch.float32, device=X.device)
        # ctx.needs_input_grad ignores the grad mode (it is True under torch.no_grad() too), and inside Function.forward
        # torch.is_grad_enabled() is always False: the wrapper reads the mode and hands it in.  Validation / test / the
        # autoregressive rollout therefore allocate no Z stash.
        need_grad = grad_mode and any(ctx.needs_input_grad)
        saved = _scratch(lib.mpgcn_bdgcn_saved_bytes(B, N, K, C, H, prec), X.device) if need_grad else None
        STASH_BYTES["bdgcn"] += saved.numel() if saved is not None else 0
        ws_bytes = lib.mpgcn_bdgcn_fwd_workspace_bytes(B, N, K, C, H, int(dynamic), prec)
        ws = _scratch(ws_bytes, X.device)
        ex = _lib.BdgcnExtras()
        preps = (None, None)
        if tc:
            # (The extras also allow handing an fp16 copy of the activation from layer to layer -- x_f16 / out_f16: the FWD_B
            # epilogue then writes that copy instead of a separate cast pass reading the fp32 activation.)
            planes = (B if dynamic else 1) * K
            with torch.cuda.device(X.device):
                go_p = _prepared_supports(lib, G_o, Goc, planes, N)
                gd_p = go_p if G_d is G_o else _prepared_supports(lib, G_d, Gdc, planes, N)
            preps = (go_p, gd_p)
            ex.go_prepared, ex.gd_prepared = _ptr(go_p), _ptr(gd_p)
        ctx.sparse_nnz = None
        with torch.cuda.device(X.device):
            if sparse:      # the stack's CSR / CSC (built once per tensor) travel as the first prepared-supports entry
                sp, ctx.sparse_nnz = _sparse_supports(lib, G_o, K, N)
                preps = (sp, None)
                _lib.check(lib.mpgcn_bdgcn_forward_sparse(_ptr(Xc), _ptr(sp), sp.numel(), ctx.sparse_nnz, _ptr(Wc), _ptr(bc), act, _ptr(out),
                                                          _ptr(saved), _ptr(ws), ws.numel(), B, N, K, C, H, _stream()), "bdgcn_forward_sparse")
            else:
                _lib.check(lib.mpgcn_bdgcn_forward_x(_ptr(Xc), _ptr(Goc), _ptr(Gdc), int(dynamic), _ptr(Wc), _ptr(bc), act, _ptr(out),
                                                     _ptr(saved), _ptr(ws), ws.numel(), B, N, K, C, H, prec, ctypes.addressof(ex), _stream()),
                           "bdgcn_forward")
        ctx.shape = (B, N, K, C, H)
        ctx.meta = (bool(dynamic), act, prec, b is not None)
        ctx.x_producer = _producer_node(X) if need_grad else None
        ctx.preps = preps
        # the support gradient reads X (dG_d = sum X Y_d): kept only when a support asks for its gradient
        ctx.sgrad = need_grad and support_grad and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2])
        empty = torch.empty(0, device=X.device)
        ctx.save_for_backward(out, Goc, Gdc, Wc, saved if saved is not None else empty, Xc if ctx.sgrad else empty)
        return out

    @staticmethod
    @_lib.engine_buffers()
    def backward(ctx, d_out):
        import ctypes
        lib = _lib.load()
        _lib.sync_deterministic()       # this thread's mode, before the workspace query (autograd's device thread: set it here)
        out, Goc, Gdc, Wc, saved, Xc = ctx.saved_tensors
        B, N, K, C, H = ctx.shape
        dynamic, act, prec, has_bias = ctx.meta
        if saved.numel() == 0:
            raise RuntimeError("mpgcn_b200.bdgcn: backward called but forward ran without requires_grad inputs")
        tc = prec == _lib.PREC_FP16_TC
        hint = _take_hint(ctx, d_out) if (tc and d_out.dtype == torch.float32 and d_out.is_contiguous()) else None
        d_out = _f32c(d_out)
        dev = d_out.device
        need_dx = ctx.needs_input_grad[0]
        dX = torch.empty((B, N, N, C), dtype=torch.float32, device=dev) if need_dx else None
        dx_absmax = torch.empty(1, dtype=torch.float32, device=dev) if (need_dx and tc) else None
        dW = torch.empty_like(Wc)
        db = torch.empty(H, dtype=torch.float32, device=dev) if has_bias else None
        ex = _lib.BdgcnExtras()
        ex.go_prepared, ex.gd_prepared = _ptr(ctx.preps[0]), _ptr(ctx.preps[1])
        ex.d_out_absmax, ex.dX_absmax = _ptr(hint), _ptr(dx_absmax)
        dGo = dGd = None
        if ctx.sparse_nnz is not None:
            sp = ctx.preps[0]
            ws = _scratch(lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, 0, prec), dev)
            with torch.cuda.device(dev):
                _lib.check(lib.mpgcn_bdgcn_backward_sparse(_ptr(d_out), _ptr(out), _ptr(sp), sp.numel(), ctx.sparse_nnz, _ptr(Wc), act,
                                                           _ptr(saved), _ptr(dX), _ptr(dW), _ptr(db), _ptr(ws), ws.numel(), B, N, K, C, H,
                                                           _stream()), "bdgcn_backward_sparse")
        elif ctx.sgrad:
            # static: one gradient for the one stack (returned for G_o; G_d is the same tensor); dynamic: one per side, which
            # autograd adds up when the caller passed one tensor as both
            if not dynamic:
                dGo = torch.empty((K, N, N), dtype=torch.float32, device=dev)
            else:
                dGo = torch.empty((B, K, N, N), dtype=torch.float32, device=dev) if ctx.needs_input_grad[1] else None
                dGd = torch.empty((B, K, N, N), dtype=torch.float32, device=dev) if ctx.needs_input_grad[2] else None
            ws = _scratch(lib.mpgcn_bdgcn_support_grad_workspace_bytes(B, N, K, C, H, int(dynamic), prec), dev)
            with torch.cuda.device(dev):
                _lib.check(lib.mpgcn_bdgcn_backward_supports(_ptr(d_out), _ptr(out), _ptr(Goc), _ptr(Gdc), int(dynamic), _ptr(Wc), act,
                                                             _ptr(saved), _ptr(dX), _ptr(dW), _ptr(db), _ptr(ws), ws.numel(), B, N, K, C,
                                                             H, prec, ctypes.addressof(ex), _ptr(Xc), _ptr(dGo), _ptr(dGd), _stream()),
                           "bdgcn_backward_supports")
        else:
            ws = _scratch(lib.mpgcn_bdgcn_bwd_workspace_bytes(B, N, K, C, H, int(dynamic), prec), dev)
            with torch.cuda.device(dev):
                _lib.check(lib.mpgcn_bdgcn_backward_x(_ptr(d_out), _ptr(out), _ptr(Goc), _ptr(Gdc), int(dynamic),
                                                      _ptr(Wc), act, _ptr(saved), _ptr(dX), _ptr(dW), _ptr(db), _ptr(ws), ws.numel(), B, N, K,
                                                      C, H, prec, ctypes.addressof(ex), _stream()), "bdgcn_backward")
        _put_hint(ctx.x_producer, dX, dx_absmax)
        return dX, dGo, dGd, dW, db, None, None, None, None, None


def _check_sparse_supports(G, precision, grad_mode: bool) -> None:
    """A sparse static stack runs the sparse fp32 kernels: a COO tensor [K,N,N] of a floating type, with no dense dimensions and no
    gradient, under precision "auto" or "fp32"."""
    if G.layout != torch.sparse_coo:
        raise NotImplementedError(f"mpgcn_b200.bdgcn: sparse supports must be a sparse COO tensor (G.to_sparse()), got layout {G.layout}")
    if G.dense_dim() != 0 or G.sparse_dim() != 3:
        raise ValueError(f"mpgcn_b200.bdgcn: a sparse support stack must be [K,N,N] with 3 sparse dimensions and no dense ones, got "
                         f"{G.sparse_dim()} sparse and {G.dense_dim()} dense")
    if not G.is_floating_point():
        raise ValueError(f"mpgcn_b200.bdgcn: sparse supports must hold floating-point values, got {G.dtype}")
    if grad_mode and G.requires_grad:
        raise NotImplementedError("mpgcn_b200.bdgcn: sparse supports have no gradient (support_grad needs a dense G); pass G.detach()")
    name = default_precision() if precision is None else precision
    if name not in _PREC_NAMES:
        raise ValueError(f"unknown precision {name!r}; expected one of {sorted(_PREC_NAMES)}")
    if name == "fp16":
        raise RuntimeError("mpgcn_b200.bdgcn: there are no fp16 sparse kernels; sparse supports run in fp32 (precision 'auto' or 'fp32')")


def bdgcn(X: torch.Tensor, G, W: torch.Tensor, b, relu: bool, precision=None, support_grad: bool = False) -> torch.Tensor:
    """out = act(cat_{o,d}(G_o^T X G_d) W + b); G is a [K,N,N] tensor or a pair of [B,K,N,N] tensors.

    support_grad=True: a G that requires grad receives dL/dG (static: one [K,N,N] gradient; dynamic: one per side of the pair).
    It adds 2 K B N^3 (C + H) flops to the backward, as much as its N^3 work without it, so it is opt-in: by default a G that
    requires grad is refused.

    A static G given as a sparse COO tensor [K,N,N] runs the fp32 layer with its four N^3 contractions replaced by gathers over
    the stored entries (precision "auto" or "fp32"; its CSR / CSC structure is built once per tensor and cached).  Only stored
    entries are multiplied, so a non-finite X does not leak through a zero of G as it does in the dense layer."""
    if isinstance(G, torch.Tensor):
        G_o = G_d = G
        dynamic = False
        if G.layout != torch.strided:
            _check_sparse_supports(G, precision, torch.is_grad_enabled())
    else:
        G_o, G_d = G
        dynamic = True
        if G_o.layout != torch.strided or G_d.layout != torch.strided:
            raise NotImplementedError("mpgcn_b200.bdgcn: sparse supports are static only; both members of a dynamic pair must be dense")
    _require_cuda(X, "X")
    for g in (G_o, G_d):
        _require_cuda(g, "G")
        if g.device != X.device:
            raise RuntimeError("mpgcn_b200: X and G must be on the same device")
    grad_mode = torch.is_grad_enabled()
    if grad_mode and (G_o.requires_grad or G_d.requires_grad) and not support_grad:
        # the reference's einsums would deliver dL/dG through autograd; the trainer never asks for it (static G is a plain
        # tensor, dynamic G comes from the data loader), and the dG stages double the layer's N^3 backward work: a support that
        # requires grad by accident is refused instead of silently paying for it (or silently getting None)
        raise NotImplementedError("mpgcn_b200.bdgcn: gradients with respect to the supports G are not implemented "
                                  "by default (pass G.detach(), or support_grad=True / BDGCN.support_grad = True to compute them)")
    return _BDGCNFn.apply(X, G_o, G_d, W, b, dynamic, 1 if relu else 0, precision, grad_mode, bool(support_grad))


# State budget of the recomputing LSTM backward with recompute=True: the chunk of cells whose rebuilt training state (and gate-
# gradient records, and a stack's gradient sequence) takes about this much.  A choice, not a tuned value: chunks of this size
# already fill every SM many times over, and it is small beside the state it replaces (tens of GB at N = 1000).
LSTM_RECOMPUTE_BUDGET_BYTES = 1 << 30


def _check_recompute(recompute) -> None:
    if not (recompute is None or isinstance(recompute, bool) or (isinstance(recompute, int) and recompute >= 1)):
        raise ValueError(f"recompute must be None, a bool or a positive number of cells per chunk, got {recompute!r}")


def lstm_recompute_chunk_cells(recompute, T, C, L) -> int:
    """Cells per chunk of the recomputing backward for `recompute` (None / False: 0, off; True: LSTM_RECOMPUTE_BUDGET_BYTES of
    workspace; an int: that many cells)."""
    if recompute is None or recompute is False:
        return 0
    if recompute is not True:
        return int(recompute)
    probe = 1 << 20        # the workspace is about linear in the chunk: size it from the query at one large chunk
    per = _lib.load().mpgcn_lstm_recompute_bwd_workspace_bytes(1, T, probe, C, L, probe, _lib.PREC_FP16_TC)
    if not per:
        raise RuntimeError(f"LSTM recompute: no tensor-core kernels for T={T}, hidden={C}, L={L}")
    return max(1, LSTM_RECOMPUTE_BUDGET_BYTES * probe // per)


def resolve_lstm_precision(name, T, C) -> int:
    name = default_precision() if name is None else name
    if name not in _PREC_NAMES:
        raise ValueError(f"unknown precision {name!r}; expected one of {sorted(_PREC_NAMES)}")
    lib = _lib.load()
    if name == "auto":
        return _lib.PREC_FP16_TC if lib.mpgcn_lstm_precision_supported(T, C, _lib.PREC_FP16_TC) else _lib.PREC_FP32
    code = _PREC_NAMES[name]
    if not lib.mpgcn_lstm_precision_supported(T, C, code):
        raise RuntimeError(f"LSTM precision {name!r} does not support T={T}, hidden={C} "
                           "(tensor path needs hidden 32, 96 or 128 and 1 <= T <= 256; fp32 path needs hidden <= 64 and a T whose "
                           "backward stash fits in shared memory, e.g. T <= 15 at hidden 64)")
    return code


def lstm_engine_supports(name, T, C) -> bool:
    """Whether `lstm_last` runs hidden size C over T steps at precision `name` (None / "auto" / "fp16" / "fp32").  "auto" resolves
    to the fp32 kernels whenever the tensor-core ones do not apply, so the resolved kernel itself is asked, not only the name."""
    try:
        code = resolve_lstm_precision(name, T, C)
    except RuntimeError:
        return False
    return bool(_lib.load().mpgcn_lstm_precision_supported(T, C, code))


class _LSTMLastFn(torch.autograd.Function):
    @staticmethod
    @_lib.engine_buffers()
    def forward(ctx, x_seq, w_ih, w_hh, b_ih, b_hh, precision, grad_mode: bool, recompute):
        lib = _lib.load()
        B, T = x_seq.shape[0], x_seq.shape[1]
        NN = x_seq[0, 0].numel()
        C = w_hh.shape[1]
        prec = resolve_lstm_precision(precision, T, C)
        xc = _f32c(x_seq)
        ws = [_f32c(t) for t in (w_ih, w_hh, b_ih, b_hh)]
        hT = torch.empty((B * NN, C), dtype=torch.float32, device=x_seq.device)
        # training: the forward keeps c_t / h_t of every step (fp16) so that the backward is one reverse walk -- unless the
        # backward is to rebuild them a chunk at a time (recompute; precision 0 keeps none anyway)
        train = grad_mode and any(ctx.needs_input_grad[:5])
        chunk = lstm_recompute_chunk_cells(recompute, T, C, 1) if (train and prec == _lib.PREC_FP16_TC) else 0
        nsave = lib.mpgcn_lstm_saved_bytes(B, T, NN, C, prec) if (train and not chunk) else 0
        saved = torch.empty(nsave, dtype=torch.uint8, device=x_seq.device) if nsave else None
        # (precision 0 and recompute keep no state, so count the request, not the buffer)
        STASH_BYTES["lstm"] += nsave if nsave else (1 if train else 0)
        with torch.cuda.device(x_seq.device):
            _lib.check(lib.mpgcn_lstm_last_forward_train(_ptr(xc), *[_ptr(t) for t in ws], _ptr(hT), _ptr(saved), nsave, B, T, NN, C, prec,
                                                         _stream()), "lstm_last_forward")
        ctx.dims = (B, T, NN, C, prec)
        ctx.lstm_saved = saved
        ctx.chunk = chunk
        ctx.save_for_backward(xc, *ws)
        return hT

    @staticmethod
    @_lib.engine_buffers()
    def backward(ctx, d_hT):
        lib = _lib.load()
        _lib.sync_deterministic()
        xc, w_ih, w_hh, b_ih, b_hh = ctx.saved_tensors
        B, T, NN, C, prec = ctx.dims
        hint = _take_hint(ctx, d_hT) if (prec == _lib.PREC_FP16_TC and d_hT.dtype == torch.float32 and d_hT.is_contiguous()) else None
        d_hT = _f32c(d_hT)
        dev = xc.device
        g_wih, g_whh = torch.empty_like(w_ih), torch.empty_like(w_hh)
        g_bih, g_bhh = torch.empty_like(b_ih), torch.empty_like(b_hh)
        d_x = torch.empty_like(xc) if ctx.needs_input_grad[0] else None
        if ctx.chunk:
            ws = _scratch(lib.mpgcn_lstm_recompute_bwd_workspace_bytes(B, T, NN, C, 1, ctx.chunk, prec), dev)
            with torch.cuda.device(dev):
                _lib.check(lib.mpgcn_lstm_backward_recompute(_ptr(xc), 1, *[_ptr_array([t]) for t in (w_ih, w_hh, b_ih, b_hh)], _ptr(d_hT),
                                                             *[_ptr_array([t]) for t in (g_wih, g_whh, g_bih, g_bhh)], _ptr(d_x), ctx.chunk,
                                                             _ptr(ws), ws.numel(), B, T, NN, C, prec, _ptr(hint), _stream()),
                           "lstm_backward_recompute")
            return d_x, g_wih, g_whh, g_bih, g_bhh, None, None, None
        saved = ctx.lstm_saved
        # with the forward's state in hand the backward needs its workspace minus the room for rebuilding that state
        ws_bytes = lib.mpgcn_lstm_bwd_workspace_bytes(B, T, NN, C, prec)
        ws = _scratch(ws_bytes - saved.numel() if saved is not None else ws_bytes, dev)
        with torch.cuda.device(dev):
            _lib.check(lib.mpgcn_lstm_last_backward_saved(_ptr(xc), _ptr(w_ih), _ptr(w_hh), _ptr(b_ih), _ptr(b_hh), _ptr(d_hT), _ptr(g_wih),
                                                          _ptr(g_whh), _ptr(g_bih), _ptr(g_bhh), _ptr(d_x), _ptr(saved),
                                                          saved.numel() if saved is not None else 0, _ptr(ws), ws.numel(), B, T, NN, C,
                                                          prec, _ptr(hint), _stream()), "lstm_last_backward")
        ctx.lstm_saved = None
        return d_x, g_wih, g_whh, g_bih, g_bhh, None, None, None


def lstm_last(x_seq: torch.Tensor, w_ih, w_hh, b_ih, b_hh, precision=None, recompute=None) -> torch.Tensor:
    """h_T of a 1-layer, input-size-1 LSTM run over every OD cell of x_seq [B,T,N,N,1] -> [B*N*N, C].
    recompute (tensor cores): True or a number of cells per chunk -> the training forward keeps no c_t / h_t and the backward
    rebuilds them a chunk at a time (lstm_recompute_chunk_cells); same h_T and dx, weight gradients up to fp32 summation order."""
    _require_cuda(x_seq, "x_seq")
    _check_recompute(recompute)
    return _LSTMLastFn.apply(x_seq, w_ih, w_hh, b_ih, b_hh, precision, torch.is_grad_enabled(), recompute)


def lstm_stack_supports(name, T, C, L) -> bool:
    """Whether `lstm_stack` runs L >= 2 layers of hidden size C over T steps at precision `name`: the tensor-core kernels at
    hidden 32 and 96 ("auto" or "fp16"); there are no fp32 stacked kernels."""
    name = default_precision() if name is None else name
    if name not in _PREC_NAMES:
        raise ValueError(f"unknown precision {name!r}; expected one of {sorted(_PREC_NAMES)}")
    code = _lib.PREC_FP16_TC if name == "auto" else _PREC_NAMES[name]
    return bool(_lib.load().mpgcn_lstm_stack_supported(T, C, L, code))


def lstm_runs_on_engine(lstm: torch.nn.LSTM, T: int, precision) -> bool:
    """Whether `lstm_module_last` runs this nn.LSTM module over T steps on the engine rather than calling the module itself.
    One layer: under "auto" wherever one of the engine's kernels applies; up to hidden 64 an explicit precision always goes
    to the engine, which refuses a shape it cannot run; above that the tensor-core kernel runs hidden 96 and 128.  L >= 2
    layers: the tensor-core kernels at hidden 32 and 96 (at 128 an upper layer's gate weights do not fit a CTA's shared
    memory, DESIGN.md 6.4), with no dropout between the layers in training; anything else stays with the module, as do
    modules the engine does not compute: without biases, bidirectional, projected, or not batch_first."""
    if lstm.input_size != 1 or not lstm.bias or lstm.bidirectional or lstm.proj_size or not lstm.batch_first:
        return False
    C, L = lstm.hidden_size, lstm.num_layers
    if L == 1:
        explicit = precision not in (None, "auto") and C <= 64
        return explicit or lstm_engine_supports(precision, T, C)
    if lstm.dropout > 0 and lstm.training:
        return False
    return lstm_stack_supports(precision, T, C, L)


def lstm_module_last(lstm: torch.nn.LSTM, x_seq: torch.Tensor, precision=None, recompute=None) -> torch.Tensor:
    """h_T of the top layer of `lstm` (batch_first, zero initial state) over every OD cell of x_seq [B,T,N,N,I] -> [B*N*N, C].
    recompute: as `lstm_last`; the module itself, where it runs, is unaffected."""
    B, T, N, N2, I = x_seq.shape
    L = lstm.num_layers
    if lstm_runs_on_engine(lstm, T, precision):
        if L == 1:
            return lstm_last(x_seq, lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0, precision=precision,
                             recompute=recompute)
        params = [getattr(lstm, f"{k}_l{l}") for l in range(L) for k in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        return lstm_stack(x_seq, params, recompute=recompute)
    # configurations without an engine kernel: input_dim > 1 (Model_Trainer.py:49-51 hard-codes input_dim=1), hidden sizes
    # above 64 other than 96 / 128, sequences longer than 256 steps above hidden 64, sequences whose fp32 backward does not fit
    # in shared memory (T > 15 at hidden 64, DESIGN.md 6.4), fp32 above 64, and stacks other than those above
    lstm_in = x_seq.permute(0, 2, 3, 1, 4).reshape(B * N * N2, T, I)
    return lstm(lstm_in)[0][:, -1, :]


def _ptr_array(ts):
    import ctypes
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


class _LSTMStackFn(torch.autograd.Function):
    @staticmethod
    @_lib.engine_buffers()
    def forward(ctx, grad_mode: bool, recompute, x_seq, *params):
        lib = _lib.load()
        B, T = x_seq.shape[0], x_seq.shape[1]
        NN = x_seq[0, 0].numel()
        L, C = len(params) // 4, params[1].shape[1]
        prec = _lib.PREC_FP16_TC
        xc = _f32c(x_seq)
        ps = [_f32c(t) for t in params]
        hT = torch.empty((B * NN, C), dtype=torch.float32, device=x_seq.device)
        # training: every layer keeps c_t / h_t of every step; inference keeps only the h sequence of the layer below (workspace),
        # and so does training with recompute (its backward rebuilds the state a chunk at a time)
        train = grad_mode and any(ctx.needs_input_grad[2:])
        chunk = lstm_recompute_chunk_cells(recompute, T, C, L) if train else 0
        need = train and not chunk
        saved = torch.empty(lib.mpgcn_lstm_stack_saved_bytes(B, T, NN, C, L, prec), dtype=torch.uint8, device=x_seq.device) if need else None
        STASH_BYTES["lstm"] += saved.numel() if saved is not None else (1 if chunk else 0)
        ws = None if need else _scratch(lib.mpgcn_lstm_stack_fwd_workspace_bytes(B, T, NN, C, L, prec), x_seq.device)
        with torch.cuda.device(x_seq.device):
            _lib.check(lib.mpgcn_lstm_stack_forward(_ptr(xc), L, *[_ptr_array(ps[k::4]) for k in range(4)], _ptr(hT), _ptr(saved),
                                                    saved.numel() if saved is not None else 0, _ptr(ws), ws.numel() if ws is not None else 0,
                                                    B, T, NN, C, prec, _stream()), "lstm_stack_forward")
        ctx.dims = (B, T, NN, C, L, prec)
        ctx.lstm_saved = saved
        ctx.chunk = chunk
        ctx.save_for_backward(xc, *ps)
        return hT

    @staticmethod
    @_lib.engine_buffers()
    def backward(ctx, d_hT):
        lib = _lib.load()
        _lib.sync_deterministic()
        xc, *ps = ctx.saved_tensors
        B, T, NN, C, L, prec = ctx.dims
        if ctx.lstm_saved is None and not ctx.chunk:
            raise RuntimeError("mpgcn_b200.lstm_stack: backward called but forward ran without requires_grad inputs")
        hint = _take_hint(ctx, d_hT) if (d_hT.dtype == torch.float32 and d_hT.is_contiguous()) else None
        d_hT = _f32c(d_hT)
        dev = xc.device
        grads = [torch.empty_like(p) for p in ps]
        d_x = torch.empty_like(xc) if ctx.needs_input_grad[2] else None
        if ctx.chunk:
            ws = _scratch(lib.mpgcn_lstm_recompute_bwd_workspace_bytes(B, T, NN, C, L, ctx.chunk, prec), dev)
            with torch.cuda.device(dev):
                _lib.check(lib.mpgcn_lstm_backward_recompute(_ptr(xc), L, *[_ptr_array(ps[k::4]) for k in range(4)], _ptr(d_hT),
                                                             *[_ptr_array(grads[k::4]) for k in range(4)], _ptr(d_x), ctx.chunk,
                                                             _ptr(ws), ws.numel(), B, T, NN, C, prec, _ptr(hint), _stream()),
                           "lstm_backward_recompute")
            return (None, None, d_x, *grads)
        saved = ctx.lstm_saved
        ws = _scratch(lib.mpgcn_lstm_stack_bwd_workspace_bytes(B, T, NN, C, L, prec), dev)
        with torch.cuda.device(dev):
            _lib.check(lib.mpgcn_lstm_stack_backward(_ptr(xc), L, *[_ptr_array(ps[k::4]) for k in range(4)], _ptr(d_hT),
                                                     *[_ptr_array(grads[k::4]) for k in range(4)], _ptr(d_x), _ptr(saved), saved.numel(),
                                                     _ptr(ws), ws.numel(), B, T, NN, C, prec, _ptr(hint), _stream()), "lstm_stack_backward")
        ctx.lstm_saved = None
        return (None, None, d_x, *grads)


def lstm_stack(x_seq: torch.Tensor, params, recompute=None) -> torch.Tensor:
    """h_T of the top layer of an L-layer, input-size-1 LSTM run over every OD cell of x_seq [B,T,N,N,1] -> [B*N*N, C];
    params: [w_ih, w_hh, b_ih, b_hh] of layer 0, then of layer 1, ... (nn.LSTM's *_l0, *_l1, ...).  Tensor cores only.
    recompute: as `lstm_last`."""
    _require_cuda(x_seq, "x_seq")
    if len(params) < 8 or len(params) % 4:
        raise ValueError(f"lstm_stack: expected 4 parameters per layer and at least 2 layers, got {len(params)}")
    if x_seq.dim() < 3 or (x_seq.dim() == 5 and x_seq.shape[-1] != 1):
        raise ValueError(f"lstm_stack: x_seq must be [B,T,N,N,1] (input size 1), got {tuple(x_seq.shape)}")
    C = params[1].shape[-1]
    for i, p in enumerate(params):
        l, k = divmod(i, 4)
        want = ((4 * C, 1 if l == 0 else C), (4 * C, C), (4 * C,), (4 * C,))[k]
        if tuple(p.shape) != want or not p.is_floating_point() or p.device != x_seq.device:
            raise ValueError(f"lstm_stack: parameter {i} (layer {l}) must be a float tensor of shape {want} on {x_seq.device}, "
                             f"got {tuple(p.shape)} {p.dtype} on {p.device}")
    _check_recompute(recompute)
    return _LSTMStackFn.apply(torch.is_grad_enabled(), recompute, x_seq, *params)


class _HeadFn(torch.autograd.Function):
    @staticmethod
    @_lib.engine_buffers()
    def forward(ctx, grad_mode, w, b, *gs):
        import ctypes
        lib = _lib.load()
        M = len(gs)
        C = gs[0].shape[-1]
        cells = gs[0].numel() // C
        gc = [_f32c(g) for g in gs]
        wc, bc = _f32c(w), _f32c(b)
        y = torch.empty(gs[0].shape[:-1] + (1,), dtype=torch.float32, device=gs[0].device)
        need = grad_mode and any(ctx.needs_input_grad)
        pre = torch.empty((M, cells), dtype=torch.float32, device=y.device) if need else None
        STASH_BYTES["head"] += pre.numel() * 4 if pre is not None else 0
        ptrs = (ctypes.c_void_p * M)(*[g.data_ptr() for g in gc])
        with torch.cuda.device(y.device):
            _lib.check(lib.mpgcn_head_forward(ptrs, _ptr(wc), _ptr(bc), _ptr(y), _ptr(pre), cells, C, M, _stream()), "head_forward")
        ctx.dims = (M, C, cells)
        ctx.g_producers = [_producer_node(g) for g in gs] if need else None
        ctx.save_for_backward(wc, pre if pre is not None else torch.empty(0, device=y.device), *gc)
        return y

    @staticmethod
    @_lib.engine_buffers()
    def backward(ctx, dy):
        import ctypes
        lib = _lib.load()
        wc, pre, *gc = ctx.saved_tensors
        M, C, cells = ctx.dims
        dy = _f32c(dy)
        if pre.numel() == 0:
            raise RuntimeError("mpgcn_b200.fc_relu_mean: backward called but forward ran without requires_grad inputs")
        dgs = [torch.empty_like(g) if ctx.needs_input_grad[3 + m] else None for m, g in enumerate(gc)]
        dw = torch.empty_like(wc)
        db = torch.empty(M, dtype=torch.float32, device=dy.device)
        ptrs = (ctypes.c_void_p * M)(*[g.data_ptr() for g in gc])
        dptrs = (ctypes.c_void_p * M)(*[(d.data_ptr() if d is not None else None) for d in dgs])
        amax = torch.empty(M, dtype=torch.float32, device=dy.device)
        with torch.cuda.device(dy.device):
            if _lib.sync_deterministic():      # fixed-order dw / db: the per-block partials need a workspace
                ws = _scratch(lib.mpgcn_head_backward_workspace_bytes(cells, C, M), dy.device)
                _lib.check(lib.mpgcn_head_backward_ex(ptrs, _ptr(wc), _ptr(pre), _ptr(dy), dptrs, _ptr(dw), _ptr(db), _ptr(amax), cells, C, M,
                                                      _ptr(ws), ws.numel(), _stream()), "head_backward_ex")
            else:
                _lib.check(lib.mpgcn_head_backward(ptrs, _ptr(wc), _ptr(pre), _ptr(dy), dptrs, _ptr(dw), _ptr(db), _ptr(amax), cells, C, M,
                                                   _stream()), "head_backward")
        for m, d in enumerate(dgs):
            _put_hint(ctx.g_producers[m], d, amax[m:m + 1])
        return (None, dw, db) + tuple(dgs)


def fc_relu_mean(gs, w, b) -> torch.Tensor:
    """(1/M) * sum_m relu(g_m @ w[m] + b[m]) for M branch activations g_m [..., C]; w [M, C], b [M] -> [..., 1].
    1 <= M <= 8 branches of one shape, C a multiple of 4 (the kernel reads float4s), all on one CUDA device."""
    gs = list(gs)
    M = len(gs)
    if not 1 <= M <= 8:
        raise ValueError(f"fc_relu_mean: 1 to 8 branches, got {M}")
    shape = tuple(gs[0].shape)
    if not shape or shape[-1] % 4 or shape[-1] == 0:
        raise ValueError(f"fc_relu_mean: branch activations must be [..., C] with C a multiple of 4, got {shape}")
    C = shape[-1]
    for m, g in enumerate(gs):
        if tuple(g.shape) != shape:
            raise ValueError(f"fc_relu_mean: branch {m} has shape {tuple(g.shape)}, branch 0 {shape}")
    if tuple(w.shape) != (M, C) or tuple(b.shape) != (M,):
        raise ValueError(f"fc_relu_mean: w must be {(M, C)} and b {(M,)} for {M} branches of width {C}, got {tuple(w.shape)} and {tuple(b.shape)}")
    dev = gs[0].device
    for what, t in [("w", w), ("b", b)] + [(f"branch {m}", g) for m, g in enumerate(gs)]:
        if t.device != dev:
            raise ValueError(f"fc_relu_mean: {what} is on {t.device}, branch 0 on {dev}")
    _require_cuda(gs[0], "branch activation")
    return _HeadFn.apply(torch.is_grad_enabled(), w, b, *gs)
