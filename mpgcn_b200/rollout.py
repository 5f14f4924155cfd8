"""Autoregressive multi-step forecast = the inner loop of the reference's `ModelTrainer.test`
(Model_Trainer.py:157-165): `pred_len` forward passes under no_grad, each feeding its own prediction back into the
observation window.  At the reference's real problem size (N = 47 prefectures) one forward is ~60 short kernels and the
loop is launch-bound, so the step (forward + window slide) is captured once in a CUDA graph and replayed
(SURVEY.md section 8(f) rank 3).  Results are identical to the eager loop: the same kernels run on the same buffers.
"""
from __future__ import annotations

import torch


def _eager(model, x_seq, G_list, pred_len):
    outs, cur = [], x_seq
    for _ in range(pred_len):
        step = model(x_seq=cur, G_list=G_list)
        cur = torch.cat([cur[:, 1:], step], dim=1)
        outs.append(step)
    return torch.cat(outs, dim=1)


def forecast(model, x_seq: torch.Tensor, G_list, pred_len: int, use_cuda_graph: bool = True) -> torch.Tensor:
    """x_seq (B, T, N, N, 1) -> (B, pred_len, N, N, 1).  `model` is an `mpgcn_b200.MPGCN` (or reference-shaped) module."""
    assert pred_len >= 1
    was_training = model.training
    model.eval()
    try:
        with torch.no_grad():
            if not (use_cuda_graph and x_seq.is_cuda and pred_len > 1):
                return _eager(model, x_seq, G_list, pred_len)
            static_x = x_seq.clone()
            side = torch.cuda.Stream(device=x_seq.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):               # warm-up: one-time function attributes, allocator pools
                for _ in range(2):
                    model(x_seq=static_x, G_list=G_list)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_y = model(x_seq=static_x, G_list=G_list)
                static_x.copy_(torch.cat([static_x[:, 1:], static_y], dim=1))
            static_x.copy_(x_seq)
            outs = []
            for _ in range(pred_len):
                graph.replay()
                outs.append(static_y.clone())
            return torch.cat(outs, dim=1)
    finally:
        model.train(was_training)


class _GraphedInference:
    """`model.forward` replacement installed by `install`: under torch.no_grad() in eval mode on CUDA, a call whose input
    shape and support tensors (identity + version) match the last captured call replays that CUDA graph -- copy x in,
    replay, clone y out -- and anything else (training, grad mode, new supports) falls through to / re-captures the
    normal forward.  `ModelTrainer.test` (Model_Trainer.py:157-165) calls the model `pred_len` times per batch with the
    same supports: one capture, pred_len - 1 replays; the window slide stays the trainer's own `torch.cat`."""

    def __init__(self, model):
        self.model = model
        self.eager = model.forward          # the bound, un-patched method
        self.key = None
        self.graph = self.static_x = self.static_y = self.keep = None
        self.captures = self.replays = 0

    @staticmethod
    def _flat(G_list):
        out = []
        for g in G_list:
            out.extend(g if isinstance(g, (tuple, list)) else [g])
        return out

    def __call__(self, x_seq, G_list):
        if torch.is_grad_enabled() or self.model.training or not x_seq.is_cuda:
            return self.eager(x_seq=x_seq, G_list=G_list)
        gs = self._flat(G_list)
        key = (tuple(x_seq.shape), x_seq.device, tuple((id(g), g._version, (g._values() if g.is_sparse else g).data_ptr()) for g in gs))
        if key != self.key:
            self.key = None
            self.graph = self.static_x = self.static_y = None
            static_x = x_seq.clone()
            side = torch.cuda.Stream(device=x_seq.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):               # warm-up outside the capture: function attributes, support staging
                self.eager(x_seq=static_x, G_list=G_list)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_y = self.eager(x_seq=static_x, G_list=G_list)
            self.graph, self.static_x, self.static_y, self.keep, self.key = graph, static_x, static_y, gs, key
            self.captures += 1
        self.static_x.copy_(x_seq)
        self.graph.replay()
        self.replays += 1
        return self.static_y.clone()


def install(model):
    """Opt-in: route the model's inference calls through a captured CUDA graph (see _GraphedInference).  Returns the model.
    `model.forward.captures / .replays` count what happened; `uninstall(model)` restores the plain forward."""
    if not isinstance(getattr(model, "forward", None), _GraphedInference):
        model.forward = _GraphedInference(model)
    return model


def uninstall(model):
    if isinstance(model.__dict__.get("forward"), _GraphedInference):
        del model.__dict__["forward"]
    return model
