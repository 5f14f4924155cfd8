"""A whole training step -- forward, loss, backward, optimizer update -- captured ONCE in a CUDA graph and replayed.

At the reference's real problem size (N = 47 prefectures, Data_Container_OD.py:16) one step of the hot path is ~120 kernels of a
few microseconds each: the GPU idles between launches and the step costs what the Python / launch overhead costs.  Shapes are static from step to step (`DataLoader(batch_size=...)`,
Model_Trainer.py:94-115 -- the last, smaller batch of an epoch simply runs eagerly), so the step is captured with its
inputs in fixed device buffers and replayed: copy the batch in, `graph.replay()`, read the loss.

    step = GraphedTrainStep(model, criterion, optimizer, example=(x_seq, y_true, G_static, (G_o, G_d)))
    loss = step(x_seq, y_true, G_o, G_d)          # same arithmetic, same kernels, one launch

What is captured is exactly `Model_Trainer.py:107-115`: `y_pred = model(x_seq=..., G_list=[G, (G_o, G_d)])`,
`loss = criterion(y_pred, y_true)`, `optimizer.zero_grad()`, `loss.backward()`, `optimizer.step()`.  The optimizer must be
capture-safe (`torch.optim.Adam(..., capturable=True)`; the trainer's `Model_Trainer.py:74-77` Adam takes that flag unchanged).
The support staging cache of `mpgcn_b200.ops` is cleared before the capture so that the fp16 conversion of the (per-batch)
dynamic supports is part of the graph.  The graph keeps the kernels of the torch.use_deterministic_algorithms setting in force at
capture (the fixed-order reductions or the atomic ones, DESIGN.md section 11): changing the flag later does not change a replay.
"""
from __future__ import annotations

import torch

from . import ops


class GraphedTrainStep:
    def __init__(self, model, criterion, optimizer, example, warmup: int = 3, branch_streams=None):
        """branch_streams: True -> the model's branches are captured on parallel streams (fork / join inside the graph): at
        launch-bound sizes the kernels of the two branches then run side by side; None -> leave `model.branch_streams` as it is."""
        if branch_streams is not None:
            model.branch_streams = bool(branch_streams)
        x, y, G_static, (g_o, g_d) = example
        if not x.is_cuda:
            raise RuntimeError("GraphedTrainStep needs CUDA tensors (the engine has no CPU path)")
        for group in optimizer.param_groups:
            if not group.get("capturable", False):
                raise ValueError("GraphedTrainStep: build the optimizer with capturable=True (e.g. torch.optim.Adam(params, lr, capturable=True))")
        self.model, self.criterion, self.optimizer = model, criterion, optimizer
        self.G_static = G_static
        self.x, self.y, self.g_o, self.g_d = (t.detach().clone() for t in (x, y, g_o, g_d))
        self.shapes = tuple(tuple(t.shape) for t in (self.x, self.y, self.g_o, self.g_d))
        side = torch.cuda.Stream(device=x.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):                   # eager warm-up on a side stream: attributes, allocator pools, Adam state
            for _ in range(warmup):
                self._step_body()
        torch.cuda.current_stream().wait_stream(side)
        ops._SUPPORT_CACHE.clear()                      # the staging of the supports must be INSIDE the graph (new G_o / G_d every batch)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss = self._step_body()
        ops._SUPPORT_CACHE.clear()
        self.replays = 0

    def _step_body(self):
        y_pred = self.model(x_seq=self.x, G_list=[self.G_static, (self.g_o, self.g_d)])
        loss = self.criterion(y_pred, self.y)
        self.optimizer.zero_grad(set_to_none=False)     # gradients live in fixed buffers across replays
        loss.backward()
        self.optimizer.step()
        return loss

    def matches(self, x, y, g_o, g_d) -> bool:
        return tuple(tuple(t.shape) for t in (x, y, g_o, g_d)) == self.shapes

    def __call__(self, x, y, g_o, g_d):
        """One training step on this batch; returns the loss (a device scalar that the next call overwrites -- `.item()` or
        clone it).  A batch of another shape (the last one of an epoch) runs the same step eagerly."""
        if not self.matches(x, y, g_o, g_d):
            keep = (self.x, self.y, self.g_o, self.g_d)
            self.x, self.y, self.g_o, self.g_d = x, y, g_o, g_d
            try:
                return self._step_body().detach()
            finally:
                self.x, self.y, self.g_o, self.g_d = keep
        self.x.copy_(x, non_blocking=True)
        self.y.copy_(y, non_blocking=True)
        self.g_o.copy_(g_o, non_blocking=True)
        self.g_d.copy_(g_d, non_blocking=True)
        self.graph.replay()
        self.replays += 1
        return self.loss
