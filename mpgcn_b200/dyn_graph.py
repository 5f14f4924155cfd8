"""Dynamic O / D graphs from the OD history on the GPU: drop-in for ``DataInput.construct_dyn_G``
(reference ``Data_Container_OD.py:39-59``), which makes ``2 * 7 * N^2`` Python-level scipy calls (14 M at N = 1000).

    from mpgcn_b200.dyn_graph import construct_dyn_G, install
    O_dyn_G, D_dyn_G = construct_dyn_G(OD_data, split_ratio=[6.4, 1.6, 2])      # [N, N, 7] float64 each, as the reference
    install(Data_Container_OD.DataInput)        # or: replace the reference's method in place (keeps its signature)

Same slot averaging, same cosine distance (scipy's, clipped to [0, 2], NaN for a zero vector), same eq.-(7) quirk
(column i against ROW j, ``Data_Container_OD.py:56``).  Arithmetic is fp32 on the device (the reference: float64 on the
host), so values agree to ~1e-6 absolute.
"""
import numpy as np
import torch

from . import _lib


def _history_len(num_days: int, split_ratio, perceived_period: int) -> int:
    train_len = int(num_days * split_ratio[0] / sum(split_ratio))           # Data_Container_OD.py:40
    return (train_len // perceived_period) * perceived_period               # :41-42 (the remainder is dropped)


@_lib.engine_buffers()
def construct_dyn_G(OD_data, split_ratio, perceived_period: int = 7, device=None):
    """OD_data [days, N, N, 1] (numpy or torch, un-normalised) -> (O_dyn_G, D_dyn_G), numpy float64 [N, N, perceived_period]."""
    od = torch.as_tensor(np.asarray(OD_data) if not isinstance(OD_data, torch.Tensor) else OD_data)
    if od.dim() == 4:
        assert od.shape[-1] == 1
        od = od[..., 0]
    assert od.dim() == 3 and od.shape[1] == od.shape[2], "OD_data must be [days, N, N(, 1)]"
    P = int(perceived_period)
    used = _history_len(od.shape[0], list(split_ratio), P)
    if used < P:
        raise ValueError(f"construct_dyn_G: {od.shape[0]} days leave no complete period of {P} in the training split")
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("mpgcn_b200.dyn_graph runs on a CUDA device only (there is no CPU path)")
    lib = _lib.load()
    _lib.sync_deterministic()            # fixed-order column norms under torch.use_deterministic_algorithms(True)
    N = od.shape[1]
    hist = od[:used].to(device=dev, dtype=torch.float32).contiguous()
    o_g = torch.empty((P, N, N), dtype=torch.float32, device=dev)
    d_g = torch.empty_like(o_g)
    ws = torch.empty(max(int(lib.mpgcn_dyn_graph_workspace_bytes(P, N)), 256), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.mpgcn_dyn_graph_build(hist.data_ptr(), used // P, o_g.data_ptr(), d_g.data_ptr(), P, N, ws.data_ptr(), ws.numel(),
                                             torch.cuda.current_stream().cuda_stream), "dyn_graph_build")
    # the reference stacks the slots on the last axis and works in float64
    return (o_g.permute(1, 2, 0).contiguous().cpu().numpy().astype(np.float64),
            d_g.permute(1, 2, 0).contiguous().cpu().numpy().astype(np.float64))


def install(data_input_cls):
    """Replace ``DataInput.construct_dyn_G`` (same signature: self, OD_data, perceived_period=7) by the GPU version."""
    def _method(self, OD_data, perceived_period: int = 7):
        return construct_dyn_G(OD_data, self.params['split_ratio'], perceived_period)
    data_input_cls.construct_dyn_G = _method
    return data_input_cls
