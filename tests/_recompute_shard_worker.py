"""torchrun worker for tests/test_gpu_lstm_recompute.py: the NCCL worker of the sharded-model tests (_shard_nccl_worker.py) with
`model.lstm_recompute = True` for the sharded model only, so that its LSTM runs the recomputing backward while the whole model
it is compared with keeps the stored state.  `recompute_calls` in the result counts the LSTM calls that took that path on rank 0."""
import json
import os
import socket
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _shard_nccl_worker as base  # noqa: E402
from mpgcn_b200 import ops, shard  # noqa: E402

CALLS = [0]


def _install():
    sharded_forward, chunk_cells = shard.sharded_forward, ops.lstm_recompute_chunk_cells

    def counting_chunk_cells(recompute, *a):
        n = chunk_cells(recompute, *a)
        CALLS[0] += n > 0
        return n

    def recompute_sharded_forward(model, *a, **kw):
        model.lstm_recompute = True
        try:
            return sharded_forward(model, *a, **kw)
        finally:
            model.lstm_recompute = None

    ops.lstm_recompute_chunk_cells = counting_chunk_cells
    base.shard.sharded_forward = recompute_sharded_forward


def run(world, tmp_path, models):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = tmp_path / f"recompute-{world}.json"
    spec = json.dumps(dict(kind="row", peer=False, models=list(models)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
                        "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__), spec, str(out)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return json.load(open(out))


if __name__ == "__main__":
    _install()
    base.main(json.loads(sys.argv[1]), sys.argv[2])
    if os.path.exists(sys.argv[2]):          # rank 0 wrote the rows
        res = json.load(open(sys.argv[2]))
        res["recompute_calls"] = CALLS[0]
        json.dump(res, open(sys.argv[2], "w"))
