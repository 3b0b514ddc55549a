"""GPU suite, needs >= 2 devices (skipped otherwise): gene shards over NCCL through the C ABI equal
the single-GPU fit -- the exchange before the trend step and the end-of-call exchange of the result tables, through grouped NCCL
all-gathers and through the peer-memory push kernel (CUDA IPC windows, NVLink stores), with ragged shards, eager and as a replayed
CUDA graph (tests/multi_gpu_worker.py)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_devices():
    try:
        import torch

        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("exchange", ["nccl", "peer"])
@pytest.mark.parametrize("world,N,G,design", [(2, 60, 3001, "factorial"), (2, 200, 4000, "two_level")])
def test_sharded_fit_equals_single_gpu_fit(world, N, G, design, exchange):
    if _n_devices() < world:
        pytest.skip(f"needs {world} GPUs")
    env = dict(os.environ, PDQ_MG_N=str(N), PDQ_MG_G=str(G), PDQ_MG_DESIGN=design, PDQ_MG_EXCHANGE=exchange, PDQ_PEER_TIMEOUT_MS="20000")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tests", "multi_gpu_worker.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    line = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert r.returncode == 0 and line, r.stdout[-2000:] + r.stderr[-2000:]
    rec = json.loads(line[-1])
    assert rec["ok"], rec
