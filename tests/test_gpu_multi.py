"""Multi-GPU parity of the voxel-sharded global-BA step under pytest -m gpu: launches tests/multi_gpu_worker.py with torchrun on 2 GPUs
(sharded LM solve, an empty shard, sharded HBA window — each compared with the single-process oracle inside the worker).
Skipped on a machine with fewer than 2 GPUs; `python -m pytest tests -m gpu` on a multi-GPU machine runs it."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_sharded_global_ba_two_gpus():
    port = 29600 + os.getpid() % 300
    env = dict(os.environ, NCCL_DEBUG="WARN")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "multi_gpu_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    sys.stdout.write(r.stdout[-4000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "FAIL" not in r.stdout and r.stdout.count("OK") >= 4
