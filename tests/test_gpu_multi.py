"""N>1 on real GPUs: the sharded batch (NCCL all-gather) returns the same bytes as a single rank (SURVEY.md §8e).
Needs >= 2 visible GPUs; skipped on a 1-GPU box, where tests/test_sharding.py (gloo) covers the logic."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu


def test_sharded_batch_equals_single_rank_nccl():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least 2 GPUs")
    world = 2 if n < 4 else 4
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "multi_gpu_worker.py")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                          "--master-addr", "127.0.0.1", "--master-port", str(port), worker], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-4000:]
    assert "MULTI_GPU_OK world=%d" % world in out.stdout
