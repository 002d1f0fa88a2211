"""Two-GPU check of the data-parallel training step (needs >= 2 CUDA devices; skipped otherwise): overlapped bucketed
all-reduce == plain all-reduce == single-device gradient of the global batch, and per-rank prior draws differ."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu


def test_two_gpu_training_step_gradients():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29711", os.path.join(root, "tests", "dp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "DP_WORKER_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
