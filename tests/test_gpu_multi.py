"""Needs >= 2 GPUs on the box (skipped otherwise): the graphed training step with the gradient exchange over NCCL, launched
like a multi-GPU bench.py run (one process per GPU)."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs on the box")
def test_graphed_step_ranks_agree_over_nccl():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(29600 + os.getpid() % 300), os.path.join(ROOT, "tools", "ddp_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "ddp_check world=2" in r.stdout
