"""Column-sharded decode on 2 GPUs == single-GPU decode (tools/tp_check.py under torchrun).  Skipped with a single GPU;
the host-side logic is covered on CPU by tests/test_tp_gloo.py."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tp2_matches_single_gpu():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29655", os.path.join(ROOT, "tools", "tp_check.py"), "test-small"]
    r = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert "TP_CHECK PASS" in r.stdout, r.stdout[-3000:]
