"""Multi-GPU numerics (needs >= 2 GPUs on the box; skipped otherwise): launches tests/run_dist_parity.py under
torchrun with 2 ranks over NCCL and requires 'DIST PARITY OK'."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_two_rank_nccl_gradients_equal_global_batch():
    port = 29600 + (os.getpid() % 300)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "run_dist_parity.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    sys.stdout.write(out.stdout[-3000:])
    assert out.returncode == 0 and "DIST PARITY OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
