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
# the second setting runs one head-backward launch and all-reduce per head, then the all-reduce of the remaining tail
# (theta, loss slot, flag) -- a wrong tail range only shows with more than one rank -- and leaves 32 SMs to NCCL
@pytest.mark.parametrize("dp_env", [{}, {"DCA_DP_SPLIT_HEADS": "1", "DCA_DP_RESERVE_SMS": "32"}])
def test_two_rank_nccl_gradients_equal_global_batch(dp_env):
    port = 29600 + (os.getpid() % 300) + 300 * len(dp_env)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "run_dist_parity.py")]
    env = {k: v for k, v in os.environ.items() if not k.startswith("DCA_DP_")}
    env.update(dp_env)
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    sys.stdout.write(out.stdout[-3000:])
    assert out.returncode == 0 and "DIST PARITY OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
