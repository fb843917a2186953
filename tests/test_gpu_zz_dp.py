"""N-GPU data parallelism of the product path == the 1-GPU step on the global batch (needs >= 2 GPUs: run with
`python -m pytest tests/test_gpu_zz_dp.py -m gpu` on a machine with two GPUs; skipped with one)."""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.parametrize("kind", ["ctc", "hybrid"])
def test_dp_step_equals_single_gpu_step_on_the_global_batch(kind):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tests", "dp_worker.py"), kind]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, (out.stdout[-2000:], out.stderr[-4000:])
    assert "DP_OK" in out.stdout
