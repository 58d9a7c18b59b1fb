"""Window functions across two ranks (NCCL, two H100s): the rank-ordered concatenation of every rank's output equals the
single-GPU output bit for bit, float SUM / AVG included, also with one rank holding no rows."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_nccl_world2_window():
    from datafusion_archive_b200 import engine
    if engine.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29681", os.path.join(ROOT, "tests", "window_mp_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    assert "MP_WINDOW_OK world=2" in p.stdout
