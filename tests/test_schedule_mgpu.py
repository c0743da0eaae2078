"""-m gpu: launches tests/mgpu_schedule.py on 2 and 4 GPUs of the box; skipped where there are fewer."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world", [2, 4])
def test_schedule_across_ranks(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29531 + 7 * world),
           os.path.join(ROOT, "tests", "mgpu_schedule.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stderr[-4000:]
    assert "[mgpu-schedule] PASS" in r.stdout
