"""Constant LiDAR poses on two ranks (skipped when the box has fewer than two GPUs): tools/mgpu_fixed_lidar_check.py under
torchrun — a nonzero lvba_lidar_opts::pose_fixed is LVBA_ERR_UNSUPPORTED with an active communicator, in the one-shot call and in
lvba_lidar_reset_lm, and an all-zero mask solves as no mask."""
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


@pytest.mark.gpu
def test_mask_under_a_communicator_is_unsupported():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    port = 29600 + (os.getpid() + 700) % 1000
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(ROOT / "tools" / "mgpu_fixed_lidar_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(ROOT), timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("MGPU_FIXED_LIDAR PASS") == 2, r.stdout[-3000:]
