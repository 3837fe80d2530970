"""Data-parallel steps over several images and data_parallel(nerf.render_frames) on real devices: one torch.distributed.run job
with 2 or 4 ranks (NCCL), skipped below 2 devices.  On one GPU, test_train_images_sharded_gpu.py plays the ranks in one
process; test_train_images_sharded_cpu.py covers the render_frames wrapper's host logic on gloo."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs at least 2 GPUs")
def test_sharded_image_steps_and_frames_match_single_gpu(built_lib):
    n = min(torch.cuda.device_count(), 4)
    n = 1 << (n.bit_length() - 1)  # 2 or 4 ranks: the 1024-ray batch and the 512-ray frame call split evenly
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29543", os.path.join(ROOT, "tests", "mgpu_images_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    sys.stdout.write(res.stdout[-3000:])
    sys.stderr.write(res.stderr[-3000:])
    assert res.returncode == 0
    for name in ("images_steps_lockstep", "dp_render_frames"):
        assert f"MGPU_OK {name}" in res.stdout, name
