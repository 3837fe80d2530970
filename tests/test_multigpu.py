"""Multi-GPU checks of the split `north_star` names (SURVEY.md §8e) on real devices: launched as one torch.distributed.run job
with one rank per visible GPU (NCCL over NVLink); skipped below 2 devices.  The world_size-2 gloo tests on CPU
(test_parallel_gloo.py, test_data_parallel_gloo.py) cover the same host logic without GPUs.  On one GPU,
test_sharded_fp64_gpu.py plays the ranks in one process: row shards and the drop-in wrapper's shards bit for bit against the
unsharded call, the sharded training batch's loss gradient, shard gradients, their sum and the regulariser against float64."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs at least 2 GPUs")
def test_sharded_paths_match_single_gpu(built_lib):
    n = min(torch.cuda.device_count(), 4)
    n = 1 << (n.bit_length() - 1)  # 2 or 4 ranks (verified on the box; bench.py covers 8): the 128-row test frame and the 256-ray batch split evenly
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "mgpu_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    sys.stdout.write(res.stdout[-3000:])
    sys.stderr.write(res.stderr[-3000:])
    assert res.returncode == 0
    for name in ("rows_bit_identical", "dp_validation_bit_identical", "dp_train_gradients", "fused_trainer_sharded"):
        assert f"MGPU_OK {name}" in res.stdout, name
