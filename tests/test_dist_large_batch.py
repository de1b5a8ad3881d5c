"""Data-parallel steps above GG_MAX_BATCH pairs with one rank per GPU (world = min(GPUs, 4)): replicas bit-identical, the
merged gradient equal to the one-GPU simulation of the same world, the C loop equal to the step loop, GraphGAN.train()
with batch 4096, and the peer-memory transport still refusing such batches (tests/dist_large_batch_worker.py)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_nccl_data_parallel_large_batches():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(min(n, 4)), "--master-addr",
           "127.0.0.1", "--master-port", "29663", os.path.join(ROOT, "tests", "dist_large_batch_worker.py"), "multi"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0 and "DP_MULTI_OK" in r.stdout, r.stdout[-3000:]
