"""The batch split of the DiT forward over two GPUs (parallel.enable_cfg_parallel): FP8 weights and FP8 attention, bit-identical to the
single-GPU forward on both ranks.  Needs >= 2 GPUs; skipped on a single-GPU machine.

The sample offsets, the exchange and every mode are covered on one GPU by tests/test_gpu_cfg_parallel_one_gpu.py (host barrier).  What
only this test covers is the real multi-GPU machinery: the device flag barrier, the CUDA IPC handle exchange through torch.distributed,
and peer stores over NVLink into the other GPU's memory."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_batch_split_fp8_is_bit_identical_on_two_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port",
           "29523", os.path.join(ROOT, "tests", "cfg_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, "the batch-split forward differs from the single-GPU forward (see output)"
