"""The call-pair split over two GPUs (parallel.enable_cfg_parallel_calls): FP8 weights, FP8 attention and TeaCache, bit-identical to the
single-GPU loop on both ranks with every TeaCache decision kept.  Needs >= 2 GPUs; skipped on a single-GPU machine.

The pairing, the exchange and every mode are covered on one GPU by tests/test_gpu_cfg_calls_one_gpu.py (host barrier).  What only this
test covers is the real multi-GPU machinery: the device flag barrier, the CUDA IPC handle exchange through torch.distributed, and peer
stores over NVLink into the other GPU's memory."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_call_pair_fp8_teacache_is_bit_identical_on_two_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port",
           "29524", os.path.join(ROOT, "tests", "cfg_calls_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, "the call-pair split differs from the single-GPU loop (see output)"
