"""Sequence-parallel DiT forward (tokens of one edit split over the GPUs of a node, q/k/v and attention output exchanged by peer
stores inside the kernels, csrc/seqpar.cuh) against the single-GPU forward: bit-identical on every rank.  Needs >= 2 GPUs;
skipped on a single-GPU machine.

The kernels, their address arithmetic and the host wiring are covered on one GPU by tests/test_gpu_seqpar_one_gpu.py (host
barrier, world 2 to 8).  What only this test covers is the real multi-GPU machinery: the device flag barrier (sp_barrier_kernel),
the CUDA IPC handle exchange through torch.distributed, and peer stores over NVLink into another GPU's memory."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_sequence_parallel_forward_is_bit_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least two GPUs")
    world = 2
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1", "--master-port",
           "29517", os.path.join(ROOT, "tests", "sp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, "sequence-parallel forward differs from the single-GPU forward (see output)"
