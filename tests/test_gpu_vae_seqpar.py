"""The VAE split over the GPUs of a node (row bands, halo rows by peer store, csrc/vae.cu) against the single-GPU call: bit-identical
on every rank.  Needs >= 2 GPUs; skipped on a single-GPU machine.

tests/test_gpu_vae_seqpar_one_gpu.py covers the kernels, their address arithmetic and the host wiring on one GPU (host barrier, world 2
to 8).  What only this test covers is the real multi-GPU machinery: the device flag barrier, the CUDA IPC handle exchange through
torch.distributed, and peer stores over NVLink into another GPU's memory."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_split_vae_is_bit_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least two GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port",
           "29519", os.path.join(ROOT, "tests", "vae_sp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0, "the split VAE differs from the single-GPU call (see output)"
