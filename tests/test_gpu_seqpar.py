"""The splits over the GPUs of a node against the single-GPU calls, bit-identical on every rank: the sequence-parallel DiT forward
(tokens of one edit split, q/k/v and attention output exchanged by peer stores inside the kernels, csrc/seqpar.cuh) and the VAE
(row bands, halo rows by peer store, csrc/vae.cu).  Needs >= 2 GPUs; skipped on a single-GPU machine.

The kernels, their address arithmetic and the host wiring are covered on one GPU by tests/test_gpu_seqpar_one_gpu.py and
tests/test_gpu_vae_seqpar_one_gpu.py (host barrier, world 2 to 8).  What only these tests cover is the real multi-GPU machinery: the
device flag barrier (sp_barrier_kernel), the CUDA IPC handle exchange through torch.distributed, and peer stores over NVLink into
another GPU's memory."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torchrun(check, port, world=2):
    """tests/sp_worker.py `check` under torchrun on `world` GPUs; its exit code."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs at least {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1", "--master-port",
           str(port), os.path.join(ROOT, "tests", "sp_worker.py"), check]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    sys.stdout.write(r.stdout[-4000:])
    sys.stderr.write(r.stderr[-2000:])
    return r.returncode


@pytest.mark.gpu
def test_sequence_parallel_forward_is_bit_identical():
    assert _torchrun("dit", 29517) == 0, "sequence-parallel forward differs from the single-GPU forward (see output)"


@pytest.mark.gpu
def test_split_vae_is_bit_identical():
    assert _torchrun("vae", 29519) == 0, "the split VAE differs from the single-GPU call (see output)"
