"""Build libchronoedit_b200.so in-tree with nvcc for sm_90a (cross-compiles on a GPU-less box).

    python -m chronoedit_b200.build [--force]

Objects are cached under chronoedit_b200/build/ and rebuilt when a source or header is newer.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "lib", "libchronoedit_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
    "-I", INCLUDE, "-I", CSRC,
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: chronoedit_b200 needs the CUDA 12.9 toolkit to build its sm_90a kernels")


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    nvcc = _nvcc()
    hdr_mtime = max(os.path.getmtime(os.path.join(d, f)) for d in (CSRC, INCLUDE) for f in os.listdir(d)
                    if f.endswith((".cuh", ".h")))
    jobs = []
    objs = []
    for src in sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + ".o")
        objs.append(o)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_mtime):
            jobs.append([nvcc, *NVCC_FLAGS, *(["-Xptxas", "-v"] if verbose else []), "-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r.stderr

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        logs = list(ex.map(run, jobs))
    if verbose:
        for l in logs:
            sys.stderr.write(l)
    if jobs or not os.path.exists(LIB):
        run([nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
