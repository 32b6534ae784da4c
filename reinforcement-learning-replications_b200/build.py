"""Build libb200rl.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python reinforcement-learning-replications_b200/build.py [--force] [--verbose]

The .so and the per-source objects under build/ are git-ignored build products; nvcc needs no GPU, so the library can
be cross-compiled on a machine without one.
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200rl.so")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default",
    "-I", os.path.join(ROOT, "include"), "-I", CSRC,
]
OBJ_DIR = os.path.join(HERE, "build")  # per-source objects (git-ignored); only stale ones are recompiled


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _headers():
    return glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(ROOT, "include", "*.h"))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(d) > t for d in sources() + _headers())


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libb200rl.so needs the CUDA toolkit (12.x, sm_90a) to build")
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdr_time = max(os.path.getmtime(h) for h in _headers())
    jobs, objs = [], []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_time):
            jobs.append([nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src])
    procs = [subprocess.Popen(c, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for c in jobs]
    failed = False
    for c, pr in zip(jobs, procs):  # one nvcc per source file, all at once
        out, _ = pr.communicate()
        if verbose or pr.returncode != 0:
            sys.stderr.write(out)
        failed |= pr.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed building libb200rl.so")
    tmp = LIB + ".tmp"  # link beside the target and rename: a reader never sees a half-written library
    r = subprocess.run([nvcc, "--shared", "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a", "-o", tmp]
                       + objs, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("linking libb200rl.so failed")
    os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
