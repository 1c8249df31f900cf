"""Build the C-ABI shared library in-tree with nvcc for sm_90a (H100)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpulser_b200.so")
SOURCES = ["plan.cu"]
DEPS = ["plan.cu", "kernels.cuh", "spline.hpp", "../../include/pulser_b200.h"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libpulser_b200.so")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(
        os.path.getmtime(os.path.join(CSRC, d)) > t
        for d in DEPS
        if os.path.exists(os.path.join(CSRC, d))
    )


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    cmd = [
        _nvcc(),
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-lineinfo", "-O3", "-std=c++17",
        "-Xcompiler", "-fPIC,-O2,-Wall",
        "-Xptxas", "-v" if verbose else "-O3",
        "-shared", "-o", LIB,
    ] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stdout + res.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
