"""Build libicaf_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m icafusion_b200.build [--force]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libicaf_b200.so")
SOURCES = ["api.cu", "conv_gemm.cu", "attn.cu", "image.cu", "pool.cu", "dmff.cu", "nms.cu", "loss.cu", "wgrad.cu", "train.cu",
           "attn_bwd.cu", "augment.cu", "bottleneck.cu", "metrics.cu",
           "confluence.cu"]
HEADERS = ["ptx.cuh", "icaf_internal.cuh", "conv_common.cuh", "staging.cuh", os.path.join("..", "..", "include", "icaf_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math=false"]


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build libicaf_b200.so")
    return exe


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = _nvcc()
    objs = []
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]
    procs = []
    for s in SOURCES:
        obj = os.path.join(CSRC, s[:-3] + ".o")
        cmd = [nvcc, *flags, "-c", os.path.join(CSRC, s), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            print(out)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {s}")
    cmd = [nvcc, *NVCC_FLAGS[:2], "-shared", "-o", LIB, *objs, "-lcudart"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
