"""Builds libkeystone_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m keystone_b200.build [--force]

The objects and the shared library land in keystone_b200/lib/, which git ignores.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libkeystone_b200.so")
SOURCES = ["tc_kernels.cu", "aux_kernels.cu", "solve_kernels.cu", "engine.cu", "bwls.cu", "krr.cu", "lbfgs.cu", "sparse.cu", "logistic.cu", "pca.cu", "fisher.cu", "gmm_fit.cu", "sift.cu", "hog_daisy.cu", "augment.cu", "text.cu", "io.cu"]
HEADERS = ["tc_common.cuh", "cluster.cuh", "kernels.h", "operand_split.cuh", "lbfgs_core.cuh", "lower_table.h", "engine.h", os.path.join("..", "..", "include", "keystone_b200.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "-DKS_BUILD",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = True) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    nvcc = _nvcc()
    hdrs = [os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS]
    objs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(LIBDIR, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd), flush=True)
            subprocess.check_call(cmd)
    if force or _stale(LIB, objs):
        # cudart is linked statically so the library loads (and exports its symbols) on a box without a GPU driver;
        # cuSOLVER / NCCL / the driver entry point for cuTensorMapEncodeTiled are resolved at run time.
        # linked under a temporary name and renamed: a snapshot of the tree never sees a half-written library
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB + ".tmp"] + objs + ["-cudart", "static", "-ldl", "-lpthread"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
