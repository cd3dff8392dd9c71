#!/usr/bin/env python3
"""Builds the in-tree native libraries of minbpe_b200 (no network, no JIT cache):

  libb200bpe.so    hand-written sm_90a (H100) kernels + the C ABI of include/b200bpe.h   (nvcc)
  libbpesynth.so   synthetic corpus generator for bench/tests                             (gcc)

nvcc cross-compiles without a GPU.  Called by __graft_entry__.build().
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUDA_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]


def _stale(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def build(force=False, verbose=False):
    cu_sources = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cu", ".cuh", ".inl", ".h"))]
    cu_sources.append(os.path.join(HERE, "..", "..", "include", "b200bpe.h"))
    so = os.path.join(HERE, "libb200bpe.so")
    if force or _stale(so, cu_sources):
        cmd = [NVCC] + CUDA_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", so, os.path.join(HERE, "b200bpe.cu")]
        subprocess.check_call(cmd, cwd=HERE)
    syn = os.path.join(HERE, "libbpesynth.so")
    if force or _stale(syn, [os.path.join(HERE, "synth.c")]):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-o", syn, os.path.join(HERE, "synth.c"), "-lm", "-lpthread"],
                              cwd=HERE)
    return so, syn


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
