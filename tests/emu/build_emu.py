#!/usr/bin/env python3
"""TEST INFRASTRUCTURE.  Builds tests/emu/_build/libb200bpe_emu.so: the sources of minbpe_b200/csrc (kernels AND host
side, unchanged apart from the two syntactic rewrites below) compiled with g++ against the CPU SIMT emulator
tests/emu/cuda_emu.h.  Same C ABI as libb200bpe.so; loaded only by tests/test_emu_*.py through BPE_LIB_PATH.

Rewrites (everything else is handled by cuda_emu.h and the BPE_SIMT_EMU branches of the PTX helpers in common.cuh /
k_xchg.cuh):
    kernel<<<grid, block, smem, stream>>>(args)   ->  EMU_LAUNCH((kernel), (grid, block, smem, stream), (args))
    extern __shared__ [__align__(n)] T name[];    ->  T *name = reinterpret_cast<T *>(emu::dyn_smem());
    __noinline__                                  ->  EMU_NOINLINE   (libstdc++ uses the former spelling itself)
"""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "minbpe_b200", "csrc")
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libb200bpe_emu.so")

LAUNCH = re.compile(r"([A-Za-z_]\w*(?:<[^<>;(){}]*>)?)\s*<<<")
EXTERN_SHARED = re.compile(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?([\w ]+?)\s+(\w+)\s*\[\s*\]\s*;")


def _match_paren(s, i):
    """s[i] == '(' -> index just past the matching ')' (string/char literals are not used inside launch arguments)."""
    depth = 0
    for j in range(i, len(s)):
        if s[j] == "(":
            depth += 1
        elif s[j] == ")":
            depth -= 1
            if depth == 0:
                return j + 1
    raise ValueError("unbalanced parentheses in a kernel launch")


def rewrite(src):
    out, pos = [], 0
    while True:
        m = LAUNCH.search(src, pos)
        if not m:
            out.append(src[pos:])
            break
        end_cfg = src.index(">>>", m.end())
        k = end_cfg + 3
        while src[k].isspace():
            k += 1
        assert src[k] == "(", "kernel launch without an argument list"
        end_args = _match_paren(src, k)
        out.append(src[pos:m.start()])
        out.append(f"EMU_LAUNCH(({m.group(1)}), ({src[m.end():end_cfg]}), {src[k:end_args]})")
        pos = end_args
    src = "".join(out)
    src = src.replace("__noinline__", "EMU_NOINLINE")
    src = EXTERN_SHARED.sub(lambda m: f"{m.group(1)} *{m.group(2)} = reinterpret_cast<{m.group(1)} *>(emu::dyn_smem());", src)
    return src


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".inl", ".h")))


def build(force=False):
    os.makedirs(os.path.join(OUT, "src"), exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in sources()] + [os.path.join(HERE, f) for f in ("cuda_emu.h", "cuda_emu.cpp", "build_emu.py")]
    deps.append(os.path.join(ROOT, "include", "b200bpe.h"))
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in deps):
        return LIB
    for f in sources():
        text = rewrite(open(os.path.join(CSRC, f)).read())
        text = text.replace('#include "../../include/b200bpe.h"', '#include "b200bpe.h"')
        name = "b200bpe_emu.cpp" if f == "b200bpe.cu" else f
        if f == "b200bpe.cu":
            text = '#include "cuda_emu.h"\n' + text
        with open(os.path.join(OUT, "src", name), "w") as fh:
            fh.write(text)
    opt = os.environ.get("EMU_OPT", "-O1")
    # EMU_SANITIZE=1: UBSan's alignment check turns every vector access of the kernels (uint2 / uint4 / ulonglong2 loads and
    # stores carry their CUDA alignment here) into a trap when the address is not aligned as the GPU requires — x86 itself
    # would not notice.  Load the result with LD_PRELOAD=$(g++ -print-file-name=libubsan.so) under python.
    # Also checked: shift counts >= the operand width (x86 masks the count, the GPU's shl/shr clamp: `1u << 32` is 1 here and 0
    # there — code that reaches such a shift computes different things on the two) and indices past the end of arrays of
    # known size (shared-memory and local arrays).
    checks = "alignment,shift,bounds"
    san = [f"-fsanitize={checks}", f"-fno-sanitize-recover={checks}"] if os.environ.get("EMU_SANITIZE") else []
    # -Wno-subobject-linkage: the owner types of b200bpe.cu (DevBuf, Event, PairTable) sit in an anonymous namespace so that
    # they export nothing from the library; the handle and the sub-states of the .inl files (headers to g++) hold them as
    # fields, which is fine in this one translation unit
    cmd = ["g++", "-std=c++17", opt, "-g", "-fPIC", "-shared", "-fno-strict-aliasing", "-Wno-unknown-pragmas", "-Wno-attributes",
           "-Wno-subobject-linkage"] + san + [
           "-I", HERE, "-I", os.path.join(ROOT, "include"), "-I", os.path.join(OUT, "src"),
           os.path.join(OUT, "src", "b200bpe_emu.cpp"), os.path.join(HERE, "cuda_emu.cpp"), "-o", LIB, "-lpthread"]
    if san:
        cmd[cmd.index("-o") + 1] = LIB.replace(".so", "_ubsan.so")
    subprocess.check_call(cmd)
    return cmd[cmd.index("-o") + 1]


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
