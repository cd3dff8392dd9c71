#!/usr/bin/env python3
"""The o200k (GPT-4o) split pattern on the device (DESIGN.md §17) on one H100.  Prints one JSON line.

  parity   device chunk offsets of the synthetic corpus (seed 1337) under O200K_SPLIT_PATTERN against the host split
           (presplit.chunk_offsets, `regex` on the host cores): must be identical.
  split    device time of the split kernels (BPE_OPT_KERNEL_TIMING -> init_ms of bpe_load_text_gpt4) for the GPT-4 and the
           o200k pattern, alternated, --runs each; and the GB/s of text they make.
  train    RegexTokenizer(O200K_SPLIT_PATTERN).train_from_file(dedup=True) to vocab --vocab on the corpus written to a
           temporary file, timed; its first --check merges against oracle.c_train weighted over the host chunks.

Usage: python bench_split_o200k.py [--mib 1024] [--runs 3] [--vocab 32768] [--check 256]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1]), "sm_clock_mhz": float(q[2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--vocab", type=int, default=32768)
    ap.add_argument("--check", type=int, default=256)
    a = ap.parse_args()
    info = gpu_info()
    if "H100" not in info["name"]:
        sys.exit(f"bench_split_o200k.py measures on an H100; device 0 is {info['name']}")
    import oracle
    from minbpe_b200 import O200K_SPLIT_PATTERN, RegexTokenizer
    from minbpe_b200 import engine as E
    from minbpe_b200.presplit import chunk_offsets
    from minbpe_b200.synth import generate
    raw = generate(1337, a.mib << 20)
    out = {"gpu": info, "corpus_bytes": int(raw.size)}

    t0 = time.perf_counter()
    host = chunk_offsets(O200K_SPLIT_PATTERN, raw)
    out["host_split_s"] = round(time.perf_counter() - t0, 2)
    eng = E.Engine(0)
    eng.set_option(E.OPT_SPLIT_PATTERN, 3)
    dev = eng.split_gpt4(raw)
    out["parity"] = {"chunks_host": int(host.size), "chunks_device": int(dev.size), "identical": bool(np.array_equal(host, dev))}
    del dev

    eng.set_option(E.OPT_KERNEL_TIMING, 1)
    split = {"gpt4": [], "o200k": []}
    for _ in range(a.runs + 1):                       # the first round warms up and is dropped
        for name, pat in (("gpt4", 0), ("o200k", 3)):
            eng.set_option(E.OPT_SPLIT_PATTERN, pat)
            eng.load_text_gpt4(raw)
            split[name].append(eng.timing()["init_ms"])
    eng.set_option(E.OPT_KERNEL_TIMING, 0)
    eng.close()
    out["split_ms"] = {k: [round(x, 2) for x in v[1:]] for k, v in split.items()}
    out["split_gb_s"] = {k: round(raw.size / (min(v[1:]) * 1e-3) / 1e9, 1) for k, v in split.items()}

    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "corpus.txt")
        raw.tofile(path)
        tok = RegexTokenizer(O200K_SPLIT_PATTERN)
        t0 = time.perf_counter()
        tok.train_from_file(path, a.vocab, dedup=True)
        out["train_from_file_dedup_s"] = round(time.perf_counter() - t0, 2)
    ub, uo, uw = oracle.c_dedup_chunks(raw, host)
    wp, _, wn = oracle.c_train(ub.astype(np.int32), uo, a.check, weights=uw)
    got = [list(p) for p in tok.merges][: a.check]
    out["train"] = {"vocab": a.vocab, "merges": len(tok.merges), "checked_merges": int(wn),
                    "first_merges_equal_oracle": got == wp.tolist()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
