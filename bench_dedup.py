#!/usr/bin/env python3
"""Training on the distinct chunks of a text (bpe_load_text_gpt4_dedup + bpe_train, DESIGN.md §14) against the plain path
(bpe_load_text_gpt4 + bpe_train), on one H100.  Prints one JSON line.

  cfg3   1 GiB synthetic (seed 1337), vocab 32,768, from a pinned host text: the two paths alternated, 3 runs each; load
         ms, loop ms, stream tokens and the chunk counters of each run.  Every run's merges and counts must be identical
         (the plain path is the one bench.py and tests/test_gpu_full.py check against the oracle).
  cfg4   4 GiB synthetic (seed 1338): the first 1,024 merges on both paths, which must be identical; then the dedup path
         to vocab 100,000 or to exhaustion.
  big    16 GiB (seed 1338) with dedup on one GPU: more text than the plain path's 8 B of HBM per byte fits in 80 GB.
         Reported as skipped when the host has too little free memory for the text.

Usage: python bench_dedup.py [--cfg3-mib 1024] [--cfg4-mib 4096] [--big-mib 16384] [--runs 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1]), "sm_clock_mhz": float(q[2])}


def pinned(raw):
    import torch
    return torch.from_numpy(raw).pin_memory().numpy()


def host_free_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def run(eng, text, merges, dedup):
    t0 = time.perf_counter()
    if dedup:
        eng.load_text_gpt4_dedup(text)
    else:
        eng.load_text_gpt4(text)
    tokens = eng.stream_len()
    load_ms = (time.perf_counter() - t0) * 1e3
    p, c, d = eng.train(merges)
    tm = eng.timing()
    r = {"load_ms": round(load_ms, 1), "loop_ms": round(tm["loop_ms"], 1), "stream_tokens": int(tokens), "merges": int(d),
         "kernel_launches": int(tm["kernel_launches"])}
    if dedup:
        r["dedup_stats"] = eng.dedup_stats()
    return r, p, c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg3-mib", type=int, default=1024)
    ap.add_argument("--cfg4-mib", type=int, default=4096)
    ap.add_argument("--big-mib", type=int, default=16384)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    if "H100" not in info["name"]:
        sys.exit(f"bench_dedup.py measures on an H100; device 0 is {info['name']}")
    from minbpe_b200.engine import Engine
    from minbpe_b200.synth import generate
    eng = Engine(0)
    out = {"gpu": info}

    # ---- cfg3: plain and dedup alternated ----
    text = pinned(generate(1337, a.cfg3_mib << 20))
    runs, ref, same = {"plain": [], "dedup": []}, None, True
    for _ in range(a.runs):
        for kind in ("plain", "dedup"):
            r, p, c = run(eng, text, 32512, kind == "dedup")
            key = (p.tobytes(), c.tobytes())
            ref = key if ref is None else ref
            same = same and key == ref
            runs[kind].append(r)
    out["cfg3"] = {"mib": a.cfg3_mib, "vocab": 32768, "runs": runs, "parity_merges_and_counts_identical": same}
    del text

    # ---- cfg4: first 1,024 merges on both paths, then dedup to the end ----
    text = pinned(generate(1338, a.cfg4_mib << 20))
    rp, pp, cp = run(eng, text, 1024, False)
    rd, pd, cd = run(eng, text, 1024, True)
    t0 = time.perf_counter()
    full, pf, cf = run(eng, text, 100000 - 256, True)
    full["seconds"] = round(time.perf_counter() - t0, 2)
    out["cfg4"] = {"mib": a.cfg4_mib, "first_1024": {"plain": rp, "dedup": rd,
                                                     "parity_identical": bool(np.array_equal(pp, pd) and np.array_equal(cp, cd))},
                   "dedup_to_end": full, "prefix_matches_first_1024": bool(np.array_equal(pf[:1024], pp) and np.array_equal(cf[:1024], cp))}
    del text

    # ---- 16 GiB on one GPU, dedup only ----
    need = (a.big_mib << 20) + (8 << 30)
    if host_free_bytes() < need:
        out["big"] = {"mib": a.big_mib, "skipped": f"host has {host_free_bytes() >> 30} GiB free, needs {need >> 30} GiB"}
    else:
        text = generate(1338, a.big_mib << 20)
        t0 = time.perf_counter()
        r, p, c = run(eng, text, 32512, True)
        r["seconds"] = round(time.perf_counter() - t0, 2)
        out["big"] = {"mib": a.big_mib, "vocab": 32768, "dedup": r,
                      "plain_would_need_gib": round(8 * (a.big_mib << 20) / 2 ** 30, 1)}
        del text
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
