#!/usr/bin/env python3
"""Time k_hist_dense, the byte-pair histogram that builds the first pair table of every training on a byte stream, on
the 1 GiB synthetic corpus (seed 1337, GPT-4 chunks, as bench.py's headline workload).

    python bench_hist_dense.py [--lib A.so --lib B.so ...] [--rounds 3] [--reps 5] [--size-mib 1024]

Every library is timed in its own worker process, and the libraries take turns round by round, so that two builds
(say the parent commit's and this one's) are compared under the same conditions.  A worker loads the stream, runs
train(1) `reps` times and reports, per call, the device time of the k_hist_dense kernel (torch.profiler, CUDA activity)
and bpe_timing.init_ms (CUDA events around the whole initial statistics).  Prints one JSON line with the GPU's name and
power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def worker(corpus, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from minbpe_b200 import engine as E
    raw = np.load(corpus + ".raw.npy", mmap_mode="r")
    offs = np.load(corpus + ".offs.npy", mmap_mode="r")
    raw, offs = np.ascontiguousarray(raw), np.ascontiguousarray(offs)
    eng = E.Engine(0)
    eng.set_option(E.OPT_HIST_KERNEL, 2)
    kernel_ms, init_ms, pairs = [], [], None
    for r in range(reps + 1):                                  # call 0 warms up
        eng.load_stream(raw, offs)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            p, c, d = eng.train(1)
            torch.cuda.synchronize()
        assert eng.timing()["hist_kernel"] == 2
        ks = [e for e in prof.events() if e.name.startswith("k_hist_dense(") or e.name == "k_hist_dense"]
        assert len(ks) == 1, sorted({e.name for e in prof.events()})[:20]
        if r:
            kernel_ms.append(ks[0].device_time / 1e3)
            init_ms.append(eng.timing()["init_ms"])
        pairs = (p.tolist(), c.tolist())
    eng.close()
    print(json.dumps({"kernel_ms": kernel_ms, "init_ms": init_ms, "merge": pairs}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", help="libb200bpe.so to time (default: the one built in this tree)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--size-mib", type=int, default=1024)
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.worker, a.reps)
    import torch
    from bench import make_corpus
    libs = a.lib or [os.path.join(ROOT, "minbpe_b200", "csrc", "libb200bpe.so")]
    with tempfile.TemporaryDirectory() as tmp:
        corpus = os.path.join(tmp, "corpus")
        raw, offs, _ = make_corpus(a.size_mib << 20, 1337)
        np.save(corpus + ".raw.npy", raw)
        np.save(corpus + ".offs.npy", offs)
        del raw, offs
        res = {lib: [] for lib in libs}
        for _ in range(a.rounds):
            for lib in libs:
                env = dict(os.environ, BPE_LIB_PATH=lib)
                out = subprocess.run([sys.executable, __file__, "--worker", corpus, "--reps", str(a.reps)], env=env, check=True,
                                     stdout=subprocess.PIPE, text=True).stdout
                res[lib].append(json.loads(out.strip().splitlines()[-1]))
    merges = {json.dumps(r["merge"]) for rs in res.values() for r in rs}
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    summary = {}
    for lib, rs in res.items():
        k = [x for r in rs for x in r["kernel_ms"]]
        i = [x for r in rs for x in r["init_ms"]]
        summary[lib] = {"kernel_ms_median": float(np.median(k)), "kernel_ms_min": min(k), "kernel_ms_max": max(k),
                        "kernel_ms_per_round": [float(np.median(r["kernel_ms"])) for r in rs],
                        "init_ms_median": float(np.median(i))}
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": power.splitlines()[0] if power else None,
                      "size_mib": a.size_mib, "same_merge": len(merges) == 1, "libs": summary}))


if __name__ == "__main__":
    main()
