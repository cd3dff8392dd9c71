#!/usr/bin/env python3
"""Kernel time of every merge pass in bench.py's timed window, grouped by the number of merges (members) a pass carries
(DESIGN.md §3 "Batched merges", §4).  Prints one JSON line.

The window is bench.py's: cfg3 (1 GiB synthetic, seed 1337, GPT-4 split), train(W) and then the K timed merges.  Its
pass partition comes from the host model tests/batch_model.py, run on the oracle's distinct chunks with their counts.
The window is then replayed as one train(nk_i) call per pass: a pass never carries more members than the merges left
in its call, so each call is exactly that pass, and its merge_kernel_ms, tokens_in and tokens_out (OPT_KERNEL_TIMING)
belong to it alone.  The replayed merges and counts must equal those of one train(K) call, and the calls' tokens_in
must add up to that call's (a call split into two passes would read the stream twice).

Bytes of a pass: 4·tokens_in read + 4·tokens_out written, over its kernel time (as bench.py's roofline.achieved).
Each pass time is the median over --runs replays.  BPE_LIB_PATH selects another build of libb200bpe.so.

Usage: python bench_merge_passes.py [--size-mib 1024] [--warmup 3] [--steps 32] [--runs 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def window_partition(raw, offs, W, K):
    """Member counts of the passes of train(K, first_idx=256+W) after train(W), from the host model."""
    import oracle
    from batch_model import partition
    ub, uo, uw = oracle.c_dedup_chunks(raw, offs)
    ids = ub.astype(np.int32)
    head = partition(ids, uo, W, weights=uw)
    win = partition(head.final, head.final_offs, K, first_idx=256 + W, weights=uw)
    return win.sizes, win.merges, win.counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=1024)
    ap.add_argument("--seed", type=int, default=1337)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    import bench
    W, K = a.warmup, a.steps

    raw, offs, _ = bench.make_corpus(a.size_mib << 20, a.seed)
    t0 = time.perf_counter()
    sizes, model_merges, model_counts = window_partition(raw, offs, W, K)
    model_s = time.perf_counter() - t0

    import torch
    from minbpe_b200 import engine as E
    torch.cuda.set_device(0)
    gpu = bench.gpu_identity(0)
    eng = E.Engine(0)
    eng.set_option(E.OPT_KERNEL_TIMING, 1)
    eng.set_option(E.OPT_HIST_KERNEL, 2)   # as bench.py's timed window

    # the window in one call: the merges, counts and tokens_in the replay must reproduce
    eng.load_stream(raw, offs)
    eng.train(W)
    ref_p, ref_c, done = eng.train(K, first_idx=256 + W)
    tm = eng.timing()
    assert done == K
    assert np.array_equal(ref_p, model_merges) and np.array_equal(ref_c, model_counts), "device window != host model"
    whole = {"merge_kernel_ms": tm["merge_kernel_ms"], "loop_ms": tm["loop_ms"], "tokens_in": int(tm["tokens_in"]),
             "tokens_out": int(tm["tokens_out"])}

    per_run = []
    for _ in range(a.runs):
        eng.load_stream(raw, offs)
        eng.train(W)
        torch.cuda.synchronize()
        got_p, got_c, rows, i = [], [], [], W
        for nk in sizes:
            p, c, d = eng.train(nk, first_idx=256 + i)
            assert d == nk
            t = eng.timing()
            rows.append((t["merge_kernel_ms"], int(t["tokens_in"]), int(t["tokens_out"])))
            got_p.append(p)
            got_c.append(c)
            i += nk
        assert np.array_equal(np.concatenate(got_p), ref_p) and np.array_equal(np.concatenate(got_c), ref_c), \
            "replayed passes != one train(K) call"
        assert sum(r[1] for r in rows) == whole["tokens_in"], "a replayed call took more than one pass"
        per_run.append(rows)
    eng.close()

    passes = []
    for k, nk in enumerate(sizes):
        ms = float(np.median([run[k][0] for run in per_run]))
        n_in, n_out = per_run[0][k][1], per_run[0][k][2]
        passes.append({"members": nk, "kernel_ms": round(ms, 4), "tokens_in": n_in, "tokens_out": n_out,
                       "replaced_frac": round((n_in - n_out) / n_in, 5), "GBps": round(4.0 * (n_in + n_out) / (ms / 1e3) / 1e9, 1)})
    groups = {}
    for nk in sorted(set(sizes)):
        sel = [p for p in passes if p["members"] == nk]
        ms = sum(p["kernel_ms"] for p in sel)
        byt = sum(4.0 * (p["tokens_in"] + p["tokens_out"]) for p in sel)
        groups[str(nk)] = {"passes": len(sel), "kernel_ms": round(ms, 3), "GBps": round(byt / (ms / 1e3) / 1e9, 1)}
    one = [p for p in passes if p["members"] == 1]
    many = [p for p in passes if p["members"] > 1]

    def rate(sel):
        ms = sum(p["kernel_ms"] for p in sel)
        return sum(4.0 * (p["tokens_in"] + p["tokens_out"]) for p in sel) / (ms / 1e3) / 1e9 if sel else None

    r1, rb = rate(one), rate(many)
    peak, peak_src = bench.measured_peak()
    print(json.dumps({
        "metric": "merge_pass_GBps", "gpu": gpu, "lib": E.LIB_PATH,
        "window": f"cfg3 {a.size_mib} MiB seed {a.seed}, merges {W}..{W + K - 1}", "runs": a.runs, "model_s": round(model_s, 1),
        "pass_members": sizes, "whole_window": whole,
        "kernel_ms_sum": round(sum(p["kernel_ms"] for p in passes), 3),
        "one_member_GBps": r1, "batched_GBps": rb, "batched_over_one": (rb / r1) if (r1 and rb) else None,
        "peak_GBps": peak, "peak_source": peak_src, "by_members": groups, "passes": passes}), flush=True)


if __name__ == "__main__":
    main()
