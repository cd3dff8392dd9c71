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

What k_merge_seg really stores is less: nothing for a segment the pass leaves alone, and for the others only the tail
from the first changed token on.  A host model counts those bytes on a --model-mib prefix of the corpus, whose segments
are the load's 512-token blocks: the window's merges are applied pass by pass, and for every segment the pass touches
the model takes its first replaced or dropped token and its new count.  Two write-back rules are counted, from the
start of the 128-token row of that token (`row`) and from the start of its 32-byte sector (`sector`), each up to the
new count rounded up to 16 bytes.  Per pass, the prefix's stored bytes per token read scale to the pass's tokens_in,
and `real_GBps_<rule>` = (4·tokens_in + stored bytes) / kernel time.  Edge records are left out.

The line also carries the copy ceiling (median of --copy-runs device-to-device copies of a 4 GiB tensor, alternating
direction, as (read + write bytes) / time) and the GPU's name, power limit and the SM clock read every 100 ms during the replays (min, max).

Usage: python bench_merge_passes.py [--size-mib 1024] [--warmup 3] [--steps 32] [--runs 5] [--model-mib 16]"""
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


def writeback_model(raw, offs, head_merges, window_merges, sizes, model_bytes):
    """Per pass of the window: (tokens read, bytes stored under the `row` rule, under the `sector` rule) on a prefix of
    the corpus cut at a chunk start (see the module doc)."""
    from batch_model import SEG_TOKENS, merge
    offs = np.asarray(offs, dtype=np.int64)
    cut = int(offs[np.searchsorted(offs, model_bytes, side="right") - 1]) if offs.size and offs[-1] > 0 else len(raw)
    cut = cut if cut > 0 else len(raw)
    ids = np.frombuffer(raw, dtype=np.uint8)[:cut].astype(np.int32)
    start = np.zeros(len(ids), dtype=bool)
    start[offs[offs < cut]] = True
    start[0] = True
    pos = np.arange(len(ids), dtype=np.int64)
    for j, pair in enumerate(head_merges):
        ids, start, pos = merge(ids, start, tuple(int(x) for x in pair), 256 + j, pos)
    z, k, out = 256 + len(head_merges), 0, []
    for nk in sizes:
        ids0, pos0 = ids, pos
        for pair in window_merges[k:k + nk]:
            ids, start, pos = merge(ids, start, tuple(int(x) for x in pair), z, pos)
            z += 1
        k += nk
        # a token of the stream before the pass changed if it was dropped or now holds another id
        at = np.searchsorted(pos, pos0)
        kept = (at < len(pos)) & (pos[np.minimum(at, len(pos) - 1)] == pos0)
        changed = ~kept
        changed[kept] = ids[at[kept]] != ids0[kept]
        seg0 = pos0 // SEG_TOKENS
        nseg = int(seg0[-1]) + 1 if len(seg0) else 0
        first_idx = np.searchsorted(seg0, np.arange(nseg))             # index of each segment's token 0
        new_count = np.bincount(pos // SEG_TOKENS, minlength=nseg)
        ch = np.flatnonzero(changed)
        first = np.full(nseg, SEG_TOKENS, dtype=np.int64)
        np.minimum.at(first, seg0[ch], ch - first_idx[seg0[ch]])
        hit = first < SEG_TOKENS
        vend = (new_count[hit] + 3) // 4 * 16                            # bytes up to the new end in 16-byte vectors
        row = np.maximum(vend - (first[hit] // 128) * 512, 0).sum()
        sector = np.maximum(vend - (first[hit] // 8) * 32, 0).sum()
        out.append((len(ids0), int(row), int(sector)))
    return out


def copy_ceiling(runs, nbytes=4 << 30):
    """Median (read + write bytes) / time of device-to-device copies of an nbytes tensor, alternating direction."""
    import torch
    a = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    a.fill_(1)
    b.copy_(a)
    torch.cuda.synchronize()
    ts = []
    for i in range(runs):
        src, dst = (a, b) if i % 2 == 0 else (b, a)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src)
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) / 1e3)
    del a, b
    torch.cuda.empty_cache()
    t = float(np.median(ts))
    return {"bytes_per_copy": nbytes, "runs": runs, "median_s": round(t, 5), "GBps": round(2.0 * nbytes / t / 1e9, 1)}


def clock_sampler(gpu=0):
    """nvidia-smi reading the SM clock (MHz) every 100 ms until clock_samples stops it; None where it cannot start."""
    import subprocess
    try:
        return subprocess.Popen(["nvidia-smi", "-i", str(gpu), "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                 "-lms", "100"], text=True, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    except Exception:
        return None


def clock_samples(proc):
    """Stop the sampler: {min, max, samples} of the SM clocks it read, or None."""
    if proc is None:
        return None
    proc.terminate()
    try:
        out = proc.communicate(timeout=30)[0]
    except Exception:
        proc.kill()
        out = proc.communicate()[0]
    mhz = [float(x) for x in out.split() if x.replace(".", "", 1).isdigit()]
    return {"min": min(mhz), "max": max(mhz), "samples": len(mhz)} if mhz else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mib", type=int, default=1024)
    ap.add_argument("--seed", type=int, default=1337)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--model-mib", type=int, default=16)
    ap.add_argument("--copy-runs", type=int, default=7)
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
    head_p, _, _ = eng.train(W)
    ref_p, ref_c, done = eng.train(K, first_idx=256 + W)
    tm = eng.timing()
    assert done == K
    assert np.array_equal(ref_p, model_merges) and np.array_equal(ref_c, model_counts), "device window != host model"
    whole = {"merge_kernel_ms": tm["merge_kernel_ms"], "loop_ms": tm["loop_ms"], "tokens_in": int(tm["tokens_in"]),
             "tokens_out": int(tm["tokens_out"])}

    t0 = time.perf_counter()
    wb = writeback_model(raw, offs, head_p, ref_p, sizes, a.model_mib << 20)
    model_s += time.perf_counter() - t0

    per_run = []
    sampler = clock_sampler(0)   # the SM clock while the replays run
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
    clocks = clock_samples(sampler)
    eng.close()
    ceiling = copy_ceiling(a.copy_runs)

    passes = []
    for k, nk in enumerate(sizes):
        ms = float(np.median([run[k][0] for run in per_run]))
        n_in, n_out = per_run[0][k][1], per_run[0][k][2]
        m_in, m_row, m_sector = wb[k]
        w_row, w_sector = n_in * m_row / m_in, n_in * m_sector / m_in    # stored bytes, scaled to the whole stream
        passes.append({"members": nk, "kernel_ms": round(ms, 4), "tokens_in": n_in, "tokens_out": n_out,
                       "replaced_frac": round((n_in - n_out) / n_in, 5), "GBps": round(4.0 * (n_in + n_out) / (ms / 1e3) / 1e9, 1),
                       "write_bytes_row": int(w_row), "write_bytes_sector": int(w_sector),
                       "real_GBps_row": round((4.0 * n_in + w_row) / (ms / 1e3) / 1e9, 1),
                       "real_GBps_sector": round((4.0 * n_in + w_sector) / (ms / 1e3) / 1e9, 1)})
    groups = {}
    for nk in sorted(set(sizes)):
        sel = [p for p in passes if p["members"] == nk]
        ms = sum(p["kernel_ms"] for p in sel)
        byt = sum(4.0 * (p["tokens_in"] + p["tokens_out"]) for p in sel)
        real = {r: round(sum(4.0 * p["tokens_in"] + p["write_bytes_" + r] for p in sel) / (ms / 1e3) / 1e9, 1) for r in ("row", "sector")}
        groups[str(nk)] = {"passes": len(sel), "kernel_ms": round(ms, 3), "GBps": round(byt / (ms / 1e3) / 1e9, 1),
                           "real_GBps_row": real["row"], "real_GBps_sector": real["sector"]}
    one = [p for p in passes if p["members"] == 1]
    many = [p for p in passes if p["members"] > 1]

    def rate(sel):
        ms = sum(p["kernel_ms"] for p in sel)
        return sum(4.0 * (p["tokens_in"] + p["tokens_out"]) for p in sel) / (ms / 1e3) / 1e9 if sel else None

    r1, rb = rate(one), rate(many)
    peak, peak_src = bench.measured_peak()
    print(json.dumps({
        "metric": "merge_pass_GBps", "gpu": gpu, "sm_clock_mhz": clocks, "lib": E.LIB_PATH,
        "window": f"cfg3 {a.size_mib} MiB seed {a.seed}, merges {W}..{W + K - 1}", "runs": a.runs, "model_s": round(model_s, 1),
        "pass_members": sizes, "whole_window": whole,
        "kernel_ms_sum": round(sum(p["kernel_ms"] for p in passes), 3),
        "one_member_GBps": r1, "batched_GBps": rb, "batched_over_one": (rb / r1) if (r1 and rb) else None,
        "peak_GBps": peak, "peak_source": peak_src, "copy_ceiling": ceiling,
        "write_model": {"prefix_mib": a.model_mib, "row_over_sector": round(sum(p["write_bytes_row"] for p in passes) /
                                                                            max(1, sum(p["write_bytes_sector"] for p in passes)), 4)},
        "by_members": groups, "passes": passes}), flush=True)


if __name__ == "__main__":
    main()
