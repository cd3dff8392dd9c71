#!/usr/bin/env python3
"""Training on the distinct chunks of a file across N ranks (dist.train_file_dedup, DESIGN.md §14): the phases of the
sharded load, and the unsharded dedup path for comparison.  Prints one JSON line.

One process (no torchrun): the ranks N = 1, 2, 4, 8 are played one after another on GPU 0, on the cfg4 corpus (4 GiB
synthetic, seed 1338) and on a high-cardinality corpus of random lowercase words (seed 7).  Per N: the time each shard
takes to count its distinct chunks (bpe_load_text_gpt4_dedup of its byte range), to read them back (chunk_entries +
chunk_weights), the host concatenation, the merge on the device (bpe_load_chunks_weighted_dedup) and the merge loop.
Entries, weights, merges and counts must equal those of one bpe_load_text_gpt4_dedup of the whole file.  On one GPU the
wall time N GPUs would need for the load is not measured: "estimated_load_ms" = slowest shard (count + read back) +
concatenation + merge is an estimate and is labelled so.

Under torchrun with more than one rank (one GPU per rank, NCCL): the same phases on the real group, the all-gather
included, each the maximum over the ranks.

The corpora are written to a temporary file (the ranks map it, as train_file_dedup does) and removed afterwards.

Usage: python bench_dedup_sharded.py [--mib 4096] [--words-mib 256] [--merges 32512] [--ranks 1,2,4,8]"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader,nounits", "-i", str(index)],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1]), "sm_clock_mhz": float(q[2])}


def words_corpus(seed, nbytes, pool=1 << 21, block=16 << 20):
    """`nbytes` of lowercase words of 3..10 random letters, separated by spaces, drawn from a pool of `pool` words."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(3, 11, size=pool)
    letters = rng.integers(97, 123, size=int(lens.sum()), dtype=np.uint8)
    starts = np.zeros(pool, dtype=np.int64)
    starts[1:] = np.cumsum(lens[:-1])
    out = np.empty(nbytes, dtype=np.uint8)
    pos = 0
    while pos < nbytes:
        pick = rng.integers(0, pool, size=block // 7)
        wl = lens[pick] + 1                                       # the word and a space
        ends = np.cumsum(wl)
        total = int(ends[-1])
        rel = np.arange(total, dtype=np.int64) - np.repeat(ends - wl, wl)   # position inside its word
        src = np.repeat(starts[pick], wl) + rel
        blk = letters[np.minimum(src, letters.size - 1)]
        blk[np.repeat(wl - 1, wl) == rel] = 32
        m = min(total, nbytes - pos)
        out[pos:pos + m] = blk[:m]
        pos += m
    out[-1] = 10
    return out


def temp_file(raw):
    for d in (tempfile.gettempdir(), "/dev/shm"):
        if os.path.isdir(d) and shutil.disk_usage(d).free > raw.size + (1 << 30):
            fd, path = tempfile.mkstemp(suffix=".txt", dir=d)
            os.close(fd)
            raw.tofile(path)
            return path
    raise SystemExit(f"no temporary directory with {raw.size >> 20} MiB free for the corpus")


def ms(t0):
    return round((time.perf_counter() - t0) * 1e3, 1)


def play(eng, path, world, merges, ref):
    """Every rank's count and read-back on this GPU, one after another; then the merge and the loop."""
    from minbpe_b200.dist import shard_byte_range
    size = os.path.getsize(path)
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    count_ms, read_ms, parts = [], [], []
    for r in range(world):
        lo, hi = shard_byte_range(size, r, world, lambda a, b: mm[a:b], empty_tail=True)
        t0 = time.perf_counter()
        nc, _ = eng.load_text_gpt4_dedup(mm[lo:hi])
        count_ms.append(ms(t0))
        t0 = time.perf_counter()
        b, o = eng.chunk_entries()
        parts.append((b, o, eng.chunk_weights(), nc))
        read_ms.append(ms(t0))
    del mm
    t0 = time.perf_counter()
    datas = [p[0] for p in parts]
    base = np.cumsum([0] + [d.size for d in datas[:-1]], dtype=np.uint64)
    data = np.concatenate(datas)
    offsets = np.concatenate([p[1] + b for p, b in zip(parts, base)])
    weights = np.concatenate([p[2] for p in parts])
    concat_ms = ms(t0)
    t0 = time.perf_counter()
    n = eng.load_chunks_weighted_dedup(data, offsets, weights)
    merge_ms = ms(t0)
    st = eng.dedup_stats()
    b, o = eng.chunk_entries()
    w = eng.chunk_weights()
    p, c, d = eng.train(merges)
    loop_ms = round(eng.timing()["loop_ms"], 1)
    same = (ref is None or (np.array_equal(b, ref["bytes"]) and np.array_equal(o, ref["offsets"]) and np.array_equal(w, ref["weights"])
                            and np.array_equal(p, ref["pairs"]) and np.array_equal(c, ref["counts"])))
    slowest = max(a + b for a, b in zip(count_ms, read_ms))
    return {"ranks": world, "shard_count_ms": count_ms, "shard_read_back_ms": read_ms, "concat_ms": concat_ms,
            "merge_input_entries": int(offsets.size), "merge_ms": merge_ms, "entries": int(n), "slots_used": st["slots_used"],
            "loop_ms": loop_ms, "merges": int(d), "estimated_load_ms": round(slowest + concat_ms + merge_ms, 1),
            "identical_to_unsharded": bool(same)}


def single_gpu(a):
    from minbpe_b200.engine import Engine
    from minbpe_b200.synth import generate
    info = gpu_info(0)
    if "H100" not in info["name"]:
        sys.exit(f"bench_dedup_sharded.py measures on an H100; device 0 is {info['name']}")
    eng = Engine(0)
    out = {"gpu": info, "mode": "ranks played one after another on one GPU",
           "estimated_load_ms": "max over shards of (count + read back) + concat + merge: an estimate, not a measurement on N GPUs"}
    for name, make in (("cfg4", lambda: generate(1338, a.mib << 20)), ("words", lambda: words_corpus(7, a.words_mib << 20))):
        path = temp_file(make())
        try:
            t0 = time.perf_counter()
            nc, ne = eng.load_text_gpt4_dedup(np.memmap(path, dtype=np.uint8, mode="r"))
            whole_ms = ms(t0)
            b, o = eng.chunk_entries()
            ref = {"bytes": b, "offsets": o, "weights": eng.chunk_weights()}
            ref["pairs"], ref["counts"], d = eng.train(a.merges)
            res = {"mib": os.path.getsize(path) >> 20, "text_chunks": int(nc),
                   "unsharded": {"load_ms": whole_ms, "entries": int(ne), "loop_ms": round(eng.timing()["loop_ms"], 1), "merges": int(d)},
                   "sharded": [play(eng, path, n, a.merges, ref) for n in a.ranks]}
            out[name] = res
        finally:
            os.unlink(path)
    eng.close()
    print(json.dumps(out))


def multi_gpu(a):
    """torchrun: one GPU per rank; every phase's wall time, maximum over the ranks."""
    import torch
    import torch.distributed as dist
    from minbpe_b200.dist import count_file_shard, load_merged_shards
    from minbpe_b200.engine import Engine
    from minbpe_b200.synth import generate
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, world = dist.get_rank(), dist.get_world_size()
    eng = Engine(local)
    out = {"gpu": gpu_info(local), "mode": f"torchrun, {world} ranks, one GPU each; each phase the maximum over the ranks"}
    for name, make in (("cfg4", lambda: generate(1338, a.mib << 20)), ("words", lambda: words_corpus(7, a.words_mib << 20))):
        path = None
        if rank == 0:
            path = temp_file(make())
        box = [path]
        dist.broadcast_object_list(box, src=0)
        path = box[0]
        try:
            times = {}
            dist.barrier()
            t0 = time.perf_counter()
            part = count_file_shard(eng, path, rank, world)
            times["count_and_read_back_ms"] = ms(t0)
            t0 = time.perf_counter()
            parts = [None] * world
            dist.all_gather_object(parts, part)
            times["all_gather_ms"] = ms(t0)
            t0 = time.perf_counter()
            n = load_merged_shards(eng, parts)
            times["concat_and_merge_ms"] = ms(t0)
            p, c, d = eng.train(a.merges)
            times["loop_ms"] = round(eng.timing()["loop_ms"], 1)
            dist.barrier()
            t = torch.tensor(list(times.values()), dtype=torch.float64, device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            res = dict(zip(times, [round(float(x), 1) for x in t.tolist()]))
            res.update(entries=int(n), merges=int(d), mib=os.path.getsize(path) >> 20)
            out[name] = res
        finally:
            dist.barrier()
            if rank == 0:
                os.unlink(path)
    eng.close()
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=4096)
    ap.add_argument("--words-mib", type=int, default=256)
    ap.add_argument("--merges", type=int, default=32512)
    ap.add_argument("--ranks", type=lambda s: [int(x) for x in s.split(",")], default=[1, 2, 4, 8])
    a = ap.parse_args()
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        multi_gpu(a)
    else:
        single_gpu(a)


if __name__ == "__main__":
    main()
