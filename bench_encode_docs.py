#!/usr/bin/env python3
"""Encoding many documents (RegexTokenizer.encode_ordinary_batch: bpe_encode_docs, DESIGN.md §16) on one H100.  Prints one
JSON line.

  The 1 GiB cfg3 corpus (synthetic, seed 1337) cut into documents of log-normal length around 4 KiB at letter+space points,
  as bench_dedup_docs.py cuts it, encoded with a 32,512-merge table (train_from_file(dedup=True) on the same bytes).  The
  documents are handed to encode_ordinary_batch in groups of --group-mib (a caller that streams a dataset), and the lists
  it returns are dropped after the checks.  Reported per run:
    host_assembly_s   the method's own Python up to its device call: checks, utf-8 encode, join, offsets
    device_s          the Engine.encode_docs calls (upload, split, memo encode, ids back), wall time
    list_building_s   after the device call: one list of ids per document
    documents/s, MiB/s of the whole method
  A group of --group-mib >= ITERATOR_BATCH_BYTES is one device call, so the three add up to the method's time.
  Parity: the cuts are provable chunk boundaries, so the ids of a group's documents, concatenated, must equal
  encode_text_gpt4 of the group's bytes; and on the first --loop-docs documents the batch must equal the per-document
  encode_ordinary loop, which is timed as the comparison.

Usage: python bench_encode_docs.py [--mib 1024] [--doc-kib 4] [--runs 2] [--group-mib 64] [--loop-docs 4000]"""
import argparse
import json
import os
import random
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_dedup import gpu_info  # noqa: E402
from bench_dedup_docs import documents, lognormal_cuts  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--doc-kib", type=float, default=4)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--group-mib", type=int, default=64)
    ap.add_argument("--loop-docs", type=int, default=4000)
    a = ap.parse_args()
    info = gpu_info()
    if "H100" not in info["name"]:
        sys.exit(f"bench_encode_docs.py measures on an H100; device 0 is {info['name']}")
    from minbpe_b200 import RegexTokenizer
    from minbpe_b200.synth import generate
    V = 32768

    raw = generate(1337, a.mib << 20)
    sp = np.flatnonzero(raw[1:] == 0x20) + 1
    prev = raw[sp - 1]
    points = sp[((prev >= 0x41) & (prev <= 0x5A)) | ((prev >= 0x61) & (prev <= 0x7A))]
    ends = lognormal_cuts(raw.size, points, a.doc_kib * 1024, random.Random(1337))
    docs = documents(raw, ends)
    lens = np.diff(np.asarray([0] + ends))
    tok = RegexTokenizer()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "cfg3.txt")
        raw.tofile(path)
        t0 = time.perf_counter()
        tok.train_from_file(path, V, dedup=True)
        train_s = time.perf_counter() - t0
    groups, g0, size = [], 0, 0                     # document index ranges of about group_mib each
    for j, n in enumerate(lens.tolist()):
        size += n
        if size >= a.group_mib << 20 or j + 1 == len(lens):
            groups.append((g0, j + 1, ends[g0 - 1] if g0 else 0, ends[j]))
            g0, size = j + 1, 0
    out = {"gpu": info, "mib": a.mib, "vocab": V, "merges": len(tok.merges), "train_from_file_dedup_s": round(train_s, 3),
           "documents": len(docs), "doc_bytes_median": int(np.median(lens)), "doc_bytes_mean": round(float(lens.mean()), 1),
           "group_mib": a.group_mib, "groups": len(groups), "batch_bytes": RegexTokenizer.ITERATOR_BATCH_BYTES}

    eng = tok.engine
    real = eng.encode_docs
    calls = []

    def timed(*args, **kw):
        t0 = time.perf_counter()
        r = real(*args, **kw)
        calls.append((t0, time.perf_counter()))
        return r
    merges = tok._merge_array()
    tok.encode_ordinary_batch(docs[: groups[0][1]])           # warm-up: tables, memo, buffers
    runs = []
    for _ in range(a.runs):
        eng.encode_docs = timed
        total = dev = lst = 0.0
        n_ids = n_calls = 0
        equal = True
        for d0, d1, b0, b1 in groups:
            calls.clear()
            t0 = time.perf_counter()
            got = tok.encode_ordinary_batch(docs[d0:d1])
            t1 = time.perf_counter()
            total += t1 - t0
            dev += sum(e - s for s, e in calls)
            lst += t1 - calls[-1][1]
            n_calls += len(calls)
            whole = eng.encode_text_gpt4(raw[b0:b1].tobytes(), merges)
            n_ids += int(whole.size)
            equal = equal and np.array_equal(np.concatenate([np.asarray(d, dtype=np.int32) for d in got]), whole)
            del got
        del eng.encode_docs
        st = eng.encode_stats()
        runs.append({"total_s": round(total, 3), "host_assembly_s": round(total - dev - lst, 3), "device_s": round(dev, 3),
                     "list_building_s": round(lst, 3), "documents_per_s": round(len(docs) / total, 1),
                     "mib_per_s": round(a.mib / total, 1), "device_mib_per_s": round(a.mib / dev, 1), "ids": n_ids,
                     "device_calls": n_calls,
                     "ids_equal_whole_text_encode": bool(equal), "last_call_pieces": st["pieces"],
                     "last_call_new_chunks": st["new_chunks"], "last_call_fallback_pieces": st["fallback_pieces"]})
    out["runs"] = runs

    # the comparison: the per-document encode loop on the first loop_docs documents
    few = docs[: a.loop_docs]
    t0 = time.perf_counter()
    loop = [tok.encode_ordinary(d) for d in few]
    loop_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    batch = tok.encode_ordinary_batch(few)
    batch_s = time.perf_counter() - t0
    fb = sum(len(d.encode("utf-8")) for d in few) / 2 ** 20
    out["loop"] = {"documents": len(few), "mib": round(fb, 2), "per_document_loop_s": round(loop_s, 3),
                   "loop_documents_per_s": round(len(few) / loop_s, 1), "batch_s": round(batch_s, 3),
                   "batch_documents_per_s": round(len(few) / batch_s, 1), "speedup": round(loop_s / batch_s, 2),
                   "ids_equal": batch == loop}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
