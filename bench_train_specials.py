#!/usr/bin/env python3
"""Training with special tokens (DESIGN.md §18) on one H100.  Prints one JSON line.

The 1 GiB synthetic corpus (seed 1337) is cut at letter+space points into documents of log-normal length around 4 KiB, as
in bench_dedup_docs.py, and the documents are joined with <|endoftext|> into a temporary file.  Two runs alternate, `runs`
times each, to vocab 32,768:
  specials   train_from_file(path, dedup=True, special_tokens={"<|endoftext|>": 32768}): the counting session finds the
             separators on the device (spec_find) and leaves them out of the count
  iterator   train_from_iterator(documents) without specials, on the same documents
Both train on the same chunks, so their merges and counts must be identical.  Reported per run: load (split + count, all
that comes before the merge loop), the merge loop, chunks and entries; the card's name and power limit are read in the same
run.

Usage: python bench_train_specials.py [--mib 1024] [--doc-kib 4] [--runs 3]"""
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

EOT = "<|endoftext|>"


def timed_run(tok, fn):
    """fn() trains tok; -> (total s, merge loop s, pairs, counts): the engine's train call is timed and its result kept"""
    eng, got = tok.engine, {}
    train = eng.train

    def wrapped(*a, **k):
        t0 = time.perf_counter()
        r = train(*a, **k)
        got["loop"], got["r"] = time.perf_counter() - t0, r
        return r
    eng.train = wrapped
    t0 = time.perf_counter()
    try:
        fn()
    finally:
        del eng.train
    return time.perf_counter() - t0, got["loop"], got["r"][0], got["r"][1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--doc-kib", type=float, default=4)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    info = gpu_info()
    if "H100" not in info["name"]:
        sys.exit(f"bench_train_specials.py measures on an H100; device 0 is {info['name']}")
    from minbpe_b200 import RegexTokenizer
    from minbpe_b200.synth import generate
    V = 32768
    raw = generate(1337, a.mib << 20)
    sp = np.flatnonzero(raw[1:] == 0x20) + 1
    prev = raw[sp - 1]
    points = sp[((prev >= 0x41) & (prev <= 0x5A)) | ((prev >= 0x61) & (prev <= 0x7A))]
    ends = lognormal_cuts(raw.size, points, a.doc_kib * 1024, random.Random(1337))
    docs = documents(raw, ends)
    del raw
    assert not any(EOT in d for d in docs)
    out = {"gpu": info, "mib": a.mib, "vocab": V, "documents": len(docs)}
    runs = {"specials": [], "iterator": []}
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "docs_eot.txt")
        with open(path, "w", encoding="utf-8") as f:
            f.write(EOT.join(docs))
        out["file_bytes"] = os.path.getsize(path)
        for _ in range(a.runs):
            for name in ("specials", "iterator"):
                tok = RegexTokenizer()
                if name == "specials":
                    fn = lambda: tok.train_from_file(path, V, dedup=True, special_tokens={EOT: V})   # noqa: E731
                else:
                    fn = lambda: tok.train_from_iterator(docs, V)   # noqa: E731
                total, loop, pairs, counts = timed_run(tok, fn)
                st = tok.engine.dedup_stats()
                runs[name].append({"load_s": round(total - loop, 3), "loop_s": round(loop, 3), "total_s": round(total, 3),
                                   "chunks": st["text_chunks"], "entries": st["entries"], "pieces": st["pieces"]})
                key = (pairs.tobytes(), counts.tobytes())
                results.setdefault(name, key)
                runs[name][-1]["same_as_first_run"] = results[name] == key
                del tok
    out["runs"] = runs
    out["merges_and_counts_equal"] = results["specials"] == results["iterator"]
    for name in runs:
        out[name + "_median_load_s"] = float(np.median([r["load_s"] for r in runs[name]]))
        out[name + "_median_loop_s"] = float(np.median([r["loop_s"] for r in runs[name]]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
