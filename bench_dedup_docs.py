#!/usr/bin/env python3
"""Training from a stream of documents (RegexTokenizer.train_from_iterator: the counting session of DESIGN.md §15) on one
H100, phase by phase.  Prints one JSON line.

  docs   the 1 GiB cfg3 corpus (synthetic, seed 1337) cut into documents of log-normal length around 4 KiB at letter+space
         points, through train_from_iterator to vocab 32,768.  Reported per run: host batch assembly (the method's own
         Python: encode, join, offsets), device add_docs (split + count), finish, the merge loop, documents/s.  Parity: the
         merges and counts must equal train_from_file(dedup=True) on the same bytes, which holds exactly because the cuts
         are provable chunk boundaries.
  cut    a 64 MiB slice cut at arbitrary character positions (boundaries that change the split): the first 1,024 merges
         and counts must equal the oracle's weighted loop over the per-document `regex` chunks.

Usage: python bench_dedup_docs.py [--mib 1024] [--doc-kib 4] [--runs 2] [--check-mib 64]"""
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


def lognormal_cuts(n, points, doc_bytes, rng):
    """Document ends: log-normal lengths around doc_bytes, each moved to the next allowed point (points sorted)."""
    ends, pos = [], 0
    while True:
        pos = int(pos + max(1.0, rng.lognormvariate(np.log(doc_bytes), 0.8)))
        k = int(np.searchsorted(points, pos))
        if k >= len(points):
            break
        pos = int(points[k])
        ends.append(pos)
    return ends + [n]


def documents(raw, ends):
    docs, prev = [], 0
    for e in ends:
        docs.append(raw[prev:e].tobytes().decode("utf-8"))
        prev = e
    return docs


class Timed:
    """Wall time of the engine calls train_from_iterator makes (each one returns after its device work)."""

    def __init__(self, eng):
        self.eng, self.t = eng, {"add_docs": 0.0, "finish": 0.0, "train": 0.0}
        self.calls = 0
        for name, key in (("dedup_add_docs", "add_docs"), ("dedup_finish", "finish"), ("train", "train")):
            setattr(eng, name, self._wrap(getattr(eng, name), key))

    def _wrap(self, fn, key):
        def f(*a, **k):
            t0 = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                self.t[key] += time.perf_counter() - t0
                self.calls += key == "add_docs"
        return f

    def restore(self):
        for name in ("dedup_add_docs", "dedup_finish", "train"):
            delattr(self.eng, name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--doc-kib", type=float, default=4)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--check-mib", type=int, default=64)
    a = ap.parse_args()
    info = gpu_info()
    if "H100" not in info["name"]:
        sys.exit(f"bench_dedup_docs.py measures on an H100; device 0 is {info['name']}")
    from minbpe_b200 import RegexTokenizer
    from minbpe_b200.synth import generate
    out = {"gpu": info}
    V = 32768

    # ---- the cfg3 corpus as documents cut at letter+space points ----
    raw = generate(1337, a.mib << 20)
    sp = np.flatnonzero(raw[1:] == 0x20) + 1
    prev = raw[sp - 1]
    points = sp[((prev >= 0x41) & (prev <= 0x5A)) | ((prev >= 0x61) & (prev <= 0x7A))]
    ends = lognormal_cuts(raw.size, points, a.doc_kib * 1024, random.Random(1337))
    docs = documents(raw, ends)
    lens = np.diff(np.asarray([0] + ends))
    out["docs"] = {"mib": a.mib, "vocab": V, "documents": len(docs), "doc_bytes_median": int(np.median(lens)),
                   "doc_bytes_mean": round(float(lens.mean()), 1), "batch_bytes": RegexTokenizer.ITERATOR_BATCH_BYTES}
    runs, ref = [], None
    for _ in range(a.runs):
        tok = RegexTokenizer()
        T = Timed(tok.engine)
        t0 = time.perf_counter()
        tok.train_from_iterator(docs, V)
        total = time.perf_counter() - t0
        T.restore()
        ingest = total - T.t["finish"] - T.t["train"]       # iterator + batch assembly + add_docs
        host = ingest - T.t["add_docs"]
        st = tok.engine.dedup_stats()
        runs.append({"total_s": round(total, 3), "host_assembly_s": round(host, 3), "device_add_docs_s": round(T.t["add_docs"], 3),
                     "add_docs_calls": T.calls, "finish_s": round(T.t["finish"], 3), "loop_s": round(T.t["train"], 3),
                     "loop_ms_device": round(tok.last_timing["loop_ms"], 1),
                     "documents_per_s": round(len(docs) / ingest, 1), "ingest_mib_per_s": round(a.mib / ingest, 1),
                     "pieces": st["pieces"], "entries": st["entries"], "text_chunks": st["text_chunks"]})
        key = list(tok.merges.items())
        ref = key if ref is None else ref
        runs[-1]["same_as_first_run"] = key == ref
        del tok
    out["docs"]["runs"] = runs
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "cfg3.txt")
        raw.tofile(path)
        whole = RegexTokenizer()
        t0 = time.perf_counter()
        whole.train_from_file(path, V, dedup=True)
        out["docs"]["train_from_file_dedup_s"] = round(time.perf_counter() - t0, 3)
    out["docs"]["parity_equals_train_from_file_dedup"] = list(whole.merges.items()) == ref
    del docs, whole

    # ---- a slice cut at arbitrary character positions, against the oracle ----
    import regex

    import oracle
    from minbpe_b200.tokenizer import GPT4_SPLIT_PATTERN
    text = raw[: a.check_mib << 20].tobytes().decode("utf-8", errors="ignore")
    rng = random.Random(7)
    cuts, pos = [], 0
    while True:
        pos += max(1, int(rng.lognormvariate(np.log(a.doc_kib * 1024), 0.8)))
        if pos >= len(text):
            break
        cuts.append(pos)
    docs = [text[i:j] for i, j in zip([0] + cuts, cuts + [len(text)])]
    pat = regex.compile(GPT4_SPLIT_PATTERN)
    chunks = [c.encode("utf-8") for d in docs for c in pat.findall(d)]
    offs = np.zeros(len(chunks), dtype=np.uint64)
    offs[1:] = np.cumsum([len(c) for c in chunks[:-1]])
    ub, uo, uw = oracle.c_dedup_chunks(np.frombuffer(b"".join(chunks), dtype=np.uint8), offs)
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, 1024, weights=uw)
    tok = RegexTokenizer()
    tok.train_from_iterator(docs, 256 + 1024)
    eng = tok.engine                  # the counts: the same session through the engine
    eng.dedup_begin()
    for d0 in range(0, len(docs), 4096):
        part = [s.encode("utf-8") for s in docs[d0: d0 + 4096]]
        o = np.zeros(len(part), dtype=np.uint64)
        o[1:] = np.cumsum([len(b) for b in part[:-1]])
        eng.dedup_add_docs(b"".join(part), o)
    eng.dedup_finish()
    p, c, d = eng.train(1024)
    out["cut"] = {"mib": a.check_mib, "documents": len(docs), "merges": 1024,
                  "merges_equal_oracle": bool(wd == d == 1024 and np.array_equal(p, wp)),
                  "counts_equal_oracle": bool(np.array_equal(c, wc)),
                  "tokenizer_merges_equal_oracle": [list(m) for m in tok.merges] == wp.tolist()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
