#!/usr/bin/env python3
"""Special-token sets of 1 to 65,536 specials on one H100 (DESIGN.md §19).  Prints one JSON line.

The 1 GiB synthetic corpus (seed 1337) is cut at letter+space points into documents of log-normal length around 4 KiB, as
in bench_train_specials.py, and the documents are joined by separators into a temporary file per arm:
  k1       {"<|endoftext|>"}, every separator that one
  llama3   Llama 3's 256 special tokens, the separators drawn from all 256
  k4096    <|reserved_{i}|> for i < 4,096, the separators drawn from all of them
  k65536   <|reserved_{i}|> for i < 65,536, likewise
The corpus holds no "<|", and no special is a prefix of another, so the separators are the only occurrences.  Timed per
arm, `runs` times: encode_file(path, "all") and train_from_file(path, vocab 32,768, special_tokens=set).  The separators are
left out of training, so every arm must give the same merges and counts; encode_file must give the k1 arm's ids once every
special's id is mapped to the k1 separator's.  The bench asserts both.  The matcher's device time (k_special_find, one
launch per 1 GiB piece) is taken from torch.profiler in four more encode_file calls per arm, apart from the timed runs.
The host-path arm encodes a 64 MiB slice with the 256 Llama 3 specials as encode() did when a set was too large for the
device (re.split, then encode_ordinary per part) and as encode() does now on the device; the ids must be identical.
The card's name and power limit are read in the same run.

Usage: python bench_special_sets.py [--mib 1024] [--doc-kib 4] [--runs 2] [--host-mib 64]"""
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
from bench_dedup_docs import lognormal_cuts  # noqa: E402

V = 32768


def llama3_names():
    r = [f"<|reserved_special_token_{i}|>" for i in range(251)]
    return (["<|begin_of_text|>", "<|end_of_text|>"] + r[0:4] + ["<|start_header_id|>", "<|end_header_id|>", r[4], "<|eot_id|>"]
            + r[5:])


ARMS = {"k1": ["<|endoftext|>"], "llama3": llama3_names(), "k4096": [f"<|reserved_{i}|>" for i in range(4096)],
        "k65536": [f"<|reserved_{i}|>" for i in range(65536)]}


def write_arm(path, raw, ends, names, seed):
    """the documents joined by separators drawn from `names` (the same draw sequence for every arm)"""
    rng = random.Random(seed)
    seps = [n.encode() for n in names]
    with open(path, "wb") as f:
        prev = 0
        for e in ends:
            f.write(raw[prev:e].tobytes())
            if e < raw.size:
                f.write(seps[rng.randrange(len(seps))])
            prev = e


def matcher_ms(tok, path, pieces, tries=4):
    """device ms of k_special_find summed over the launches of one encode_file, the median over the profiled calls that
    recorded one launch per piece (a trace can miss a launch; such a call is left out), and how many calls that was"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    got = []
    for _ in range(tries):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            tok.encode_file(path, "all")
            torch.cuda.synchronize()
        us, calls = 0.0, 0
        for a in prof.key_averages():
            if "k_special_find" in a.key:
                us += getattr(a, "device_time_total", 0) or getattr(a, "self_device_time_total", 0)
                calls += a.count
        if calls == pieces:
            got.append(us / 1000.0)
    return (float(np.median(got)) if got else None), len(got)


def host_encode(tok, text, special):
    """encode(text, allowed_special=special) through the host split: re.split at the specials, encode_ordinary per part"""
    import regex as re
    ids = []
    for part in re.split("(" + "|".join(re.escape(k) for k in special) + ")", text):
        if part in special:
            ids.append(special[part])
        else:
            ids.extend(tok.encode_ordinary(part))
    return ids


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=1024)
    ap.add_argument("--doc-kib", type=float, default=4)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--host-mib", type=int, default=64)
    a = ap.parse_args()
    info = gpu_info()
    if "H100" not in info["name"]:
        sys.exit(f"bench_special_sets.py measures on an H100; device 0 is {info['name']}")
    from minbpe_b200 import RegexTokenizer
    from minbpe_b200.synth import generate
    raw = generate(1337, a.mib << 20)
    assert b"<|" not in raw.tobytes(), "the corpus holds a '<|': a special could occur outside the separators"
    sp = np.flatnonzero(raw[1:] == 0x20) + 1
    prev = raw[sp - 1]
    points = sp[((prev >= 0x41) & (prev <= 0x5A)) | ((prev >= 0x61) & (prev <= 0x7A))]
    ends = lognormal_cuts(raw.size, points, a.doc_kib * 1024, random.Random(1337))
    out = {"gpu": info, "mib": a.mib, "vocab": V, "documents": len(ends)}
    arms, first_ids, first_train = {}, None, None
    with tempfile.TemporaryDirectory() as tmp:
        for name, names in ARMS.items():
            special = {k: V + i for i, k in enumerate(names)}
            path = os.path.join(tmp, name + ".txt")
            write_arm(path, raw, ends, names, 1)
            r = {"k": len(names), "file_bytes": os.path.getsize(path), "encode_s": [], "train_s": []}
            for _ in range(a.runs):
                tok = RegexTokenizer()
                t0 = time.perf_counter()
                tok.train_from_file(path, V, special_tokens=special)
                r["train_s"].append(round(time.perf_counter() - t0, 3))
                t0 = time.perf_counter()
                ids = tok.encode_file(path, "all")
                r["encode_s"].append(round(time.perf_counter() - t0, 3))
            trained = (list(tok.merges.items()), tok.vocab)
            if first_train is None:
                first_train = trained
            r["same_merges_as_k1"] = trained == first_train
            assert r["same_merges_as_k1"], name
            ids = np.asarray(ids)
            r["ids"] = int(ids.size)
            r["separators"] = int((ids >= V).sum())
            ids[ids >= V] = V
            if first_ids is None:
                first_ids = ids
            r["same_ids_as_k1"] = bool(np.array_equal(ids, first_ids))
            assert r["same_ids_as_k1"], name
            del ids
            pieces = -(-r["file_bytes"] // (1 << 30))
            ms, n = matcher_ms(tok, path, pieces)
            r["matcher_ms"] = None if ms is None else round(ms, 3)
            r["matcher_calls_kept"] = n
            r["matcher_ms_per_gib"] = None if ms is None else round(ms / (r["file_bytes"] / (1 << 30)), 3)
            r["median_encode_s"] = float(np.median(r["encode_s"]))
            r["median_train_s"] = float(np.median(r["train_s"]))
            arms[name] = r
            if name == "llama3":     # the host-path arm on a slice of this file, with the tokenizer just trained
                with open(path, "rb") as f:
                    head = f.read(a.host_mib << 20)
                text = head[: head.rfind(b"<|")].decode("utf-8")
                tok.register_special_tokens(special)
                t0 = time.perf_counter()
                want = host_encode(tok, text, special)
                host_s = time.perf_counter() - t0
                t0 = time.perf_counter()
                got = tok.encode(text, allowed_special="all")
                dev_s = time.perf_counter() - t0
                assert got == want, "device and host paths differ"
                out["host_arm"] = {"k": len(names), "bytes": len(text.encode()), "host_s": round(host_s, 3),
                                   "device_s": round(dev_s, 3), "ids_identical": True}
            del tok
    out["arms"] = arms
    print(json.dumps(out))


if __name__ == "__main__":
    main()
