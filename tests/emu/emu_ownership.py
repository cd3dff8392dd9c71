#!/usr/bin/env python3
"""TEST INFRASTRUCTURE (run by tests/test_emu_ownership.py in a subprocess with BPE_LIB_PATH = the emulator build).

Device-memory ownership of the host side: the emulator counts live allocations, their bytes and their peak, and live
events (emu_alloc_stats), and can make the k-th cudaMalloc from now fail (emu_fail_alloc).

  released      create, every family below, destroy (per-kernel timing on, so the timing events exist): nothing is left
  sweep FAMILY  for every allocation k of a clean run: with allocation k failing the family returns BPE_ERR_CUDA, the same
                sequence on the same handle then gives the clean output, and destroying the handle leaves nothing live
  peak          a load_stream of 2n bytes after one of n bytes never holds an old and a new stream buffer together
"""
import ctypes
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import regex  # noqa: E402

from minbpe_b200 import engine as E  # noqa: E402
from minbpe_b200.tokenizer import GPT4_SPLIT_PATTERN, split_text  # noqa: E402

LIB = E.load_library()
LIB.emu_alloc_stats.argtypes = [ctypes.POINTER(ctypes.c_ulonglong)]
LIB.emu_fail_alloc.argtypes = [ctypes.c_ulonglong]
SPECIAL = (b"<|endoftext|>", 100257)


def stats():
    """-> (live allocations, live bytes, peak live bytes since the last call, live events, cudaMalloc calls so far)"""
    a = (ctypes.c_ulonglong * 5)()
    LIB.emu_alloc_stats(a)
    return tuple(int(x) for x in a)


def _text(n_words, seed):
    rng = random.Random(seed)
    words = ["the", "token", "merges", "pairs", "of", "bytes", "123", "45678", "don't", "GPU", "été", "日本",
             "\n", "!!", "x"]
    return "".join(rng.choice(words) + (" " if rng.random() < 0.7 else "") for _ in range(n_words))


TEXT = _text(600, 1)
DATA, OFFS = split_text(regex.compile(GPT4_SPLIT_PATTERN), TEXT)
LONG_TEXT = _text(16000, 2)                     # >= 64 KiB: the memoised encode path
LONG_DATA, LONG_OFFS = split_text(regex.compile(GPT4_SPLIT_PATTERN), LONG_TEXT)
assert len(LONG_DATA) >= 1 << 16
SPEC_TEXT = TEXT[:900] + "<|endoftext|>" + TEXT[900:1800] + "<|endoftext|>" + TEXT[1800:]
DOCS = [TEXT[i:i + 500].encode() for i in range(0, len(TEXT), 500)]


def _merges():
    e = E.Engine(0)
    e.load_stream(DATA, OFFS)
    pairs, _, _ = e.train(40)
    e.close()
    return pairs


MERGES = _merges()


def _vocab():
    toks = [bytes([i]) for i in range(256)]
    for a, b in MERGES:
        toks.append(toks[a] + toks[b])
    vb = np.frombuffer(b"".join(toks), dtype=np.uint8)
    vl = np.array([len(t) for t in toks], dtype=np.uint32)
    vs = np.zeros(len(toks), dtype=np.uint64)
    np.cumsum(vl[:-1], out=vs[1:])
    return vb, vs, vl


def _weighted():
    chunks = {}
    for s, t in zip(OFFS, list(OFFS[1:]) + [len(DATA)]):
        chunks[bytes(DATA[s:t])] = chunks.get(bytes(DATA[s:t]), 0) + 1
    data = b"".join(chunks)
    offs = np.cumsum([0] + [len(c) for c in chunks][:-1]).astype(np.uint64)
    return data, offs, np.array(list(chunks.values()), dtype=np.uint64)


def _train(e):
    return e.train(30)


def _weighted_train(e):
    e.set_option(E.OPT_SEG_FILTER, 0)           # not on a weighted stream (a family before it may have switched it on)
    return e.train(30)


def f_train(e):
    e.set_option(E.OPT_TABLE_LOG2, 10)          # small table: the loop grows it (rehash)
    e.load_stream(DATA, OFFS)
    return _train(e)


def f_train_filter(e):
    e.set_option(E.OPT_SEG_FILTER, 2)
    e.load_stream(DATA, OFFS)
    return _train(e)


def f_ids(e):
    ids = np.frombuffer(DATA, dtype=np.uint8).astype(np.int32)
    e.load_ids(ids, OFFS)
    e.merge(int(MERGES[0][0]), int(MERGES[0][1]), 256)
    return e.get_stats()


def f_replay(e):
    e.load_stream(DATA, OFFS)
    e.replay(MERGES)
    return e.read_stream()


def f_encode_short(e):
    return e.encode(DATA, OFFS, MERGES)


def f_encode_long(e):
    e.set_option(E.OPT_ENC_MEMO_LOG2, 6)        # a tiny memo: pieces fall back to the general path
    return e.encode(LONG_DATA, LONG_OFFS, MERGES)


def f_encode_text(e):
    return e.encode_text_gpt4(TEXT.encode(), MERGES)


def f_encode_special(e):
    return e.encode_text_gpt4(SPEC_TEXT.encode(), MERGES, specials=[SPECIAL])


def f_decode(e):
    ids = np.concatenate([np.arange(256 + len(MERGES), dtype=np.int32), np.frombuffer(DATA[:300], dtype=np.uint8).astype(np.int32)])
    return e.decode(ids, *_vocab())


def f_session(e):
    e.set_option(E.OPT_DEDUP_LOG2, 6)           # a small chunk table: entries without a slot as well
    e.dedup_begin()
    doc_offs = np.cumsum([0] + [len(d) for d in DOCS][:-1]).astype(np.uint64)
    e.dedup_add_docs(b"".join(DOCS), doc_offs)
    e.dedup_add_docs(DOCS[0], [0])
    r1 = (e.dedup_finish(), e.chunk_entries(), e.chunk_weights())
    return r1, e.load_text_gpt4_dedup(TEXT.encode()), e.chunk_entries(), e.chunk_weights()


def f_weighted(e):
    e.load_chunks_weighted(*_weighted())
    return _weighted_train(e)


def f_weighted_dedup(e):
    data, offs, w = _weighted()
    half = len(offs) // 2
    both = data + data[:int(offs[half])]        # the first half twice: equal entries merge
    offs2 = np.concatenate([offs, offs[:half] + len(data)]).astype(np.uint64)
    e.load_chunks_weighted_dedup(both, offs2, np.concatenate([w, w[:half]]))
    return _weighted_train(e)


FAMILIES = {
    "train": f_train, "train_filter": f_train_filter, "ids": f_ids, "replay": f_replay, "encode_short": f_encode_short,
    "encode_long": f_encode_long, "encode_text": f_encode_text, "encode_special": f_encode_special, "decode": f_decode,
    "session": f_session, "weighted": f_weighted, "weighted_dedup": f_weighted_dedup,
}


def same(a, b):
    if isinstance(a, (tuple, list)):
        return isinstance(b, (tuple, list)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return np.array_equal(np.asarray(a), np.asarray(b))
    return a == b


def expect_cuda_error(fn, what):
    try:
        fn()
    except E.EngineError as ex:
        assert "failed (-1)" in str(ex), f"{what}: not BPE_ERR_CUDA: {ex}"
        return
    raise AssertionError(f"{what}: the failed allocation was not reported")


def check_released(base, what):
    live = stats()
    assert live[0] == base[0] and live[3] == base[3], f"{what}: {live[0] - base[0]} allocations, {live[3] - base[3]} events left live"


def released():
    base = stats()
    e = E.Engine(0)
    e.set_option(E.OPT_KERNEL_TIMING, 1)
    for name, fn in FAMILIES.items():
        fn(e)
    e.close()
    check_released(base, "released")


def sweep(name):
    if name == "create":
        base = stats()
        E.Engine(0).close()
        n = stats()[4] - base[4]
        for k in range(1, n + 1):
            LIB.emu_fail_alloc(k)
            expect_cuda_error(lambda: E.Engine(0), f"create, allocation {k}")
            LIB.emu_fail_alloc(0)
            check_released(base, f"create, allocation {k}")
            E.Engine(0).close()
            check_released(base, f"create, allocation {k}")
        return n
    fn = FAMILIES[name]
    base = stats()
    e = E.Engine(0)
    before = stats()[4]
    want = fn(e)
    n = stats()[4] - before
    e.close()
    check_released(base, f"{name}, clean run")
    assert n > 0, f"{name}: no allocation"
    for k in range(1, n + 1):
        e = E.Engine(0)
        LIB.emu_fail_alloc(k)
        expect_cuda_error(lambda: fn(e), f"{name}, allocation {k}")
        LIB.emu_fail_alloc(0)
        got = fn(e)
        assert same(got, want), f"{name}, allocation {k}: the run after the failure differs from the clean run"
        e.close()
        check_released(base, f"{name}, allocation {k}")
    return n


def peak():
    # A second load of 2n bytes after one of n grows the two stream buffers.  The staging copies of that call (the text
    # piece, the offsets piece) are 2n + 256 bytes; one old stream buffer (4 bytes per token of the first load, 4n bytes)
    # does not fit under that margin, so holding an old buffer and a new one together exceeds the bound.
    n = 1 << 16
    text = np.frombuffer(_text(n, 3).encode()[:2 * n], dtype=np.uint8)
    assert text.size == 2 * n
    e = E.Engine(0)
    e.load_stream(text[:n])
    before = stats()[1]                         # the peak restarts here
    e.load_stream(text)
    live, peak_bytes = stats()[1:3]
    staging = ((2 * n + 255) & ~255) + 256
    e.close()
    assert live > before, "the second load did not grow the stream buffers"
    assert peak_bytes <= live + staging, f"peak {peak_bytes} > live {live} + staging {staging}: old and new stream buffers coexisted"

if __name__ == "__main__":
    what = sys.argv[1]
    if what == "released":
        released()
    elif what == "peak":
        peak()
    else:
        print(f"{what}: {sweep(what)} allocations swept")
    print("ok")
