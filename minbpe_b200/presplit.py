"""
Host pre-split for large corpora: the reference's ``regex.findall(pattern, text)`` (regex.py:41)
run on several host cores and returned as chunk start offsets (bytes) instead of a list of str.

The GPT-2/GPT-4/o200k split patterns can be restarted at any point that lies between a letter and a
following U+0020: no alternative of these patterns matches a letter followed by a space inside
one chunk (DESIGN.md §17 for o200k), and the patterns have no look-behind, so findall(left) + findall(right) ==
findall(whole) at such a cut (SURVEY.md §8e; tests/test_host.py::test_parallel_split checks it
against single-process findall).  For any other pattern the split runs in one process.
"""
import multiprocessing as mp
import os

import numpy as np
import regex as re

from .tokenizer import GPT2_SPLIT_PATTERN, GPT4_SPLIT_PATTERN, O200K_SPLIT_PATTERN


def host_cores():
    """Cores this process may really use: the affinity mask capped by the cgroup CPU quota (a 128-thread box
    with cpu.max = 16 cores runs 64 workers at a quarter speed each — the round-1 reference arm did that)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(int(q) / int(per))))
    except Exception:  # noqa: BLE001
        pass
    return max(1, n)


_SAFE_PATTERNS = (GPT2_SPLIT_PATTERN, GPT4_SPLIT_PATTERN, O200K_SPLIT_PATTERN)
_G = {}


def chunk_offsets_1proc(compiled, data):
    """Chunk start offsets (uint64, bytes) of ``data`` (utf-8 bytes); requires the matches to tile
    the text, which holds for the GPT-2/GPT-4 patterns (SURVEY.md Appendix A.9)."""
    text = bytes(data).decode("utf-8")
    chunks = compiled.findall(text)
    if not chunks:
        return np.zeros(0, dtype=np.uint64)
    char_len = np.fromiter(map(len, chunks), dtype=np.int64, count=len(chunks))
    if int(char_len.sum()) != len(text) or int(char_len.min()) <= 0:
        raise ValueError("pattern does not tile the text; use RegexTokenizer.train(text) instead")
    char_off = np.zeros(len(chunks), dtype=np.int64)
    np.cumsum(char_len[:-1], out=char_off[1:])
    if len(text) == len(data):
        return char_off.astype(np.uint64)
    raw = np.frombuffer(data, dtype=np.uint8)
    return np.flatnonzero((raw & 0xC0) != 0x80)[char_off].astype(np.uint64)


def safe_cuts(raw, n_pieces):
    """About n_pieces-1 cut positions p with raw[p-1] an ASCII letter and raw[p] == 0x20."""
    n = raw.size
    cuts = []
    for k in range(1, n_pieces):
        lo = n * k // n_pieces
        window = raw[lo: min(n, lo + (1 << 20))]
        prev = window[:-1]
        is_letter = ((prev >= 65) & (prev <= 90)) | ((prev >= 97) & (prev <= 122))
        hit = np.flatnonzero(is_letter & (window[1:] == 32))
        if hit.size:
            p = lo + int(hit[0]) + 1
            if not cuts or p > cuts[-1]:
                cuts.append(p)
    return cuts


def _work(args):
    lo, hi = args
    return chunk_offsets_1proc(_G["compiled"], _G["raw"][lo:hi].tobytes()) + np.uint64(lo)


def chunk_offsets(pattern, data, workers=None):
    """Chunk start offsets of utf-8 ``data`` (bytes / uint8 array) under ``pattern``."""
    raw = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    compiled = re.compile(pattern)
    workers = workers or min(host_cores(), 64)
    if pattern not in _SAFE_PATTERNS or workers <= 1 or raw.size < (8 << 20):
        return chunk_offsets_1proc(compiled, raw.tobytes())
    pieces = max(workers * 4, 1)
    cuts = [0] + safe_cuts(raw, pieces) + [raw.size]
    spans = [(a, b) for a, b in zip(cuts[:-1], cuts[1:]) if b > a]
    _G["compiled"], _G["raw"] = compiled, raw
    try:
        with mp.get_context("fork").Pool(workers) as pool:
            parts = pool.map(_work, spans)
    finally:
        _G.clear()
    return np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint64)
