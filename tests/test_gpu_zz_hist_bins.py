"""GPU: the packed byte-pair histogram (k_hist_dense_packed, BPE_OPT_HIST_KERNEL = 1) bin by bin.  Iteration 0's histogram
becomes the pair table, and every later count is that table plus deltas, so after train(1) the whole table
(debug_table) must equal the recount of the stream after that merge: an error in any of the 65,536 bins survives
there, even when the arg-max is right.

The kernel counts into 16-bit halves of shared-memory words (bin 2i low, 2i+1 high) and flushes a CTA's table after every
round of HP_ROUND_TOKENS pairs.  The streams hold every byte pair with bins 2i and 2i+1 at different counts (a carry into
the neighbour bin or a lost half shows), with and without chunk marks (at multiples of 512 among them), and one repeated
byte, an even and an odd bin, sized so that a CTA's round holds exactly HP_ROUND_TOKENS pairs of that one bin, and that
size +-1, 511, 512, 513 tokens, for one and two rounds per CTA."""
import os
import re

import numpy as np
import pytest

import oracle
from batch_model import merge, stats, table_dict

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _hp(name):
    with open(os.path.join(ROOT, "minbpe_b200", "csrc", "k_stats.cuh")) as f:
        return int(re.search(rf"#define {name} (\d+)", f.read()).group(1))


HP_THREADS, HP_SEGS_PER_WARP = _hp("HP_THREADS"), _hp("HP_SEGS_PER_WARP")
HP_ROUND_TOKENS = (HP_THREADS // 32) * HP_SEGS_PER_WARP * 512


def _sms():
    """The SM count the library launches k_hist_dense_packed with (one CTA per SM)."""
    if "emu" in os.path.basename(os.environ.get("BPE_LIB_PATH", "")):   # the CPU SIMT emulator's build
        return int(os.environ.get("EMU_SMS", "2"))
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def de_bruijn_256():
    """Order-2 de Bruijn sequence over 256 symbols, closed: 65,537 bytes holding each of the 65,536 pairs once."""
    a = [0] * 512
    seq = []

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1: p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, 256):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    seq.append(seq[0])
    return np.asarray(seq, dtype=np.uint8)


def all_pairs_stream(marks):
    """Every byte pair, bins 2i and 2i+1 at different counts: the de Bruijn sequence, then for every odd bin 1 + (bin >> 9) % 3
    more copies as 2-byte chunks, and 7 more of one pair (a unique arg-max).  marks: chunk starts inside the de Bruijn
    part at every multiple of 512 and at 1000 random places, else one chunk there."""
    db = de_bruijn_256()
    bins = np.arange(65536)
    extra = np.where(bins & 1, 1 + (bins >> 9) % 3, 0)
    extra[0x4142] += 7
    rep = np.repeat(bins, extra)
    tail = np.stack([rep >> 8, rep & 255], axis=1).reshape(-1).astype(np.uint8)
    data = np.concatenate([db, tail])
    offs = [0]
    if marks:
        rng = np.random.default_rng(5)
        offs += list(range(512, len(db), 512)) + rng.integers(1, len(db), 1000).tolist()
    offs += list(range(len(db), len(data), 2))
    return data, np.unique(np.asarray(offs, dtype=np.uint64))


def _check_train1(eng, data, offs):
    eng.load_stream(data, offs)
    p, c, d = eng.train(1)
    assert eng.timing()["hist_kernel"] == 1
    ids = data.astype(np.int32)
    wp, wc, wd, fin = oracle.c_train(ids, offs, 1, want_final=True)
    assert d == wd == 1 and np.array_equal(p, wp) and np.array_equal(c, wc)
    start = np.zeros(len(ids), dtype=bool)
    start[offs.astype(np.int64)] = True
    f_ids, f_start, _ = merge(ids, start, tuple(int(x) for x in wp[0]), 256)
    assert np.array_equal(f_ids, fin)
    assert eng.debug_table() == table_dict(*stats(fin, f_start))


def _engine(kernel=1):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_HIST_KERNEL, kernel)
    return eng


@pytest.mark.parametrize("marks", [False, True])
def test_all_byte_pairs(marks):
    data, offs = all_pairs_stream(marks)
    start = np.zeros(len(data), dtype=bool)
    start[offs.astype(np.int64)] = True
    pairs, counts = stats(data.astype(np.int32), start)
    full = np.zeros(65536, dtype=np.int64)
    full[pairs[:, 0] * 256 + pairs[:, 1]] = counts
    if not marks:
        assert (full > 0).all() and (full[0::2] != full[1::2]).all()     # every bin, neighbours apart
    eng = _engine()
    _check_train1(eng, data, offs)
    eng.close()


def _run_sizes():
    base = _sms() * HP_ROUND_TOKENS
    return [r * base + d for r in (1, 2) for d in (0, 1, -1, 511, -511, 512, -512, 513, -513)]


@pytest.mark.parametrize("byte", [0x62, 0x61])          # bin 0x6262 is even, 0x6161 odd
def test_one_bin_at_the_round_size(byte):
    eng = _engine()
    for n in _run_sizes():
        data = np.full(n, byte, dtype=np.uint8)
        eng.load_stream(data, None)
        p, c, d = eng.train(1)
        assert eng.timing()["hist_kernel"] == 1
        assert d == 1 and p.tolist() == [[byte, byte]] and c.tolist() == [n - 1], n
        # after the merge: n // 2 tokens 256 (and one byte left over when n is odd)
        want = {}
        if n // 2 >= 2:
            want[(256, 256)] = n // 2 - 1
        if n % 2:
            want[(256, byte)] = 1
        assert eng.debug_table() == want, n
    eng.close()


@pytest.mark.skipif(SMALL, reason="8 Mi tokens: too large for the emulator")
def test_large_stream_automatic_choice():
    """BPE_OPT_HIST_KERNEL = 0 at a stream of >= 8 Mi tokens of these shapes: whichever kernel the library adopts, the
    table is bin-exact."""
    data, offs = all_pairs_stream(True)
    reps = -(-(8 << 20) // len(data))
    big = np.tile(data, reps)
    boffs = np.concatenate([offs + np.uint64(k * len(data)) for k in range(reps)])
    eng = _engine(0)
    eng.load_stream(big, boffs)
    p, c, d = eng.train(1)
    assert eng.timing()["hist_kernel"] in (1, 2)
    ids = big.astype(np.int32)
    wp, wc, wd, fin = oracle.c_train(ids, boffs, 1, want_final=True)
    assert np.array_equal(p, wp) and np.array_equal(c, wc)
    start = np.zeros(len(ids), dtype=bool)
    start[boffs.astype(np.int64)] = True
    f_ids, f_start, _ = merge(ids, start, tuple(int(x) for x in wp[0]), 256)
    assert np.array_equal(f_ids, fin)
    assert eng.debug_table() == table_dict(*stats(fin, f_start))
    eng.close()

