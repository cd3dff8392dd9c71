"""GPU: every warp fold of equal keys with __match_any_sync, on the layouts where a warp's lanes leave a segment at
different trips.

Three kernels fold a warp's equal keys and let the lowest lane of each group add the group's size: k_hist_dense (the
byte-pair histogram of a byte stream's first bpe_train), k_hist_hash (bpe_get_stats) and delta_fold_add in
k_merge_seg (the statistics delta of a merge pass once its delta indices no longer fit the direct shared counters).  The
fold is only right when every lane of the warp executes every match: a lane left out, a group that mixes two trips, a
wrong leader or a wrong group size changes a count.

Histogram layouts: a byte stream from load_stream, compacted segment by segment with bpe_merge(a, b, idx < 256), so it
stays a byte stream and the next bpe_train builds its table with k_hist_dense or k_hist_dense_packed.  The segments end
up holding every count 0..512 (every residue mod 128, every trip count 0..4 of a warp's 128-token steps), in more
segments than k_hist_dense's grid has warps, with chunk marks on some segment edges and few distinct byte pairs, so the
same pair sits in many lanes of one trip and again in the segment a warp takes next.  Every case is compared exactly
with a recount of the stream (oracle), and checks a counter that shows which kernel ran."""
import os
import random
import re

import numpy as np
import pytest

import oracle
from batch_model import ROOT, merge as model_merge, partition, stats, table_dict

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller streams


def _define(fname, name):
    with open(os.path.join(ROOT, "minbpe_b200", "csrc", fname)) as f:
        return int(re.search(rf"#define {name} (\d+)", f.read()).group(1))


SEG = _define("common.cuh", "SEG_TOKENS")
MS_DELTA_WORDS = _define("k_merge_seg.cuh", "MS_DELTA_WORDS")
HD_WARPS_PER_SM = 3 * 8         # k_hist_dense: sms * 3 blocks of 256 threads (b200bpe.cu hist_dense)


def _sms():
    """The SM count the library sizes its grids with."""
    if "emu" in os.path.basename(os.environ.get("BPE_LIB_PATH", "")):   # the CPU SIMT emulator's build
        return int(os.environ.get("EMU_SMS", "2"))
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- compacted byte-stream layouts -----------------------------------------------------------------------------------
# A layout is a stream of pieces, each of which the shaping merges reduce to one token at the piece's first position:
#   length 1:        a noise byte or S alone;
#   length k, 2..31: S L^(k-1)                         -> R[k-1]  by (S, L) -> R[1], (R[1], L) -> R[2], ...
#   length 32q:      Z, S L^30, then q-1 times S L^31  -> Z R[30] F^(q-1) -> G[q-1]  by (Z, R[30]) -> G[0], (G[k-1], F) -> G[k]
# A segment's count after shaping is the number of piece starts in it; a piece longer than what is left of its segment
# runs into the next one, and one of 513..1024 tokens empties the next segment.  All ids are bytes.
S, L = 1, 2
R = [S] + list(range(3, 34))                # R[k], k = 0..31; F = R[31]
F = R[31]
Z = 40
G = list(range(41, 73))                     # G[k], k = 0..31
NOISE = (200, 201, 202)
SHORT_MAX = 31
ALLOWED = sorted(set(range(1, SHORT_MAX + 1)) | {32 * q for q in range(1, 33)})
ALLOWED_SET = set(ALLOWED)
SHAPING = ([(R[k - 1], L, R[k]) for k in range(1, 32)] + [(Z, R[30], G[0])] +
           [(G[k - 1], F, G[k]) for k in range(1, 32)])


def _piece(p, rng):
    if p == 1:
        return [rng.choice(NOISE + (S,))]
    if p <= SHORT_MAX:
        return [S] + [L] * (p - 1)
    assert p % 32 == 0
    return [Z, S] + [L] * 30 + ([S] + [L] * 31) * (p // 32 - 1)


def _feasible(t, c):
    if c == 0:
        return t == 0
    if c == 1:
        return t in ALLOWED_SET
    return c <= t <= 1024 * (c - 1) + SHORT_MAX


def _split(t, c, rng):
    """c piece lengths from ALLOWED that add up to t"""
    out = []
    while c > 1:
        top = t - (c - 1)                          # the other pieces take at least one token each
        for _ in range(20):
            if top >= 32 and rng.random() < 0.15:
                x = 32 * rng.randint(1, min(32, top // 32))
            else:
                x = rng.randint(1, min(SHORT_MAX, top))
            if _feasible(t - x, c - 1):
                break
        else:
            x = next(x for x in ALLOWED if _feasible(t - x, c - 1))
        out.append(x)
        t, c = t - x, c - 1
    assert c == 1 and t in ALLOWED_SET, (t, c)
    out.append(t)
    return out


def _segment_plan(rng, nseg):
    """Per-segment target counts: each of 0..512 at least once, then random ones, one in 16 of them 0.  A 0 follows a
    segment whose last piece can run through it (target 1..400)."""
    zeros = max(1, nseg // 16)
    want = list(range(1, SEG + 1)) + [rng.randint(1, SEG) for _ in range(max(0, nseg - zeros - SEG))]
    rng.shuffle(want)
    hosts = set(rng.sample([i for i, c in enumerate(want) if c <= 400], zeros))
    plan = []
    for i, c in enumerate(want):
        plan.append(c)
        if i in hosts:
            plan.append(0)
    return plan


def compacted_layout(seed, nseg):
    """-> (bytes uint8, chunk offsets uint64, per-segment target counts).  Segments are full (SEG tokens) at load; a
    partial last segment follows them."""
    rng = random.Random(seed)
    plan = _segment_plan(rng, nseg)
    pieces = []        # (length, marked)
    i = 0
    while i < len(plan):
        c = plan[i]
        edge_mark = rng.random() < 0.5
        if i + 1 < len(plan) and plan[i + 1] == 0:        # this segment's last piece empties the next one
            qs = [q for q in range(17, 33) if (32 * q == 2 * SEG) == (c == 1) and _feasible(2 * SEG - 32 * q, c - 1)]
            last = 32 * rng.choice(qs)
            lens = (_split(2 * SEG - last, c - 1, rng) if c > 1 else []) + [last]
            i += 2
        else:
            lens = _split(SEG, c, rng)
            i += 1
        for j, p in enumerate(lens):
            pieces.append((p, edge_mark if j == 0 else rng.random() < 0.3))
    t = rng.randint(1, SHORT_MAX)
    pieces += [(1, rng.random() < 0.5) for _ in range(t)] + [(SHORT_MAX, False)]   # partial last segment
    ids, offs, pos = [], [0], 0
    for p, marked in pieces:
        if marked and pos:
            offs.append(pos)
        ids += _piece(p, rng)
        pos += p
    data = np.asarray(ids, dtype=np.uint8)
    assert len(data) == len(plan) * SEG + t + SHORT_MAX
    return data, np.unique(np.asarray(offs, dtype=np.uint64)), plan


def shape_on_model(data, offs):
    """The shaping merges on the host: -> (ids, chunk starts, per-segment token counts)."""
    ids = data.astype(np.int32)
    start = np.zeros(len(ids), dtype=bool)
    start[offs.astype(np.int64)] = True
    pos = np.arange(len(ids), dtype=np.int64)
    for a, b, z in SHAPING:
        ids, start, pos = model_merge(ids, start, (a, b), z, pos)
    nseg = (len(data) + SEG - 1) // SEG
    return ids, start, np.bincount(pos // SEG, minlength=nseg)


def _layout(seed):
    nseg = SEG + 60 if SMALL else max(SEG + 60, 2 * _sms() * HD_WARPS_PER_SM + 37)
    data, offs, plan = compacted_layout(seed, nseg)
    ids, start, counts = shape_on_model(data, offs)
    assert counts[: len(plan)].tolist() == plan
    assert set(range(SEG + 1)) <= set(counts.tolist())
    assert len(counts) > _sms() * HD_WARPS_PER_SM            # more segments than k_hist_dense's grid has warps
    marks_on_edges = int(np.count_nonzero(offs % SEG == 0))
    assert marks_on_edges > 10 and marks_on_edges < len(counts) - 10
    return data, offs, ids, start


def _shape_on_device(eng, data, offs, ids, shift=0):
    if shift:
        eng.load_ids(data.astype(np.int32) + shift, offs)
    else:
        eng.load_stream(data, offs)
    for a, b, z in SHAPING:
        eng.merge(a + shift, b + shift, z + shift)
    assert np.array_equal(eng.read_stream(), ids + shift)


def _engine(hist_kernel=None):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    if hist_kernel is not None:
        eng.set_option(E.OPT_HIST_KERNEL, hist_kernel)
    return eng


def _get_stats_exact(eng, ids, start):
    wp, wc = stats(ids, start)
    p, c = eng.get_stats()
    assert np.array_equal(p, wp) and np.array_equal(c, wc)            # first-occurrence order and counts
    # the device table was read back: next_pow2(max(1024, 2n)) slots of 24 bytes (bpe_get_stats)
    assert eng.timing()["d2h_bytes"] == (1 << max(10, (2 * len(ids) - 1).bit_length())) * 24


SEEDS = [11] if SMALL else [11, 12]


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("kernel", [2, 1])
def test_dense_histogram_on_compacted_segments(kernel, seed):
    """k_hist_dense (2) and k_hist_dense_packed (1) build the first table of a compacted byte stream: after train(1) the
    whole pair table equals the recount bin by bin.  bpe_get_stats (k_hist_hash) on the same stream first."""
    data, offs, ids, start = _layout(seed)
    eng = _engine(kernel)
    _shape_on_device(eng, data, offs, ids)
    _get_stats_exact(eng, ids, start)
    p, c, d = eng.train(1)
    assert eng.timing()["hist_kernel"] == kernel
    f_offs = np.flatnonzero(start).astype(np.uint64)
    wp, wc, wd, fin = oracle.c_train(ids, f_offs, 1, want_final=True)
    assert d == wd == 1 and np.array_equal(p, wp) and np.array_equal(c, wc)
    f_ids, f_start, _ = model_merge(ids, start, tuple(int(x) for x in wp[0]), 256)
    assert np.array_equal(f_ids, fin)
    assert eng.debug_table() == table_dict(*stats(f_ids, f_start))
    eng.close()


def test_get_stats_on_compacted_segments_of_wide_ids():
    """k_hist_hash on the same layout with every id moved up by 1000 (bpe_load_ids): pairs in first-occurrence order
    and their counts."""
    data, offs, ids, start = _layout(13)
    eng = _engine()
    _shape_on_device(eng, data, offs, ids, shift=1000)
    _get_stats_exact(eng, ids + 1000, start)
    eng.close()


# ---- delta_fold_add, hashed regime -----------------------------------------------------------------------------------
def delta_stream(groups, batched, n):
    """Units `x a b` (x one of `groups` ids, in random order), then `a b` alone as chunks so that (a, b) is the strict
    arg-max.  batched: the same with `y c d` and `c d`, counted so that (a, b) > (c, d) > every other pair, which makes
    the first pass carry both.  Every merge start of (a, b) in the first region has left neighbour x and right neighbour
    the next unit's x: with groups = 1 all 32 lanes of a warp's round fold one delta index, with groups = g they form
    up to g groups."""
    rng = np.random.default_rng(groups * 10 + batched)
    a, b, c, d = 10, 11, 12, 13

    def region(p, q, first_x, count, extra):
        xs = first_x + rng.integers(0, groups, count)
        unit = np.stack([xs, np.full(count, p), np.full(count, q)], axis=1).reshape(-1)
        alone = np.tile([p, q], extra)
        return unit, alone

    parts, marks, pos = [], [0], 0
    for p, q, fx, cnt, ex in [(a, b, 20, n, n // 5)] + ([(c, d, 40, n - n // 50, n // 10)] if batched else []):
        unit, alone = region(p, q, fx, cnt, ex)
        parts += [unit, alone]
        marks += [pos + len(unit) + 2 * k for k in range(ex)]
        pos += len(unit) + len(alone)
        marks.append(pos)
    data = np.concatenate(parts).astype(np.uint8)
    return data, np.unique(np.asarray([m for m in marks if m < len(data)], dtype=np.uint64))


@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("groups", [1, 2, 5, 16])
def test_hashed_delta_fold(groups, batched):
    """The statistics delta of merge passes whose NK·(2V+1) delta indices exceed MS_DELTA_WORDS (BPE_OPT_VOCAB_CAP
    raised), so delta_fold_add folds every round of 32 merge starts with __match_any_sync: merges, counts, the passes the
    host model predicts, the stream and the whole pair table."""
    from minbpe_b200 import engine as E
    n = 6000 if SMALL else 400000
    data, offs = delta_stream(groups, batched, n)
    ids = data.astype(np.int32)
    merges, cap = 4, 4000
    m = partition(ids, offs, merges)
    assert m.sizes[0] == (2 if batched else 1), m.sizes
    V = max(256 + merges, cap)
    assert all(nk * (2 * V + 1) > MS_DELTA_WORDS for nk in m.sizes)          # hashed cache, not direct counters
    wp, wc, _, fin = oracle.c_train(ids, offs, merges, want_final=True)
    eng = E.Engine(0)
    eng.set_option(E.OPT_VOCAB_CAP, cap)
    eng.load_stream(data, offs)
    p, c, d = eng.train(merges)
    assert d == merges and np.array_equal(p, wp) and np.array_equal(c, wc)
    assert eng.timing()["tokens_in"] == m.tokens_in, m.sizes                 # the passes ran as predicted
    assert np.array_equal(eng.read_stream(), fin)
    st = np.zeros(len(fin), dtype=bool)
    st[m.final_offs.astype(np.int64)] = True
    assert eng.debug_table() == table_dict(*stats(fin, st))
    eng.close()
