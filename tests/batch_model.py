"""TEST INFRASTRUCTURE.  A host model of bpe_train's pass partition: the oracle stepped the way the device steps.

At the start of every pass the device holds the pair table of the current stream; k_select_batch takes the arg-max and
as many following pairs as the rule of `predict` proves (DESIGN.md "Batched merges"), at most
min(BATCH_MAX, merges left in the bpe_train call).  A tie or a pair (a,a) gives a pass of one merge.  The merge pass
adds the stream length it read to ctl->sum_in once, so Engine.timing()["tokens_in"] of a bpe_train call is exactly
the sum over its passes of the stream length before the pass: the model predicts it, and with it whether (and how)
the device batched.

The model also reports facts about the layout the passes met (adjacent members, members next to a segment edge or a
chunk mark), so that a corpus built to produce them can be checked to still do so, and the pair-table occupancy
k_apply_delta reserves (one slot per distinct new pair of every member), from which the first table overflow
follows."""
import os
import re
from collections import Counter

import numpy as np

import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEG_TOKENS = 512
TABLE_MAX_LOAD = 0.6


def batch_max():
    """BATCH_MAX of the library's sources (the most merges one pass carries)."""
    with open(os.path.join(ROOT, "minbpe_b200", "csrc", "common.cuh")) as f:
        return int(re.search(r"#define BATCH_MAX (\d+)", f.read()).group(1))


BATCH_MAX = batch_max()


def predict(pairs, counts, cap):
    """The batch the rule allows at this step: [(pair, count)], empty when the arg-max is tied or a pair (a,a).
    With the pairs sorted by count, p1 .. pk are the next k merges when c1 > c2 > ... > ck > c(k+1), every pj has two
    different ids and the 2k ids are all distinct."""
    if len(counts) == 0:
        return []
    order = np.argsort(-counts, kind="stable")
    c = counts[order].tolist() + [0] * (cap + 1)
    p = [tuple(x) for x in pairs[order].tolist()]
    if c[0] == c[1] or p[0][0] == p[0][1]:
        return []
    ids = {p[0][0], p[0][1]}
    k = 1
    while k < cap and c[k] > c[k + 1]:
        x, y = p[k]
        if x == y or x in ids or y in ids:
            break
        ids |= {x, y}
        k += 1
    return [(p[j], c[j]) for j in range(k)]


def merge(ids, start, pair, z, pos=None):
    """base.py:25-41 over a stream whose chunk starts are marked in `start` (no pair spans two chunks).  `pos`, if
    given, is carried along: a merged token keeps the entry of its left half."""
    a, b = pair
    hit = (ids[:-1] == a) & (ids[1:] == b) & ~start[1:]
    at = np.flatnonzero(hit)
    if a == b:   # runs: greedy from the left
        keep, last = [], -2
        for q in at.tolist():
            if q != last + 1:
                keep.append(q)
                last = q
        at = np.asarray(keep, dtype=np.int64)
    ids = ids.copy()
    ids[at] = z
    drop = np.ones(len(ids), dtype=bool)
    drop[at + 1] = False
    return ids[drop], start[drop], (None if pos is None else pos[drop])


def stats(ids, start, weights=None):
    """get_stats() of the stream in first-occurrence order -> (pairs[k,2], counts[k] int64): oracle.c_get_stats, or for a
    weighted stream the sum of the entry weights over every occurrence (entry = chunk = run from one mark to the next)."""
    if weights is None:
        return oracle.c_get_stats(ids, np.flatnonzero(start).astype(np.uint64))
    if len(ids) < 2:
        return np.zeros((0, 2), dtype=np.int32), np.zeros(0, dtype=np.int64)
    ent = np.cumsum(start) - 1
    ok = ~start[1:]
    key = (ids[:-1][ok].astype(np.int64) << 32) | ids[1:][ok].astype(np.int64)
    w = np.asarray(weights, dtype=np.int64)[ent[:-1][ok]]
    uniq, first, inv = np.unique(key, return_index=True, return_inverse=True)
    cnt = np.zeros(len(uniq), dtype=np.int64)
    np.add.at(cnt, inv, w)
    order = np.argsort(first, kind="stable")
    uniq, cnt = uniq[order], cnt[order]
    return np.stack([(uniq >> 32).astype(np.int32), (uniq & 0xffffffff).astype(np.int32)], axis=1), cnt


def table_dict(pairs, counts):
    return {(int(a), int(b)): int(c) for (a, b), c in zip(pairs.tolist(), counts.tolist())}


class Pass:
    def __init__(self, members, n_before):
        self.members = members          # [((a, b), count)] in member order
        self.n_before = n_before        # stream length the pass reads
        self.new_pairs = []             # per member: distinct pairs holding its new id once it is applied


class Model:
    """Result of `partition`: passes, merges, counts, final stream, layout facts, table reservations."""

    def __init__(self):
        self.passes = []
        self.merges = []
        self.counts = []
        self.facts = Counter()
        self.init_pairs = 0

    @property
    def tokens_in(self):
        return sum(p.n_before for p in self.passes)

    @property
    def sizes(self):
        return [len(p.members) for p in self.passes]

    def tokens_in_upto(self, k):
        """tokens_in of a bpe_train(k) call on the same stream: the passes that start before merge k (a smaller cap only
        cuts the last of them short)."""
        out, i = 0, 0
        for p in self.passes:
            if i >= k:
                break
            out += p.n_before
            i += len(p.members)
        return out

    def first_overflow(self, log2, used=None):
        """(pass index, member index) of the first k_apply_delta that runs out of reserved slots in a table of 2^log2
        slots (load limit floor(0.6 * 2^log2)), or None; `used` = occupied slots when the call starts."""
        limit = int(TABLE_MAX_LOAD * (1 << log2))
        u = self.init_pairs if used is None else used
        for i, p in enumerate(self.passes):
            for j, new in enumerate(p.new_pairs):
                u += new
                if u > limit:
                    return i, j
        return None

    def used_after(self, n_passes, used=None):
        """Slots k_apply_delta has reserved after the first n_passes passes (no overflow in between)."""
        u = self.init_pairs if used is None else used
        return u + sum(sum(p.new_pairs) for p in self.passes[:n_passes])


def _layout_facts(model, ids, start, pos, members, seg_known):
    """Facts of one pass with several members, on the stream it reads."""
    n = len(ids)
    mark = np.full(n, -1, dtype=np.int64)
    for j, ((a, b), _) in enumerate(members):
        hit = np.flatnonzero((ids[:-1] == a) & (ids[1:] == b) & ~start[1:])
        mark[hit] = j
    if len(members) == BATCH_MAX:
        model.facts["full_batch"] += 1
    p = np.flatnonzero((mark[:-2] >= 0) & (mark[2:] >= 0))     # member starts two tokens apart: b_j is next to a_m
    if p.size == 0:
        return
    j, m, sep = mark[p], mark[p + 2], start[p + 2]
    model.facts["adj_chunk_mark"] += int(np.count_nonzero(sep))
    same = ~sep
    model.facts["adj_fwd"] += int(np.count_nonzero(same & (j < m)))
    model.facts["adj_rev"] += int(np.count_nonzero(same & (j > m)))
    model.facts["adj_self"] += int(np.count_nonzero(same & (j == m)))
    if seg_known:
        edge = (pos[p + 1] // SEG_TOKENS) != (pos[p + 2] // SEG_TOKENS)
        model.facts["adj_seg_edge"] += int(np.count_nonzero(same & edge))
        cross = np.flatnonzero(mark >= 0)
        model.facts["member_across_seg_edge"] += int(np.count_nonzero((pos[cross] // SEG_TOKENS) != (pos[cross + 1] // SEG_TOKENS)))


def partition(ids, offs, num_merges, first_idx=256, weights=None, cap=None):
    """Step the oracle through one bpe_train(num_merges, first_idx) call on the stream (ids, chunk offsets) the way the
    device does.  cap: most members per pass (BATCH_MAX; 1 = one merge per pass)."""
    cap = BATCH_MAX if cap is None else cap
    ids = np.ascontiguousarray(ids, dtype=np.int32)
    start = np.zeros(len(ids), dtype=bool)
    if len(ids):
        start[np.asarray(offs if offs is not None and len(offs) else [0], dtype=np.int64)] = True
    pos = np.arange(len(ids), dtype=np.int64)   # load position: segment = pos // 512 until the stream is first packed
    nseg0 = (len(ids) + SEG_TOKENS - 1) // SEG_TOKENS
    seg_known = True
    model = Model()
    i = 0
    while i < num_merges:
        pairs, counts = stats(ids, start, weights)
        if i == 0:
            model.init_pairs = len(counts)
        if len(counts) == 0:
            break
        members = predict(pairs, counts, min(cap, num_merges - i))
        if not members:
            t = int(np.argmax(counts))             # the first pair at the max: first occurrence (dict insertion order)
            members = [(tuple(int(x) for x in pairs[t]), int(counts[t]))]
        # a re-pack between host batches (maybe_repack) or the pack of a pair (a,a) refills the segments
        if nseg0 >= 64 and 2 * len(ids) < nseg0 * SEG_TOKENS:
            model.facts["repack_possible"] += 1
            seg_known = False
        if len(members) > 1:
            _layout_facts(model, ids, start, pos, members, seg_known)
        ps = Pass(members, len(ids))
        for j, (pair, count) in enumerate(members):
            z = first_idx + i + j
            ids, start, pos = merge(ids, start, pair, z, pos)
            nxt = np.empty(len(ids), dtype=bool)
            nxt[:-1] = ~start[1:]
            nxt[-1:] = False
            hz = np.flatnonzero(nxt & ((ids == z) | (np.roll(ids, -1) == z)))
            ps.new_pairs.append(len(set(zip(ids[hz].tolist(), ids[hz + 1].tolist()))))
            model.merges.append(pair)
            model.counts.append(count)
        if members[0][0][0] == members[0][0][1]:
            seg_known = False
        model.passes.append(ps)
        i += len(members)
    model.final = ids
    model.final_offs = np.flatnonzero(start).astype(np.uint64)
    model.merges = np.asarray(model.merges, dtype=np.int32).reshape(-1, 2)
    model.counts = np.asarray(model.counts, dtype=np.int64)
    return model


# ---- corpora --------------------------------------------------------------------------------------------------------
FILLER0 = 2000


class _Builder:
    """A stream of ids with chunk marks, filler ids (>= 2000) that each occur once; or, for a byte stream, filler
    bytes drawn from `pool`."""

    def __init__(self, rng, pool=None):
        self.ids, self.marks = [], []
        self.next_filler = FILLER0
        self.rng, self.pool = rng, pool

    def filler(self, k=1, mark=False):
        for q in range(k):
            if self.pool is None:
                self.put(self.next_filler, mark and q == 0)
                self.next_filler += 1
            else:
                self.put(self.pool[int(self.rng.integers(len(self.pool)))], mark and q == 0)

    def put(self, x, mark=False):
        self.ids.append(int(x))
        self.marks.append(bool(mark))

    def pad_to(self, off):
        """filler until the next token lands at offset `off` mod 512"""
        while len(self.ids) % SEG_TOKENS != off % SEG_TOKENS:
            self.filler()

    def stream(self):
        ids = np.asarray(self.ids, dtype=np.int32)
        marks = np.asarray(self.marks, dtype=bool)
        marks[0] = True
        return ids, np.flatnonzero(marks).astype(np.uint64)


def planted(seed=0, step=24, groups=2, byte_ids=False, offsets=range(509, 515)):
    """Planted layouts: pairs P1..P8 (P_i = (a_i, b_i), 16 distinct ids below 2000) with strictly decreasing counts
    `step` apart, among filler ids that each occur once.  Each group of four (P1..P4, P5..P8) is placed singly, as
    P1P2, P2P1, P1P2P3P4 and P1P1, at stream offsets 509..514 mod 512 (adjacent members on either side of a segment
    edge, members across one) and on either side of chunk marks.  The first passes then batch P1..P4 and P5..P8 with
    every adjacency in the stream; later passes batch the second-level pairs.  byte_ids: the same in bytes (the
    pairs' ids are 16 letters, the filler is drawn from 200 other byte values).  -> (ids, chunk offsets)."""
    rng = np.random.default_rng(seed)
    if byte_ids:
        a = [65 + 2 * i for i in range(4 * groups)]
        b = [66 + 2 * i for i in range(4 * groups)]
        pool = [x for x in range(256) if x not in a + b][:200]
        B = _Builder(rng, pool)
    else:
        a = [1000 + 2 * i for i in range(4 * groups)]
        b = [1001 + 2 * i for i in range(4 * groups)]
        B = _Builder(rng)
    used = Counter()

    def put_layout(order, mark_between=False):
        for q, i in enumerate(order):
            B.put(a[i], mark_between and q > 0)
            B.put(b[i])
            used[i] += 1

    for g in range(groups):
        P = [4 * g + i for i in range(4)]
        layouts = [[P[0], P[1]], [P[1], P[0]], [P[0], P[1], P[2], P[3]], [P[0], P[0]], [P[3], P[2]], [P[2], P[2]]]
        for off in offsets:                 # the layout's first token at 509 .. 514 mod 512
            for lay in layouts:
                B.pad_to(off)
                put_layout(lay)
                B.filler(1 + int(rng.integers(3)))
        # more copies anywhere: the second-level pairs get counts of their own, so that they batch as well
        copies = [10 + 3 * g, 3, 6, 2, 16 + 5 * g, 1]
        for lay in (lay for lay, c in zip(layouts, copies) for _ in range(c)):
            put_layout(lay)
            B.filler(1 + int(rng.integers(3)), mark=bool(rng.random() < 0.3))
        for _ in range(2):                  # on either side of chunk marks: a_m starts a chunk; pairs end / begin chunks
            for lay in layouts[:3]:
                B.filler(1 + int(rng.integers(3)), mark=True)
                put_layout(lay, mark_between=True)
                B.filler(1, mark=True)
    # top up singly to strictly decreasing counts, well apart; the single copies are spread over the stream
    top = max(used.values()) + 8 * groups * step
    rest = []
    for i in range(4 * groups):
        rest += [i] * (top - step * i - used[i])
    rng.shuffle(rest)
    for i in rest:
        B.filler(1 + int(rng.integers(3)), mark=bool(rng.random() < 0.2))
        put_layout([i])
    B.filler(3)
    return B.stream()


def with_filler_pairs(ids, offs, extra):
    """The stream followed by one chunk of extra + 1 new filler ids: `extra` more distinct pairs, each of count 1."""
    if extra <= 0:
        return ids, offs
    f0 = max(int(ids.max()) + 1, FILLER0)
    tail = np.arange(f0, f0 + extra + 1, dtype=np.int32)
    return np.concatenate([ids, tail]), np.concatenate([offs, np.asarray([len(ids)], dtype=np.uint64)])


def short_chunks(seed=0, n_tokens=20000, alphabet=12):
    """Many 2- and 3-token chunks over a small alphabet with skewed frequencies: merged far enough, every chunk is one
    token and most segments hold a small fraction of their 512 words.  -> (ids, chunk offsets)."""
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, alphabet + 1) ** 1.3
    p /= p.sum()
    ids, marks = [], []
    while len(ids) < n_tokens:
        k = 2 + int(rng.random() < 0.4)
        c = rng.choice(alphabet, size=k, p=p)
        ids += (c + 300).tolist()
        marks += [True] + [False] * (k - 1)
    ids = np.asarray(ids, dtype=np.int32)
    return ids, np.flatnonzero(np.asarray(marks)).astype(np.uint64)


def weighted_entries(ids, offs, seed=0, big=False):
    """Entries with weights for a load of (ids, offs) as chunks: random weights in [1, 6], and with `big` a few in the
    2^33 range, so that counts and the rule's comparisons need more than 32 bits."""
    rng = np.random.default_rng(seed)
    w = rng.integers(1, 7, size=len(offs)).astype(np.int64)
    if big:
        k = rng.choice(len(offs), size=max(1, len(offs) // 50), replace=False)
        w[k] = (1 << 33) + rng.integers(0, 1 << 20, size=len(k))
    return w
