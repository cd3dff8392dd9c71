"""TEST INFRASTRUCTURE.  A host model of bpe_train with the segment filter (BPE_OPT_SEG_FILTER; k_seg_filter.cuh): the
oracle stepped the way the device steps, with the segment every token lives in.

Layout.  A load puts the stream into 512-token segments, all full except the last.  A merge of a pair (a,b), a != b,
compacts every segment in place: a pair that spans two segments leaves the merged token in the left one and the right one
loses its first token, so segments become short or empty (segment 0 never does: nothing merges into it from the left).
A pair (a,a) packs the stream first (k_merge<true> works on a contiguous stream), and so does maybe_repack at the start of
every host batch of OPT_BATCH iterations when there are at least 64 segments and the stream fills less than half of them.

Schedule.  Mode 2 filters from the first merge, mode 1 from the host batch after the first one whose merges dropped, per
merge, fewer than nseg / 32 tokens.  While the filter is on no pass is batched; a pair (a,a) is never filtered.  A table
overflow ends the host batch after the pass that raised it.

Candidate rule (restated from the kernel's three branches, not copied): before a merge (a,b), a segment with tokens is
listed when
    interior     one of its inside pairs (x, y), y not a chunk start, has sig_bit(x, y) == sig_bit(a, b);
    right edge   its last id is a and the first token of the next non-empty segment is an unmarked b;
    left edge    its first token is an unmarked b and the last id of the previous non-empty segment is a.
A filtered merge adds the list length to bpe_timing.filter_candidates and nseg to filter_segments."""
import os
import re
from collections import Counter

import numpy as np

from batch_model import BATCH_MAX, SEG_TOKENS, TABLE_MAX_LOAD, merge, predict, stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M32 = 0xffffffff


def sig_log2():
    """SIG_LOG2 of the library's sources (log2 of the signature bits per segment)."""
    with open(os.path.join(ROOT, "minbpe_b200", "csrc", "k_seg_filter.cuh")) as f:
        return int(re.search(r"#define SIG_LOG2 (\d+)", f.read()).group(1))


SIG_LOG2 = sig_log2()


def sig_bit(x, y):
    """Signature bit of the pair (x, y) in 32-bit arithmetic; x, y scalars or integer arrays."""
    x = np.asarray(x, dtype=np.uint64)
    y = np.asarray(y, dtype=np.uint64)
    h = ((x * np.uint64(0x9e3779b1)) & np.uint64(M32)) ^ ((y * np.uint64(0x85ebca77)) & np.uint64(M32))
    h ^= h >> np.uint64(15)
    h = (h * np.uint64(0x2c1b3c6d)) & np.uint64(M32)
    h ^= h >> np.uint64(12)
    return h >> np.uint64(32 - SIG_LOG2)


def batch_fits(V):
    return V <= (1 << 21)


def auto_table_log2(n, bytes_only):
    """log2 of auto_table_cap: 2^17, or for a stream of ids the smallest power of two >= 2n + 2."""
    c = 17
    while not bytes_only and (1 << c) < 2 * n + 2:
        c += 1
    return c


class State:
    """The device state that outlives a bpe_train call: the stream, its segments, the pair table's size and occupancy."""

    def __init__(self, ids, offs, bytes_only=False):
        self.ids = np.ascontiguousarray(ids, dtype=np.int32)
        self.start = np.zeros(len(self.ids), dtype=bool)
        if len(self.ids):
            self.start[np.asarray(offs if offs is not None and len(offs) else [0], dtype=np.int64)] = True
        self.bytes_only = bytes_only
        self.max_id = 255 if bytes_only else int(self.ids.max(initial=0))
        self.pack()
        self.table_log2 = None          # no table yet: bpe_train builds one
        self.used = (0, 0)              # occupied slots, [lo, hi] (exact until a table growth)

    def pack(self):
        self.seg = np.arange(len(self.ids), dtype=np.int64) // SEG_TOKENS
        self.nseg = (len(self.ids) + SEG_TOKENS - 1) // SEG_TOKENS

    def counts(self):
        return np.bincount(self.seg, minlength=self.nseg)

    @property
    def offs(self):
        return np.flatnonzero(self.start).astype(np.uint64)


class Result:
    def __init__(self):
        self.merges, self.counts = [], []
        self.candidates = 0             # filter_candidates
        self.segments = 0               # filter_segments
        self.candidates_without_overflowed = 0     # the same sums leaving out merges whose table update overflowed
        self.segments_without_overflowed = 0
        self.tokens_in = 0
        self.facts = Counter()
        self.lists = []                 # per filtered merge: (merge index, pair, listed segments)


def candidates(st, a, b, res=None):
    """The segments k_seg_filter lists before the merge (a,b) of the stream in `st`."""
    ids, start, seg = st.ids, st.start, st.seg
    n = len(ids)
    listed = np.zeros(st.nseg, dtype=bool)
    if n == 0:
        return listed
    bab = int(sig_bit(a, b))
    inside = (seg[:-1] == seg[1:]) & ~start[1:]
    p = np.flatnonzero(inside)
    hit_sig = p[sig_bit(ids[p], ids[p + 1]) == np.uint64(bab)]
    listed[seg[hit_sig]] = True
    last = np.flatnonzero(np.append(seg[:-1] != seg[1:], True))           # last token of every non-empty segment
    first = np.flatnonzero(np.insert(seg[1:] != seg[:-1], 0, True))       # first token of every non-empty segment
    r = last[(last + 1 < n)]
    r = r[(ids[r] == a) & (ids[np.minimum(r + 1, n - 1)] == b) & ~start[np.minimum(r + 1, n - 1)]]
    listed[seg[r]] = True
    q = first[first > 0]
    q = q[(ids[q] == b) & ~start[q] & (ids[q - 1] == a)]
    listed[seg[q]] = True
    if res is not None:
        _facts(st, a, b, listed, hit_sig, r, q, res.facts)
    return listed


def _facts(st, a, b, listed, hit_sig, r, q, facts):
    """What the merge (a,b) meets, for corpora built to produce it; and the model's own guarantee: every segment the merge
    changes is listed."""
    ids, start, seg = st.ids, st.start, st.seg
    cnt = st.counts()
    occ = np.flatnonzero((ids[:-1] == a) & (ids[1:] == b) & ~start[1:])
    across = occ[seg[occ] != seg[occ + 1]]
    assert listed[seg[occ]].all() and listed[seg[across + 1]].all(), "a segment the merge changes is not listed"
    facts["filtered_merges"] += 1
    if len(occ) and len(across) == len(occ):
        facts["pair_only_across_edges"] += 1
    facts["occurrence_across_edge"] += len(across)
    gap = seg[across + 1] - seg[across]
    facts["occurrence_across_empty_segment"] += int(np.count_nonzero(gap > 1))
    facts["occurrence_across_two_empty_segments"] += int(np.count_nonzero(gap > 2))
    for k in (1, 2):
        facts[f"listed_segment_of_{k}"] += int(np.count_nonzero(listed & (cnt == k)))
    facts["empty_segments"] += int(np.count_nonzero(cnt == 0))
    if cnt[-1] == 0:
        facts["empty_last_segment"] += 1
    assert cnt[0] > 0
    # a at the end of a segment followed by a chunk-marked b: no pair, and neither edge branch lists it
    last = np.flatnonzero(np.append(seg[:-1] != seg[1:], True))
    lm = last[last + 1 < len(ids)]
    facts["marked_b_after_edge"] += int(np.count_nonzero((ids[lm] == a) & (ids[lm + 1] == b) & start[lm + 1]))
    # listed by the signature bit alone: no (a,b) inside, no edge branch
    by_edge = np.zeros(st.nseg, dtype=bool)
    by_edge[seg[r]] = True
    by_edge[seg[q]] = True
    holds = np.zeros(st.nseg, dtype=bool)
    holds[seg[occ[seg[occ] == seg[occ + 1]]]] = True
    sig_only = np.zeros(st.nseg, dtype=bool)
    sig_only[seg[hit_sig]] = True
    facts["listed_by_colliding_bit"] += int(np.count_nonzero(sig_only & ~holds & ~by_edge))


def _new_pairs(ids, start, z):
    nxt = np.empty(len(ids), dtype=bool)
    nxt[:-1] = ~start[1:]
    nxt[-1:] = False
    hz = np.flatnonzero(nxt & ((ids == z) | (np.roll(ids, -1) == z)))
    return len(set(zip(ids[hz].tolist(), ids[hz + 1].tolist())))


def _maybe_repack(st, res, filt):
    if st.nseg >= 64 and 2 * len(st.ids) < st.nseg * SEG_TOKENS:
        st.pack()
        res.facts["repack"] += 1
        if filt:
            res.facts["repack_while_filtering"] += 1


def train(st, num_merges, first_idx=256, mode=2, opt_batch=256, table_log2=0, vocab_cap=0):
    """One bpe_train(num_merges, first_idx) call on the state `st` (changed in place) with BPE_OPT_SEG_FILTER = mode,
    BPE_OPT_BATCH = opt_batch, BPE_OPT_TABLE_LOG2 = table_log2.  -> Result."""
    res = Result()
    V = max(first_idx + num_merges, st.max_id + 1, vocab_cap)
    batching = batch_fits(V)
    if st.table_log2 is None:                       # a fresh table, exactly the stream's pairs
        st.table_log2 = table_log2 or auto_table_log2(len(st.ids), st.bytes_only)
        k = len(stats(st.ids, st.start)[1])
        st.used = (k, k)
    filt = mode == 2
    done = 0
    exhausted = False
    while done < num_merges and not exhausted:
        k = min(opt_batch, num_merges - done)
        _maybe_repack(st, res, filt)
        n_batch, merges_batch = len(st.ids), 0
        for _ in range(k):
            if done + merges_batch >= num_merges:
                break
            pairs, counts = stats(st.ids, st.start)
            if len(counts) == 0:
                exhausted = True
                break
            members = predict(pairs, counts, min(BATCH_MAX, num_merges - done - merges_batch)) if batching and not filt else []
            if not members:
                t = int(np.argmax(counts))
                members = [(tuple(int(x) for x in pairs[t]), int(counts[t]))]
            res.tokens_in += len(st.ids)
            (a, b) = members[0][0]
            listed = None
            if filt and a != b:
                listed = candidates(st, a, b, res)
            if a == b:
                st.pack()
                if filt:
                    res.facts["aa_merge_while_filtering"] += 1
            before = len(counts)
            new = 0
            for j, (pair, _) in enumerate(members):
                z = first_idx + done + merges_batch + j
                st.ids, st.start, st.seg = merge(st.ids, st.start, pair, z, st.seg)
                new += _new_pairs(st.ids, st.start, z)
            if a == b:
                st.pack()
            for pair, c in members:
                res.merges.append(pair)
                res.counts.append(c)
            merges_batch += len(members)
            lo, hi = st.used[0] + new, st.used[1] + new
            limit = int(TABLE_MAX_LOAD * (1 << st.table_log2))
            assert hi <= limit or lo > limit, "table overflow undecidable from the model's bounds"
            ovf = lo > limit
            if listed is not None:
                c = int(np.count_nonzero(listed))
                res.lists.append((len(res.merges) - 1, (a, b), np.flatnonzero(listed)))
                res.candidates += c
                res.segments += st.nseg
                if not ovf:
                    res.candidates_without_overflowed += c
                    res.segments_without_overflowed += st.nseg
            if ovf:
                # handle_overflow: the table doubles (dead pairs dropped) and the pending entries go in
                res.facts["overflow"] += 1
                if listed is not None:
                    res.facts["overflow_while_filtering"] += 1
                st.table_log2 += 1
                after = len(stats(st.ids, st.start)[1])
                st.used = (after, before + new)
                assert st.used[1] <= int(TABLE_MAX_LOAD * (1 << st.table_log2)), "more than one doubling"
                break
            st.used = (lo, hi)
        done += merges_batch
        if mode == 1 and not filt and merges_batch:
            per_merge = (n_batch - len(st.ids)) // merges_batch
            if per_merge * 32 < st.nseg:
                filt = True
                res.facts["switch_on"] += 1
                res.switch_at = done
    if done:
        st.max_id = max(st.max_id, first_idx + done - 1)
    res.merges = np.asarray(res.merges, dtype=np.int32).reshape(-1, 2)
    res.counts = np.asarray(res.counts, dtype=np.int64)
    res.n_done = done
    return res


def replay(st, merges, opt_batch=256):
    """bpe_replay(merges) on a freshly loaded byte stream: one merge per round, a re-pack check every opt_batch rounds, a
    fresh table of 2^17 slots (no overflow in the streams the tests use)."""
    merges = np.asarray(merges, dtype=np.int32).reshape(-1, 2)
    res = Result()
    used = len(stats(st.ids, st.start)[1])
    for i0 in range(0, len(merges), opt_batch):
        _maybe_repack(st, res, False)
        for i in range(i0, min(i0 + opt_batch, len(merges))):
            a, b = (int(x) for x in merges[i])
            if a == b:
                st.pack()
            st.ids, st.start, st.seg = merge(st.ids, st.start, (a, b), 256 + i, st.seg)
            used += _new_pairs(st.ids, st.start, 256 + i)
            if a == b:
                st.pack()
    st.table_log2 = 17
    assert used <= int(TABLE_MAX_LOAD * (1 << 17))
    st.used = (used, used)
    st.max_id = max(st.max_id, 255 + len(merges))
    st.bytes_only = False
    return res


# ---- corpora --------------------------------------------------------------------------------------------------------
class Stream:
    def __init__(self, filler0):
        self.ids, self.marks = [], []
        self.f = filler0

    def put(self, x, mark=False):
        self.ids.append(int(x))
        self.marks.append(bool(mark))

    def filler(self, k):
        for _ in range(k):
            self.put(self.f)
            self.f += 1

    def fill_to(self, off):
        """filler until the next token lands at offset `off` of a segment"""
        while len(self.ids) % SEG_TOKENS != off % SEG_TOKENS:
            self.filler(1)

    def stream(self):
        ids = np.asarray(self.ids, dtype=np.int32)
        marks = np.asarray(self.marks, dtype=bool)
        marks[0] = True
        return ids, np.flatnonzero(marks).astype(np.uint64)


def chains(base=1000, pad_segments=0, run=True):
    """Chains that drain whole segments across their left edge.  A chain of length L is L + 1 distinct ids c0 .. cL with
    c0 at the last offset of a segment and c1 .. cL filling the next L / 512 segments; three copies give every pair
    (z, c_k+1) of the chain count 3, and the tie-break by first occurrence merges the chain left to right: every one of
    its L merges spans a segment edge, the segments it drains pass through 2, 1 and 0 tokens, and the merged token ends
    at the last offset of the first segment.  Chain C (L = 512) drains one segment, chain D (L = 1024) two; after each, a
    pair (Z, B) of count 2 spans the drained segments, and a third copy is followed by a chunk-marked B (no pair).  The
    last copy of D ends the stream (an empty last segment).  `run`: a chunk "r r r" after them, a pair (r,r) of count 2
    that merges (pack) after the chains.  `pad_segments`: segments of filler before the last copy of D (mode 1 needs
    nseg > 32 * 3 to switch on).  Filler ids start at base + 2000 and each occurs once.
    -> (ids, offs)."""
    C = list(range(base, base + 513))
    D = list(range(base + 600, base + 600 + 1025))
    B1, B2, R = base + 1700, base + 1701, base + 1702
    s = Stream(base + 2000)
    s.filler(5)

    def chain(ch, follow, mark):
        s.fill_to(SEG_TOKENS - 1)
        for x in ch:
            s.put(x)
        if follow is not None:
            s.put(follow, mark)
            s.filler(3)

    chain(C, B1, False)
    chain(D, B2, False)
    chain(C, B1, False)
    chain(D, B2, False)
    if run:
        s.put(R, True)
        s.put(R)
        s.put(R)
        s.put(R + 1, True)
    chain(C, B1, True)
    s.filler(SEG_TOKENS * pad_segments)
    chain(D, None, False)
    return s.stream()
