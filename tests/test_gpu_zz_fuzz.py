"""GPU: fixed-seed differential fuzz of every training and encode path, at the shapes where the kernels cut their work.

Every round is compared exactly with the C oracle (oracle.c_train / c_encode / c_get_stats / split_to_stream /
c_dedup_chunks, pinned to the reference by tests/golden/), and proves from the engine's counters that the device path
ran.  The shapes come from the code's own constants (read from the sources below):

- merge pass (k_merge_seg): the first changed token of a segment at every offset 0..511, segments compacted by earlier
  merges to about 128 / 256 / 384 tokens or to a few, segments that become empty, merges across a segment edge and
  pairs cut by a chunk mark, adjacent occurrences of one member and of two;
- statistics delta: for 1..BATCH_MAX members, the largest delta layout V whose NK·(2V+1) counters fit MS_DELTA_WORDS
  and the next one, and a hashed cache that spills to global atomics (ids up to 2^17);
- large rounds: streams long enough that every warp of a 132-SM H100 takes tickets of MS_BATCH segments, with batched
  passes and with the segment filter;
- split and encode: byte lengths around the 2048-byte encode tile and its 64-byte halo, the 48-byte memo key, 8192-token
  long chunks, split pieces of 4096 and 1<<14 bytes, the device thresholds of the classes; small memo tables, byte
  permutations, document edges at tile and piece edges; alphabets that reach every rule of the GPT-2, GPT-4 and o200k
  patterns;
- special tokens: sets of 1..5 and 65..300 specials of 1..48 bytes, prefix chains in both dict orders, truncated and
  adjacent occurrences, random allowed subsets;
- the reference classes' own answers (tests/golden/golden_fuzz_train.json, golden_fuzz_special.json) replayed here.

A failure names the test, seed, round and options; BPE_FUZZ_ROUND=<seed>:<round> reruns that one round."""
import contextlib
import os
import re
import sys
from collections import Counter

import numpy as np
import pytest
import regex

import oracle
from batch_model import ROOT, merge as model_merge, partition, planted, stats, table_dict, weighted_entries

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller streams, fewer rounds
ONLY = os.environ.get("BPE_FUZZ_ROUND")              # "<seed>:<round>": run that one round of the test with that seed
H100_SMS = 132


def _define(fname, name):
    with open(os.path.join(ROOT, "minbpe_b200", "csrc", fname)) as f:
        return int(re.search(rf"#define {name} (\d+)", f.read()).group(1))


SEG = _define("common.cuh", "SEG_TOKENS")
BATCH_MAX = _define("common.cuh", "BATCH_MAX")
MS_DELTA_WORDS = _define("k_merge_seg.cuh", "MS_DELTA_WORDS")
MS_BATCH = _define("k_merge_seg.cuh", "MS_BATCH")
MS_WARPS = _define("k_merge_seg.cuh", "MS_WARPS")
MS_MINBLOCKS = _define("k_merge_seg.cuh", "MS_MINBLOCKS")
MS_DCACHE = 1 << _define("k_merge_seg.cuh", "MS_DCACHE_LOG2")
E2_TILE = _define("k_encode2.cuh", "E2_THREADS") * _define("k_encode2.cuh", "E2_ITEMS")
E2_HALO = _define("k_encode2.cuh", "E2_HALO")
E2_LMAX = _define("k_encode2.cuh", "E2_LMAX")
ENC_LONG_MAX = _define("k_encode.cuh", "ENC_LONG_MAX")
SP_TILE = _define("k_split.cuh", "SP_THREADS") * _define("k_split.cuh", "SP_ITEMS")
SECTOR = 8            # tokens of a 32-byte sector
ROW = 128             # tokens of a row of k_merge_seg (32 lanes x 4)
# tokens at which every warp of the merge grid holds a ticket of MS_BATCH segments
ALL_WARPS_TOKENS = H100_SMS * MS_MINBLOCKS * MS_WARPS * MS_BATCH * SEG


def vmax(nk):
    """the largest delta layout V whose NK·(2V+1) counters fit MS_DELTA_WORDS (direct counters)"""
    return (MS_DELTA_WORDS // nk - 1) // 2


def _patterns():
    from minbpe_b200 import tokenizer as T
    return {"gpt4": (0, T.GPT4_SPLIT_PATTERN), "gpt2": (1, T.GPT2_SPLIT_PATTERN), "o200k": (3, T.O200K_SPLIT_PATTERN)}


# ---- rounds ----------------------------------------------------------------------------------------------------------
class Fuzz:
    """The rounds of one test.  Round r of seed s draws from default_rng([s, r]), so any round can be rerun alone."""

    def __init__(self, name, seed, rounds, report):
        self.name, self.seed, self.rounds, self.report = name, seed, rounds, report
        self.paths = Counter()
        self.ran = 0
        self.only = None
        if ONLY:
            s, r = (int(x) for x in ONLY.split(":"))
            self.only = r if s == seed else -1

    @property
    def complete(self):
        """every round ran: coverage over the rounds can be asserted"""
        return self.only is None

    def __iter__(self):
        for r in range(self.rounds):
            if self.only is None or self.only == r:
                yield r, np.random.default_rng([self.seed, r])

    @contextlib.contextmanager
    def round(self, r, **opts):
        try:
            yield
        except Exception as ex:
            raise AssertionError(f"{self.name}: seed {self.seed} round {r} options {opts}: {type(ex).__name__}: {ex}"
                                 f"\n  rerun: BPE_FUZZ_ROUND={self.seed}:{r}") from ex
        self.ran += 1

    def path(self, name, n=1):
        self.paths[name] += n

    def done(self):
        self.report(f"{self.name}: {self.ran} rounds; device paths " + ", ".join(f"{k} {v}" for k, v in sorted(self.paths.items())))


@pytest.fixture
def fuzz(request):
    tr = request.config.pluginmanager.get_plugin("terminalreporter")
    cap = request.config.pluginmanager.get_plugin("capturemanager")
    made = []

    def report(line):
        with cap.global_and_fixture_disabled() if cap is not None else contextlib.nullcontext():
            if tr is not None:
                tr.write_line("\n" + line)
            else:
                print(line)

    def make(seed, rounds):
        f = Fuzz(request.node.name, seed, rounds, report)
        made.append(f)
        return f
    yield make
    for f in made:
        f.done()


def _engine():
    from minbpe_b200 import engine as E
    return E.Engine(0)


def _launches(eng):
    return eng.timing()["kernel_launches"]


# ---- merge pass shapes -----------------------------------------------------------------------------------------------
PLANT_A = [1000 + 2 * i for i in range(BATCH_MAX * 2)]
PLANT_B = [1001 + 2 * i for i in range(BATCH_MAX * 2)]
EDGE_W = 1040                 # last token of the segment in front of a tiny one
SHAPE = {"c384": (1100, 1101, 1102, 1103), "c256": (1110, 1111), "c128": (1120, 1121, 1122, 1123)}
TEMPLATE0 = 1200              # tiny segments: SEG distinct ids TEMPLATE0 .. TEMPLATE0 + SEG - 1, folded from the left
FILLER0 = 2000


def shaped_stream(rng, nseg, tiny_left, first_offset):
    """(ids, chunk-start marks, plan) of nseg segments with profiles full / c384 / c256 / c128 / tiny.  Full segments
    hold planted pairs at chosen offsets (runs of one member, two members back to back, a pair cut by a chunk mark, a pair
    across the edge into the next segment); the others are built to shrink under the shaping merges of `plan` to about
    384 / 256 / 128 tokens, with a planted pair at a chosen chunk, or to `tiny_left` tokens.  The stream ends with one
    token that a planted pair reaches from the segment in front: that last segment becomes empty."""
    kinds = rng.choice(["full", "full", "full", "c384", "c256", "c128", "tiny"], size=nseg - 1).tolist()
    offsets = [(first_offset + i) % SEG for i in range(nseg)][::-1]    # popped in order: consecutive offsets from first_offset
    ids, marks = [], []
    carry = None
    nxt = [FILLER0]

    def filler(k):
        out = list(range(nxt[0], nxt[0] + k))
        nxt[0] += k
        return out

    members = int(rng.integers(1, BATCH_MAX + 1))   # pairs with strictly decreasing counts: batched passes
    weights = np.linspace(1.0, 0.4, members)
    weights /= weights.sum()

    def pick():
        return int(rng.choice(members, p=weights))
    for s, kind in enumerate(kinds):
        if kind == "tiny" and (s == 0 or kinds[s - 1] != "full"):
            kind = kinds[s] = "full"
        if kind == "full":
            seg = filler(SEG)
            mk = [False] * SEG
            mk[0] = True
            for q in range(SEG):
                if rng.random() < 0.15:
                    mk[q] = True
            o = offsets.pop() if offsets else int(rng.integers(SEG))
            j = pick()
            lay = [j]
            r = rng.random()
            if r < 0.25:
                lay = [j, j, j][: int(rng.integers(2, 4))]             # a run of one member
            elif r < 0.45 and members > 1:
                lay = [j, (j + 1) % members]                          # two members back to back
            if carry is not None:                                     # token 0 is the right half of a pair from the segment before
                seg[0], mk[0] = carry, False
                o = max(o, 1)
                carry = None
            if s + 1 >= len(kinds):
                o = min(o, SEG - 2 * len(lay) - 1)
            elif o + 2 * len(lay) >= SEG:
                kinds[s + 1] = "full"                                 # the layout reaches the last token or past it
            at = o
            for jj in lay:
                if at >= SEG:
                    break
                seg[at] = PLANT_A[jj]
                if at + 1 == SEG:
                    carry = PLANT_B[jj]                               # the pair reaches across the segment edge
                    break
                seg[at + 1] = PLANT_B[jj]
                mk[at + 1] = rng.random() < 0.05                      # now and then a chunk mark cuts the pair
                at += 2
            if s + 1 < len(kinds) and kinds[s + 1] == "tiny":
                seg[SEG - 1] = EDGE_W
            ids += seg
            marks += mk
        elif kind == "tiny":
            ids += list(range(TEMPLATE0, TEMPLATE0 + SEG))
            marks += [False] * SEG                                    # one chunk with the last token in front
        else:
            p = SHAPE[kind]
            unit = [[p[0], p[1]], [p[2]], [p[3]]] if kind == "c384" else [list(p)]    # 4 -> 3, 2 -> 1, 4 -> 1 tokens
            seg, mk = [], []
            plant_at = int(rng.integers(0, SEG // 4))
            u = 0
            while len(seg) < SEG:
                if u == plant_at and len(seg) + 4 <= SEG:
                    j = pick()
                    seg += [PLANT_A[j], PLANT_B[j]] + filler(2)
                    mk += [True, False, False, False]
                elif rng.random() < 0.03:
                    k = min(int(rng.integers(1, 4)), SEG - len(seg))  # a few extra tokens: counts near, not at, the mark
                    seg += filler(k)
                    mk += [True] * k
                else:
                    for c in unit:
                        c = c[: SEG - len(seg)]
                        if not c:
                            break
                        seg += c
                        mk += [True] + [False] * (len(c) - 1)
                u += 1
            ids += seg
            marks += mk
    # the last segment: one token, the right half of a planted pair that starts at the last token of the segment before
    j = 0
    ids[-1] = PLANT_A[j]
    marks[-1] = False
    ids.append(PLANT_B[j])
    marks.append(False)
    marks[0] = True
    assert len(ids) == len(marks) == (nseg - 1) * SEG + 1
    # shaping merges: (left, right), an int id or ("z", k) = the id made by shaping merge k
    plan = [SHAPE["c384"][:2], SHAPE["c256"][:2], SHAPE["c128"][:2], SHAPE["c128"][2:], (("z", 2), ("z", 3)),
            (TEMPLATE0, TEMPLATE0 + 1)]
    plan += [(("z", len(plan) - 1 + k), TEMPLATE0 + 1 + k) for k in range(1, SEG - tiny_left)]
    return np.asarray(ids, dtype=np.int32), np.asarray(marks, dtype=bool), plan


def pass_layout(ids, start, pos, members):
    """Per segment (load position // SEG) of the stream a pass reads: its token count, and the offset inside it of the
    first token the pass replaces or drops (-1: none); also how many members reach across a segment edge."""
    seg = pos // SEG
    nseg = int(seg.max()) + 1 if len(seg) else 0
    count = np.bincount(seg, minlength=nseg)
    first_idx = np.zeros(nseg, dtype=np.int64)
    first_idx[1:] = np.cumsum(count)[:-1]
    hit = np.zeros(len(ids), dtype=bool)
    for (a, b), _ in members:
        hit[:-1] |= (ids[:-1] == a) & (ids[1:] == b) & ~start[1:]
    ch = np.flatnonzero(hit)
    ch = np.concatenate([ch, ch + 1])
    first = np.full(nseg, SEG, dtype=np.int64)
    np.minimum.at(first, seg[ch], ch - first_idx[seg[ch]])
    first[first == SEG] = -1
    across = int(np.count_nonzero(seg[np.flatnonzero(hit)] != seg[np.flatnonzero(hit) + 1]))
    return count, first, across


def test_merge_pass_shapes(fuzz):
    """load_ids + bpe_merge (shaping) + chained bpe_train calls on streams where the first changed token of a segment
    falls at every offset 0..511, in full and in compacted segments; oracle merges, counts, stream, pair table and passes."""
    F = fuzz(101, 2 if SMALL else 6)
    offs_full, offs_compact, counts_seen = set(), set(), set()
    facts = Counter()
    for r, rng in F:
        nseg = 40 if SMALL else 700
        tiny_left = int(rng.choice([1, 2, 3]))
        ids, start, plan = shaped_stream(rng, nseg, tiny_left, first_offset=r * 290)
        with F.round(r, nseg=nseg, tiny_left=tiny_left, n=len(ids)):
            eng = _engine()
            eng.load_ids(ids, np.flatnonzero(start).astype(np.uint64))
            z = z0 = int(ids.max()) + 1
            cur, st, pos = ids, start, np.arange(len(ids), dtype=np.int64)
            for a, b in plan:                                        # shaping merges, applied one by one with bpe_merge
                a, b = (z0 + x[1] if isinstance(x, tuple) else x for x in (a, b))
                n_dev = eng.merge(a, b, z)
                cur, st, pos = model_merge(cur, st, (a, b), z, pos)
                assert n_dev == len(cur), ("bpe_merge", a, b, n_dev, len(cur))
                z += 1
            assert np.array_equal(eng.read_stream(), cur), "stream after the shaping merges"
            F.path("bpe_merge", len(plan))
            # training from here: chained calls at random merge counts
            total = 12 if SMALL else 40
            cuts = sorted(set(rng.integers(1, total, size=int(rng.integers(1, 4))).tolist()))
            calls = np.diff([0] + cuts + [total]).tolist()
            offs0 = np.flatnonzero(st).astype(np.uint64)
            wp, wc, wd, fin = oracle.c_train(cur, offs0, total, first_idx=z, want_final=True)
            fi, got_p, got_c = z, [], []
            seg_known = True
            for n in calls:
                m = partition(cur, np.flatnonzero(st).astype(np.uint64), n, first_idx=fi)
                if m.facts["repack_possible"]:
                    seg_known = False
                p, c, d = eng.train(n, first_idx=fi)
                assert _launches(eng) > 0
                assert d == len(m.merges) and np.array_equal(p, m.merges) and np.array_equal(c, m.counts), ("pass model", n)
                assert eng.timing()["tokens_in"] == m.tokens_in, ("tokens_in", n, m.sizes)
                facts.update(m.facts)
                F.path(f"passes of {max(m.sizes) if m.sizes else 0} members")
                for ps in m.passes:
                    if ps.members[0][0][0] == ps.members[0][0][1]:
                        seg_known = False                     # a pair (a,a) packs the stream: segments are refilled
                    if seg_known:
                        count, first, across = pass_layout(cur, st, pos, ps.members)
                        facts["member_across_edge"] += across
                        compact = count < SEG
                        offs_full.update(first[(first >= 0) & ~compact].tolist())
                        offs_compact.update(first[(first >= 0) & compact].tolist())
                        counts_seen.update(count.tolist())
                    for q, ((a, b), _) in enumerate(ps.members):
                        cur2, st2, pos2 = model_merge(cur, st, (a, b), fi + q, pos)
                        if seg_known:
                            facts["emptied"] += len(np.setdiff1d(np.unique(pos // SEG), np.unique(pos2 // SEG)))
                        cur, st, pos = cur2, st2, pos2
                    fi += len(ps.members)
                assert np.array_equal(cur, m.final)
                got_p.append(p)
                got_c.append(c)
            p, c = np.concatenate(got_p), np.concatenate(got_c)
            assert len(p) == wd and np.array_equal(p, wp) and np.array_equal(c, wc), "merges / counts vs oracle.c_train"
            assert np.array_equal(cur, fin)
            assert np.array_equal(eng.read_stream(), fin), "final stream"
            assert eng.debug_table() == table_dict(*stats(fin, st)), "pair table"
            eng.close()
    if F.complete:
        assert offs_compact, "no merge changed a compacted segment"
        assert facts["emptied"] > 0 and facts["member_across_edge"] > 0 and facts["adj_self"] > 0, facts
        assert any(120 <= x <= 136 for x in counts_seen) and any(250 <= x <= 262 for x in counts_seen), sorted(counts_seen)[:40]
        assert any(378 <= x <= 390 for x in counts_seen) and any(1 <= x <= 3 for x in counts_seen)
        if not SMALL:
            assert offs_full >= set(range(SEG)), sorted(set(range(SEG)) - offs_full)[:20]
            assert {o % SECTOR for o in offs_compact} == set(range(SECTOR)) and len({o % ROW for o in offs_compact}) > ROW // 2


# ---- statistics delta: direct counters and hashed cache -------------------------------------------------------------
def _train_chain(eng, F, cur, offs, calls, fi, weights=None):
    """bpe_train calls of `calls` merges each, every call checked against the pass model -> (merges, counts, model of
    the last call, first pass sizes)"""
    ps, cs, sizes = [], [], []
    for n in calls:
        m = partition(cur, offs, n, first_idx=fi, weights=weights)
        p, c, d = eng.train(n, first_idx=fi)
        assert d == len(m.merges) and np.array_equal(p, m.merges) and np.array_equal(c, m.counts), ("pass model", n)
        assert eng.timing()["tokens_in"] == m.tokens_in, ("tokens_in", n, m.sizes)
        sizes.append(m.sizes)
        ps.append(p)
        cs.append(c)
        cur, offs, fi = m.final, m.final_offs, fi + n
    return np.concatenate(ps), np.concatenate(cs), cur, offs, sizes


@pytest.mark.parametrize("nk", list(range(1, BATCH_MAX + 1)))
def test_delta_counters_at_the_threshold(fuzz, nk):
    """A pass of nk members with the largest V whose nk·(2V+1) counters fit MS_DELTA_WORDS (direct shared counters) and
    with the next V (hashed cache), on planted byte layouts with adjacent occurrences of one member and of two."""
    F = fuzz(200 + nk, 2)
    for r, rng in F:
        V = vmax(nk) + r                         # round 0: the last V with direct counters, round 1: the first hashed
        ids, offs = planted(seed=int(rng.integers(1 << 30)), byte_ids=True)
        total = 30
        calls = [nk, total - nk]                 # a call of nk merges: its first pass has nk members
        with F.round(r, nk=nk, V=V, direct=nk * (2 * V + 1) <= MS_DELTA_WORDS):
            assert 256 + total <= V
            eng = _engine()
            eng.set_option(__import__("minbpe_b200.engine", fromlist=["E"]).OPT_VOCAB_CAP, V)
            eng.load_stream(ids.astype(np.uint8), offs)
            p, c, fin, fo, sizes = _train_chain(eng, F, ids, offs, calls, 256)
            assert sizes[0] == [nk], sizes
            wp, wc, _, wfin = oracle.c_train(ids, offs, total, want_final=True)
            assert np.array_equal(p, wp) and np.array_equal(c, wc)
            assert np.array_equal(eng.read_stream(), wfin)
            st = np.zeros(len(wfin), dtype=bool)
            st[fo.astype(np.int64)] = True
            assert eng.debug_table() == table_dict(*stats(wfin, st))
            F.path("direct" if nk * (2 * V + 1) <= MS_DELTA_WORDS else "hashed")
            eng.close()


def test_hashed_delta_spills_to_global(fuzz):
    """Pairs with far more distinct neighbour ids per CTA than the MS_DCACHE slots of the hashed cache (ids up to 2^17):
    the cache fills and the rest goes to global atomics.  One pass of one member and one of two."""
    F = fuzz(250, 2)
    for r, rng in F:
        occ = 3000 if SMALL else 120000
        k = r + 1                                # members of the first pass
        pairs = [(70001, 70002), (70003, 70004)][:k]
        rows = []
        for q in range(occ):
            j = 0 if k == 1 or q % 3 else 1      # strictly decreasing counts
            x, y = rng.integers(FILLER0, 1 << 17, size=2)
            rows.append([x, pairs[j][0], pairs[j][1], y])
        ids = np.asarray(rows, dtype=np.int32).reshape(-1)
        offs = np.arange(0, len(ids), 4, dtype=np.uint64)
        offs = offs[rng.random(len(offs)) < 0.5]
        offs[0] = 0
        per_ticket = len(set(ids[: MS_BATCH * SEG].tolist()))
        with F.round(r, occ=occ, members=k, distinct_per_ticket=per_ticket):
            assert per_ticket > 2 * MS_DCACHE
            eng = _engine()
            eng.load_ids(ids, offs)
            fi = 1 << 17
            p, c, fin, fo, sizes = _train_chain(eng, F, ids, offs, [k, 4], fi)
            assert sizes[0] == [k]
            wp, wc, _, wfin = oracle.c_train(ids, offs, k + 4, first_idx=fi, want_final=True)
            assert np.array_equal(p, wp) and np.array_equal(c, wc)
            assert np.array_equal(eng.read_stream(), wfin)
            st = np.zeros(len(wfin), dtype=bool)
            st[fo.astype(np.int64)] = True
            assert eng.debug_table() == table_dict(*stats(wfin, st))
            F.path("hashed, spilled")
            eng.close()


# ---- large rounds ----------------------------------------------------------------------------------------------------
def _pair_bytes(rng, n, k=12):
    """about n bytes of units: one of k byte pairs with disjoint bytes and decreasing frequencies (the next merges are
    provably determined, so passes batch), or one filler byte; chunk marks at a sixth of the units"""
    a, b = np.arange(65, 65 + 2 * k, 2), np.arange(66, 66 + 2 * k, 2)
    pool = np.asarray([x for x in range(256) if not 65 <= x < 65 + 2 * k])
    p = 0.08 * 0.85 ** np.arange(k)
    units = rng.choice(k + 1, size=n * 2 // 3, p=np.append(p, 1 - p.sum()))
    lens = np.where(units < k, 2, 1)
    ends = np.cumsum(lens)
    units, lens, ends = units[ends <= n], lens[ends <= n], ends[ends <= n]
    starts = ends - lens
    data = np.empty(int(ends[-1]), dtype=np.uint8)
    pr = units < k
    data[starts[pr]] = a[units[pr]]
    data[starts[pr] + 1] = b[units[pr]]
    data[starts[~pr]] = pool[rng.integers(len(pool), size=int((~pr).sum()))]
    offs = starts[rng.random(len(starts)) < 1 / 6]
    return data, np.unique(np.concatenate([[0], offs])).astype(np.uint64)


@pytest.mark.parametrize("mode", ["batched", "seg_filter"])
def test_large_rounds(fuzz, mode):
    """Streams past the point where every warp of the merge grid holds tickets and reuses its stages many times:
    batched passes (k_merge_seg<false>, 1..4 members), and the segment filter (BPE_OPT_SEG_FILTER 2, k_merge_seg<true>)."""
    from minbpe_b200 import engine as E
    F = fuzz(300 + (mode == "seg_filter"), 1)
    for r, rng in F:
        n = 150000 if SMALL else ALL_WARPS_TOKENS + 700000
        data, offs = _pair_bytes(rng, n)
        total = 8 if SMALL else 16
        with F.round(r, mode=mode, n=n):
            eng = _engine()
            if mode == "seg_filter":
                eng.set_option(E.OPT_SEG_FILTER, 2)
            eng.load_stream(data, offs)
            ids = data.astype(np.int32)
            wp, wc, _, wfin = oracle.c_train(ids, offs, total, want_final=True)
            if mode == "batched":
                p, c, fin, fo, sizes = _train_chain(eng, F, ids, offs, [5, total - 5], 256)
                assert max(max(s) for s in sizes) > 1, sizes
                F.path("batched passes", sum(1 for s in sizes for x in s if x > 1))
            else:
                p1, c1, d1 = eng.train(5)
                p2, c2, d2 = eng.train(total - 5, first_idx=261)
                p, c = np.concatenate([p1, p2]), np.concatenate([c1, c2])
                t = eng.timing()
                assert t["filter_segments"] > 0 and t["filter_candidates"] > 0, t
                F.path("filtered passes")
            assert np.array_equal(p, wp) and np.array_equal(c, wc)
            got = eng.read_stream()
            assert np.array_equal(got, wfin)
            if mode == "batched":
                st = np.zeros(len(wfin), dtype=bool)
                st[fo.astype(np.int64)] = True
                assert eng.debug_table() == table_dict(*stats(wfin, st))
            eng.close()


# ---- texts -----------------------------------------------------------------------------------------------------------
WORDS = ["'s", "'S", "'t", "'T", "'re", "'RE", "'Ve", "'ll", "'LL", "'d", "'M", "don't", "DON'T", "ſ", "ſt", "Straße",
         "HelloWorld", "XMLHttpRequest", "iPhone", "McDonald's", "ǅungla", "ʰAʰb", "中文", "中A", "あ", "́", "!́abc", "ः",
         "⃝", "1́", "áb", "12", "123", "1234567", "3.14", "½", "\r\n", "\r", "\n", "\n\n", "\r\n\r\n", " \r\n", "  ",
         " ", "\t", "\u0085", "　", "𝒜", "😀", "𐍈", "𝟘𝟙", "!!", "...", "/\n/", "a/b", "x's'll", " 'sfoo",
         "the", " the", " quick", " brown", "fox", "é", "日本"]


def random_text(rng, n_chars):
    out, size = [], 0
    while size < n_chars:
        r = rng.random()
        if r < 0.6:
            w = str(rng.choice(WORDS))
        elif r < 0.9:
            w = "".join(rng.choice(list("abcdeABé日 1'\n"), size=int(rng.integers(1, 9))))
        else:
            w = "".join(rng.choice(list("xyzXYZ"), size=int(rng.integers(20, 70))))    # long letter runs
        out.append(w)
        size += len(w)
    return "".join(out)


def oracle_split(text, pattern):
    return oracle.split_to_stream(text, regex.compile(pattern))


# ---- training entry points ---------------------------------------------------------------------------------------
def test_training_entry_points(fuzz):
    """load_chunks_weighted (weights past 2^32 in some rounds), RegexTokenizer.train(dedup=True), train_from_iterator
    with and without special_tokens, BasicTokenizer.train: merges and counts of oracle.c_train on the same chunks."""
    from minbpe_b200 import BasicTokenizer, RegexTokenizer
    from minbpe_b200.tokenizer import default_engine
    F = fuzz(404, 6 if SMALL else 24)
    pats = _patterns()
    for r, rng in F:
        name = str(rng.choice(list(pats)))
        which, pattern = pats[name]
        kind = ["weighted", "dedup", "iterator", "iterator_special", "basic", "weighted"][r % 6]
        n_chars = int(rng.choice([300, 5000, 70000 if SMALL else 150000]))
        text = random_text(rng, n_chars)
        merges = int(rng.integers(5, 30 if SMALL else 80))
        with F.round(r, kind=kind, pattern=name, chars=n_chars, merges=merges):
            if kind == "weighted":
                data, offs = oracle_split(text, pattern)
                ub, uo, uw = oracle.c_dedup_chunks(data, offs)
                w = uw.astype(np.int64)
                if rng.random() < 0.5:
                    w = weighted_entries(np.zeros(0), uo, seed=int(rng.integers(1 << 30)), big=True)
                eng = _engine()
                eng.load_chunks_weighted(ub, uo, w.astype(np.uint64))
                ids = ub.astype(np.int32)
                wp, wc, wd = oracle.c_train(ids, uo, merges, weights=w)
                cut = int(rng.integers(1, merges + 1))
                p1, c1, d1 = eng.train(cut)
                assert _launches(eng) > 0
                p2, c2, d2 = eng.train(merges - cut, first_idx=256 + cut) if d1 == cut else (p1[:0], c1[:0], 0)
                assert d1 + d2 == wd and np.array_equal(np.concatenate([p1, p2]), wp) and np.array_equal(np.concatenate([c1, c2]), wc)
                F.path("load_chunks_weighted")
                eng.close()
                continue
            if kind == "basic":
                tok = BasicTokenizer()
                ids = np.frombuffer(text.encode("utf-8"), dtype=np.uint8).astype(np.int32)
                wp, wc, wd = oracle.c_train(ids, None, merges)
                tok.train(text, 256 + merges)
                assert _launches(tok.engine) > 0
                assert [list(k) for k in tok.merges] == wp.tolist()
                F.path("BasicTokenizer.train")
                continue
            tok = RegexTokenizer(pattern)
            eng = tok.engine
            if kind == "dedup":
                data, offs = oracle_split(text, pattern)
                wp, wc, wd = oracle.c_train(data.astype(np.int32), offs, merges)
                tok.train(text, 256 + merges, dedup=True)
                device = len(text.encode("utf-8")) >= tok.DEVICE_SPLIT_MIN_BYTES
                if device:
                    assert eng.dedup_stats()["text_chunks"] == len(offs)
                F.path("train(dedup) device split" if device else "train(dedup) host split")
            else:
                special = None
                cuts = sorted(rng.choice(np.arange(1, len(text)), size=min(len(text) - 1, int(rng.integers(1, 12))), replace=False).tolist())
                docs = [text[a:b] for a, b in zip([0] + cuts, cuts + [len(text)])]
                if kind == "iterator_special":
                    special = {s: 300000 + i for i, s in enumerate(random_specials(rng, int(rng.integers(1, 6))))}
                    docs = [with_occurrences(rng, d, list(special)) for d in docs]
                parts = []
                for d in docs:
                    parts += RegexTokenizer._ordinary_parts(d, special) if special else [d]
                bufs, offl, base = [], [], 0
                for part in parts:
                    d, o = oracle_split(part, pattern)
                    bufs.append(d)
                    offl.append(o + base)
                    base += len(d)
                data = np.concatenate(bufs) if bufs else np.zeros(0, np.uint8)
                offs = np.concatenate(offl).astype(np.uint64) if offl else np.zeros(0, np.uint64)
                wp, wc, wd = oracle.c_train(data.astype(np.int32), offs, merges)
                try:
                    tok.train_from_iterator(iter(docs), 256 + merges, special_tokens=special)
                except ValueError:
                    assert wd < merges
                    F.path("ran out of pairs")
                    continue
                assert eng.dedup_stats()["text_chunks"] == len(offs)
                F.path("train_from_iterator" + (" + specials" if special else ""))
                if special:
                    assert tok.special_tokens == special
            assert wd == merges and [list(k) for k in tok.merges] == wp.tolist()


# ---- encode and decode -------------------------------------------------------------------------------------------
def _vocab(merges):
    v = [bytes([i]) for i in range(256)]
    for a, b in merges.tolist():
        v.append(v[a] + v[b])
    return v


def _device_decode(eng, ids, vocab, F):
    blob = b"".join(vocab)
    lens = np.asarray([len(x) for x in vocab], dtype=np.uint32)
    starts = np.zeros(len(vocab), dtype=np.uint64)
    np.cumsum(lens[:-1], out=starts[1:])
    got, bad = eng.decode(ids, np.frombuffer(blob, dtype=np.uint8), starts, lens)
    assert bad == -1 and got == b"".join(vocab[i] for i in ids.tolist()), "bpe_decode"
    F.path("decode")


def memo_twins(rng):
    """words of 33..48 bytes that share their first 32 bytes and differ only in the rest (one memo key each)"""
    head = "".join(rng.choice(list("qwrtpsdfgh"), size=32))
    return [" " + head + "".join(rng.choice(list("zxcv"), size=int(rng.integers(1, E2_LMAX - 32)))) for _ in range(6)]


def encode_text(rng):
    r = rng.random()
    text = random_text(rng, int(rng.choice([40, 600, 3000, 20000, 90000])))
    if r < 0.4:
        twins = memo_twins(rng)
        text = "".join(str(rng.choice(twins)) + (" a" if rng.random() < 0.5 else "") for _ in range(200)) + text
    if rng.random() < 0.1:
        text += " " + "ab" * (int(rng.choice([ENC_LONG_MAX - 2, ENC_LONG_MAX, ENC_LONG_MAX + 3])) // 2)
    raw = text.encode("utf-8")
    if rng.random() < 0.5:
        cut = int(rng.choice([1, 7, 8, 9, E2_TILE - 1, E2_TILE, E2_TILE + 1, E2_TILE + E2_HALO - 1, E2_TILE + E2_HALO,
                              E2_TILE + E2_HALO + 1, SP_TILE - 1, SP_TILE, SP_TILE + 1, 2 * E2_TILE + 17, 1 << 14, (1 << 14) + 5,
                              (1 << 16) - 1, 1 << 16, (1 << 16) + 1]))
        raw = raw[:cut]
    return raw.decode("utf-8", errors="ignore")


def test_encode_and_decode(fuzz):
    """Engine.encode (host offsets), encode_text_gpt4 under every split pattern option, encode_docs with document edges
    at tile and piece edges, and the classes' encode / encode_batch / encode_ordinary_batch, against oracle.c_encode of
    the oracle split; memo tables of 2^6 and 2^8 slots, byte permutations, split pieces of 4096 and 1<<14 bytes; the
    device decode of the ids against the join of the vocabulary's bytes."""
    from minbpe_b200 import RegexTokenizer
    from minbpe_b200 import engine as E
    F = fuzz(505, 12 if SMALL else 60)
    pats = _patterns()
    train_text = random_text(np.random.default_rng(5), 40000 if SMALL else 200000)
    trained = {}
    for r, rng in F:
        name = str(rng.choice(list(pats)))
        which, pattern = pats[name]
        if name not in trained:
            t = RegexTokenizer(pattern)
            t.train(train_text, 256 + (60 if SMALL else 300))
            trained[name] = t
        tok = trained[name]
        merges = tok._merge_array()
        vocab = _vocab(merges)
        text = encode_text(rng)
        if not text:
            continue
        memo = int(rng.choice([0, 6, 8]))
        piece = int(rng.choice([0, 0, 4096, 1 << 14]))
        perm = rng.permutation(256).astype(np.uint8) if rng.random() < 0.2 else None
        with F.round(r, pattern=name, bytes=len(text.encode()), memo=memo, piece=piece, perm=perm is not None):
            eng = tok.engine
            data, offs = oracle_split(text, pattern)
            want = oracle.c_encode(data, offs, merges, perm)
            eng.set_option(E.OPT_ENC_MEMO_LOG2, memo)
            eng.set_option(E.OPT_SPLIT_PIECE, piece)
            eng.set_option(E.OPT_SPLIT_PATTERN, which)
            try:
                got = eng.encode(data, offs, merges, perm)
                assert np.array_equal(got, want), "Engine.encode (host offsets)"
                F.path("encode offsets")
                try:
                    got = eng.encode_text_gpt4(data.tobytes(), merges, perm)
                    st = eng.encode_stats()
                    assert st["pieces"] > 0
                    assert np.array_equal(got, want), "encode_text_gpt4"
                    F.path("encode_text fallback" if st["fallback_pieces"] else "encode_text memo")
                except E.EngineError as ex:        # a tiny piece size may find no letter+space cut: a clean error
                    assert "cut point" in str(ex) and piece, ex
                    F.path("no cut point")
                # documents with edges at tile and piece edges
                raw = data.tobytes()
                edges = [x for x in (E2_TILE, E2_TILE + E2_HALO, SP_TILE, 4096, 1 << 14) if x < len(raw)]
                edges += rng.integers(0, len(raw), size=int(rng.integers(0, 5))).tolist()
                bounds = sorted({0} | {e for e in edges if e > 0})
                bounds = [b for b in bounds if b == 0 or (raw[b] & 0xC0) != 0x80]   # cut at code points only
                docs = [raw[a:b] for a, b in zip(bounds, bounds[1:] + [len(raw)])]
                try:
                    ids, o = eng.encode_docs(raw, np.asarray(bounds, dtype=np.uint64), merges, perm)
                    for j, d in enumerate(docs):
                        dd, do = oracle_split(d.decode("utf-8"), pattern)
                        assert np.array_equal(ids[o[j]:o[j + 1]], oracle.c_encode(dd, do, merges, perm)), ("encode_docs", j)
                    F.path("encode_docs")
                except E.EngineError as ex:
                    assert "cut point" in str(ex) and piece, ex
                    F.path("no cut point")
            finally:
                eng.set_option(E.OPT_ENC_MEMO_LOG2, 0)
                eng.set_option(E.OPT_SPLIT_PIECE, 0)
            assert _launches(eng) > 0
            if perm is None:
                tok.DEVICE_SPLIT_MIN_BYTES = int(rng.choice([0, 1 << 16]))
                try:
                    assert tok.encode_ordinary(text) == want.tolist(), "encode_ordinary"
                    assert tok.encode(text, allowed_special="none") == want.tolist(), "encode"
                    texts = [d.decode("utf-8") for d in docs]
                    wants = [oracle.c_encode(*oracle_split(t, pattern), merges).tolist() for t in texts]
                    assert tok.encode_ordinary_batch(texts) == wants, "encode_ordinary_batch"
                    assert tok.encode_batch(texts, allowed_special="all") == wants, "encode_batch"
                    F.path("classes, device split" if tok.DEVICE_SPLIT_MIN_BYTES == 0 else "classes")
                finally:
                    tok.DEVICE_SPLIT_MIN_BYTES = RegexTokenizer.DEVICE_SPLIT_MIN_BYTES
            _device_decode(eng, want, vocab, F)


def test_memo_key_twins(fuzz):
    """Chunks of 48 bytes that share their first 32 bytes and their memo tag (tests/hash_craft.py), and differ only in
    their last 16, in one piece and across calls: the memo compares every key word, so each chunk keeps its own ids."""
    import hash_craft as H
    from minbpe_b200 import engine as E
    F = fuzz(550, 2 if SMALL else 8)
    gpt4 = _patterns()["gpt4"][1]
    d0, o0 = oracle_split(random_text(np.random.default_rng(55), 40000), gpt4)
    merges = oracle.c_train(d0.astype(np.int32), o0, 120)[0]
    for r, rng in F:
        head = bytes(rng.choice(list(b"abcdefgh"), size=32).tolist())
        a = head + bytes(rng.integers(0, 256, size=16).tolist())
        b = H.e2_collision(a, head + bytes(rng.integers(0, 256, size=8).tolist()))
        assert H.e2_tag(a) == H.e2_tag(b) and a[:32] == b[:32]
        memo = int(rng.choice([0, 6, 8]))
        fd, fo = oracle_split(random_text(rng, 70000), gpt4)
        ends = np.append(fo[1:], len(fd)).astype(np.int64)
        fill = [fd[x:y].tobytes() for x, y in zip(fo.astype(np.int64).tolist(), ends.tolist())]
        k = int(rng.integers(1, len(fill)))
        first = [a, b] if rng.random() < 0.5 else [b, a]
        with F.round(r, chunk_bytes=len(a), memo=memo):
            eng = _engine()
            eng.set_option(E.OPT_ENC_MEMO_LOG2, memo)
            for chunks in (fill[:k] + first + fill[k:] + first[::-1], fill[:k] + [a] + fill[k:], fill + [b, a, b]):
                data = np.frombuffer(b"".join(chunks), dtype=np.uint8)
                offs = np.zeros(len(chunks), dtype=np.uint64)
                np.cumsum([len(c) for c in chunks[:-1]], out=offs[1:])
                got = eng.encode(data, offs, merges)
                assert np.array_equal(got, oracle.c_encode(data, offs, merges)), "Engine.encode"
                assert eng.encode_stats()["pieces"] > 0
                F.path("memo")
            eng.close()


# ---- special tokens ----------------------------------------------------------------------------------------------
def random_specials(rng, k):
    """k distinct specials of 1..48 utf-8 bytes: prefix chains (in both dict orders), a shared first byte, random ones"""
    out = []
    base = "".join(rng.choice(list("<|>ab[]é"), size=int(rng.integers(4, 40))))
    while len(out) < k:
        r = rng.random()
        if r < 0.35:
            s = base[: int(rng.integers(1, len(base) + 1))]           # a prefix chain
        elif r < 0.6:
            s = "<" + "".join(rng.choice(list("|xyé1 "), size=int(rng.integers(0, 20))))   # shared first byte
        else:
            s = "".join(rng.choice(list("<|>/sSeE 日!\n"), size=int(rng.integers(1, 30))))
        b = s.encode("utf-8")
        if not (1 <= len(b) <= E2_LMAX) or s in out:
            continue
        out.append(s)
    if rng.random() < 0.5:
        out.sort(key=len)                                  # shorter first
    elif rng.random() < 0.5:
        out.sort(key=len, reverse=True)                    # longer first
    return out


def with_occurrences(rng, text, names):
    """the text with specials inserted: adjacent ones, truncated ones (ordinary text)"""
    if not text:
        return text
    cuts = sorted(rng.integers(0, len(text) + 1, size=int(rng.integers(1, 12))).tolist())
    out, prev = [], 0
    for c in cuts:
        out.append(text[prev:c])
        prev = c
        r = rng.random()
        s = str(rng.choice(names))
        if r < 0.6:
            out.append(s)
        elif r < 0.8:
            out.append(s + str(rng.choice(names)))              # adjacent
        else:
            out.append(s[: int(rng.integers(0, len(s)))])       # truncated
    out.append(text[prev:])
    return "".join(out)


def ref_encode(text, special, merges, pattern):
    """regex.py:152-163: re.split on the alternation in dict order, oracle.c_encode of every part"""
    if not special:
        return oracle.c_encode(*oracle_split(text, pattern), merges).tolist() if text else []
    out = []
    for i, part in enumerate(re.split("(" + "|".join(re.escape(k) for k in special) + ")", text)):
        if i % 2:
            out.append(special[part])
        elif part:
            out += oracle.c_encode(*oracle_split(part, pattern), merges).tolist()
    return out


def test_special_token_sets(fuzz):
    """Random sets of 1..5 and of 65..300 specials through encode (device front end, k_special_find) and encode_batch,
    with random allowed subsets, against re.split + oracle.c_encode."""
    from minbpe_b200 import RegexTokenizer
    F = fuzz(606, 10 if SMALL else 50)
    pats = _patterns()
    train_text = random_text(np.random.default_rng(6), 30000 if SMALL else 150000)
    trained = {}
    for r, rng in F:
        name = str(rng.choice(list(pats)))
        which, pattern = pats[name]
        if name not in trained:
            t = RegexTokenizer(pattern)
            t.train(train_text, 256 + (40 if SMALL else 200))
            trained[name] = t
        tok = trained[name]
        merges = tok._merge_array()
        k = int(rng.integers(1, 6)) if r % 2 == 0 else int(rng.integers(65, 301))
        names = random_specials(rng, k)
        special = {s: 500000 + i for i, s in enumerate(names)}
        body = random_text(rng, int(rng.choice([100, 3000, 20000])))
        text = with_occurrences(rng, body, names)
        allowed = "all" if rng.random() < 0.6 else set(rng.choice(names, size=int(rng.integers(0, k + 1)), replace=False).tolist())
        piece = int(rng.choice([0, 0, 4096]))
        with F.round(r, pattern=name, specials=k, allowed="all" if allowed == "all" else len(allowed), piece=piece):
            from minbpe_b200 import engine as E
            tok.register_special_tokens(special)
            tok.DEVICE_SPLIT_MIN_BYTES = 0
            use = special if allowed == "all" else {s: v for s, v in special.items() if s in allowed}
            try:
                want = ref_encode(text, use, merges, pattern)
                tok.engine.set_option(E.OPT_SPLIT_PIECE, piece)
                try:
                    got = tok.encode(text, allowed_special=allowed)
                    st = tok.engine.encode_stats()
                    assert got == want, "encode"
                    F.path("device specials" if use else "no specials allowed")
                    if use:
                        assert st["pieces"] > 0
                except E.EngineError as ex:
                    assert "cut point" in str(ex) and piece, ex
                    F.path("no cut point")
                tok.engine.set_option(E.OPT_SPLIT_PIECE, 0)
                cuts = sorted(set(rng.integers(0, len(text) + 1, size=4).tolist()))
                docs = [text[a:b] for a, b in zip([0] + cuts, cuts + [len(text)])]
                assert tok.encode_batch(docs, allowed_special=allowed) == [ref_encode(d, use, merges, pattern) for d in docs]
                F.path("encode_batch specials")
            finally:
                tok.engine.set_option(E.OPT_SPLIT_PIECE, 0)
                tok.DEVICE_SPLIT_MIN_BYTES = RegexTokenizer.DEVICE_SPLIT_MIN_BYTES
                tok.register_special_tokens({})


# ---- the reference classes' answers ----------------------------------------------------------------------------------
@pytest.mark.parametrize("script", ["emu_fuzz_train_ref", "emu_fuzz_special"])
def test_reference_goldens(fuzz, script, capsys):
    """tests/golden/golden_fuzz_train.json and golden_fuzz_special.json (what the unmodified reference classes returned
    on random texts) replayed in-process: train / encode / save of the classes, and encode with specials with every
    text on the device path (DEVICE_SPLIT_MIN_BYTES = 0)."""
    import importlib
    from minbpe_b200.tokenizer import default_engine
    F = fuzz(700 + (script == "emu_fuzz_special"), 1)
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    try:
        mod = importlib.import_module(script)
    finally:
        sys.path.pop(0)
    for r, _ in F:
        with F.round(r, script=script):
            assert mod.main(100, 5, False) == 0
            out = capsys.readouterr().out
            assert ("emu fuzz train ok" in out) if script == "emu_fuzz_train_ref" else ("100 of 100 rounds" in out), out
            assert _launches(default_engine()) > 0
            F.path("reference rounds", 100)
