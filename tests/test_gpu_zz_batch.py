"""GPU: the batched merge pass of bpe_train (k_select_batch, k_merge_seg's delta_batch, k_apply_delta per member,
k_wt_delta_seg), pinned to the oracle pass by pass through the host model of tests/batch_model.py.

Engine.timing()["tokens_in"] is the sum over the passes of the stream length each pass read, so it equals the model's
prediction only when the device batched exactly the members the rule proves.  The corpora plant the layouts where a
per-member delta goes wrong (adjacent members in both orders, a member next to itself, next to a segment edge or a
chunk mark), and the tests check the pair table and the stream after every merge count of the first batched passes,
chained calls, the V <= 2^21 limit of batching, table growth that lands inside a batch and weighted counts above 2^32."""
import os

import numpy as np
import pytest
import regex

import oracle
from batch_model import BATCH_MAX, partition, planted, short_chunks, stats, table_dict, weighted_entries, with_filler_pairs

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller corpora, fewer merges

GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
PLANTED_OFFSETS = range(510, 513) if SMALL else range(509, 515)
PLANTED_FACTS = ("full_batch", "adj_fwd", "adj_rev", "adj_self", "adj_seg_edge", "adj_chunk_mark", "member_across_seg_edge")


def _engine(host_batch=8):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_BATCH, host_batch)         # several host batches: maybe_repack runs between them
    return eng


class Corpus:
    def __init__(self, ids, offs, merges, first_idx=256, as_bytes=False, facts=()):
        self.ids, self.offs, self.merges, self.first_idx, self.as_bytes, self.facts = ids, offs, merges, first_idx, as_bytes, facts

    def load(self, eng):
        if self.as_bytes:
            eng.load_stream(self.ids.astype(np.uint8), self.offs)
        else:
            eng.load_ids(self.ids, self.offs)


def _planted(**kw):
    ids, offs = planted(offsets=PLANTED_OFFSETS, **kw)
    return ids, offs, int(ids.max()) + 1


def _corpus(name, taylorswift):
    if name == "planted":
        ids, offs, fi = _planted()
        return Corpus(ids, offs, 40, fi, facts=PLANTED_FACTS)
    if name == "short_chunks":
        ids, offs = short_chunks(n_tokens=8000 if SMALL else 20000)
        return Corpus(ids, offs, 120 if SMALL else 200, 512, facts=("adj_chunk_mark",))
    if name.startswith("taylorswift"):
        text = taylorswift[: 60000] if SMALL and name != "taylorswift_basic" else taylorswift
        data, offs = oracle.split_to_stream(text, GPT4 if name == "taylorswift_gpt4" else None)
        # the byte-level one: 360 segments, trained until they are less than half full (re-packing)
        facts = ("full_batch", "repack_possible") if name == "taylorswift_basic" else ("full_batch",)
        return Corpus(np.asarray(data, dtype=np.int32), offs, 320 if name == "taylorswift_basic" else (150 if SMALL else 300),
                      as_bytes=True, facts=facts)
    from minbpe_b200.synth import generate
    text = generate(1337, (64 << 10) if SMALL else (512 << 10)).tobytes().decode("utf-8")
    data, offs = oracle.split_to_stream(text, GPT4)
    return Corpus(np.asarray(data, dtype=np.int32), offs, 150 if SMALL else 300, as_bytes=True, facts=("full_batch",))


@pytest.mark.parametrize("name", ["planted", "short_chunks", "taylorswift_basic", "taylorswift_gpt4", "synth"])
def test_partition_and_parity(name, taylorswift):
    """Merges and counts are the oracle's, the stream is the oracle's, and tokens_in is the model's: the device batched
    exactly the members the rule proves, no fewer and no more."""
    c = _corpus(name, taylorswift)
    wp, wc, wd, fin = oracle.c_train(c.ids, c.offs, c.merges, first_idx=c.first_idx, want_final=True)
    m = partition(c.ids, c.offs, c.merges, c.first_idx)
    assert np.array_equal(m.merges, wp) and np.array_equal(m.counts, wc) and np.array_equal(m.final, fin)
    for f in c.facts:
        assert m.facts[f] > 0, (name, f, dict(m.facts))
    assert max(m.sizes) > 1
    eng = _engine()
    c.load(eng)
    p, cnt, d = eng.train(c.merges, first_idx=c.first_idx)
    tm = eng.timing()
    assert d == wd and np.array_equal(p, wp) and np.array_equal(cnt, wc)
    assert tm["tokens_in"] == m.tokens_in, (tm["tokens_in"], m.tokens_in, m.sizes)
    assert np.array_equal(eng.read_stream(), fin)
    assert eng.debug_table() == table_dict(*stats(m.final, _starts(m)))
    eng.close()


def _starts(m):
    s = np.zeros(len(m.final), dtype=bool)
    s[m.final_offs.astype(np.int64)] = True
    return s


def test_table_at_every_cut():
    """train(k) for every k through the first batched passes: max_iter cuts a batch after each member index.  The
    incremental table equals the recount of the oracle's stream after k merges, and the stream equals that stream."""
    ids, offs, fi = _planted()
    K = 16 if SMALL else 40
    m = partition(ids, offs, K, fi)
    assert m.sizes[:3] == [BATCH_MAX] * 3          # P1..P4, P5..P8, then four second-level pairs
    eng = _engine()
    cut_at = set()
    for k in range(1, K + 1):
        mk = partition(ids, offs, k, fi)
        assert mk.tokens_in == m.tokens_in_upto(k)
        if k <= 3 * BATCH_MAX:
            cut_at.add(mk.sizes[-1])
        eng.load_ids(ids, offs)
        p, c, d = eng.train(k, first_idx=fi)
        assert d == k and np.array_equal(p, m.merges[:k]) and np.array_equal(c, m.counts[:k]), k
        assert eng.timing()["tokens_in"] == mk.tokens_in, (k, mk.sizes)
        _, _, _, fin = oracle.c_train(ids, offs, k, first_idx=fi, want_final=True)
        assert np.array_equal(mk.final, fin)
        assert np.array_equal(eng.read_stream(), fin), k
        assert eng.debug_table() == table_dict(*oracle.c_get_stats(fin, mk.final_offs)), k
    assert cut_at == set(range(1, BATCH_MAX + 1))   # the last pass of a call held 1 .. BATCH_MAX members
    eng.close()


def test_continuation_of_chained_calls():
    """Calls of irregular sizes, each continuing the previous one's table: together they equal one call of the total, and
    each call batched as the model does with that call's cap."""
    ids, offs, fi = _planted()
    sizes = [3, 1, 4, 1, 5, 9, 2, 6]
    total = sum(sizes)
    wp, wc, wd = oracle.c_train(ids, offs, total, first_idx=fi)
    eng = _engine()
    eng.load_ids(ids, offs)
    cur, cur_offs, at = ids, offs, 0
    got_p, got_c = [], []
    for s in sizes:
        m = partition(cur, cur_offs, s, fi + at)
        p, c, d = eng.train(s, first_idx=fi + at)
        assert d == s and np.array_equal(p, m.merges) and np.array_equal(c, m.counts), at
        assert eng.timing()["tokens_in"] == m.tokens_in, (at, m.sizes)
        got_p.append(p)
        got_c.append(c)
        cur, cur_offs, at = m.final, m.final_offs, at + s
    assert np.array_equal(np.concatenate(got_p), wp) and np.array_equal(np.concatenate(got_c), wc)
    assert np.array_equal(eng.read_stream(), cur)
    assert eng.debug_table() == table_dict(*oracle.c_get_stats(cur, cur_offs))
    eng.close()


def test_batch_fits_edge():
    """V = 2^21 is the largest vocabulary that batches; 2^21 + 1 applies one merge per pass.  Both give the same merges,
    table and stream, and tokens_in tells which partition ran.  A stream with ids up to 2^21 - 64 and new ids up to V - 1
    puts delta indices at the top of every member's vector."""
    from minbpe_b200 import engine as E
    ids, offs, fi = _planted()
    K = 8 if SMALL else 24
    batched = partition(ids, offs, K, fi)
    single = partition(ids, offs, K, fi, cap=1)
    assert np.array_equal(batched.merges, single.merges) and batched.tokens_in < single.tokens_in
    out = {}
    for cap, m in ((1 << 21, batched), ((1 << 21) + 1, single)):
        eng = _engine()
        eng.set_option(E.OPT_VOCAB_CAP, cap)
        eng.load_ids(ids, offs)
        p, c, d = eng.train(K, first_idx=fi)
        assert d == K and np.array_equal(p, m.merges) and np.array_equal(c, m.counts), cap
        assert eng.timing()["tokens_in"] == m.tokens_in, cap
        out[cap] = (p.tolist(), c.tolist(), eng.debug_table(), eng.read_stream().tolist())
        eng.close()
    assert out[1 << 21] == out[(1 << 21) + 1]
    # ids near the top: filler ids end at 2^21 - 64, the K new ids end at V - 1 = 2^21 - 1
    top = (1 << 21) - 64
    hi = ids.copy()
    f = hi >= 2000
    hi[f] = hi[f] - int(hi[f].max()) + top
    fi_hi = (1 << 21) - K
    m = partition(hi, offs, K, fi_hi)
    wp, wc, wd = oracle.c_train(hi, offs, K, first_idx=fi_hi)
    assert np.array_equal(m.merges, wp) and max(m.sizes) == BATCH_MAX
    eng = _engine()
    eng.load_ids(hi, offs)
    p, c, d = eng.train(K, first_idx=fi_hi)
    assert d == K and np.array_equal(p, wp) and np.array_equal(c, wc)
    assert eng.timing()["tokens_in"] == m.tokens_in
    assert eng.debug_table() == table_dict(*oracle.c_get_stats(m.final, m.final_offs))
    eng.close()


@pytest.mark.parametrize("member", [1, 2, 3])
def test_table_growth_inside_a_batch(member):
    """The first table overflow lands on member 1, 2 or 3 of the first pass (the model's reservation count against the load
    limit floor(0.6 * 2^log2) says where): the host grows the table and re-runs every member's apply.  Merges stay the
    oracle's, for several host batch sizes, and the grown table equals the recount."""
    from minbpe_b200 import engine as E
    assert member < BATCH_MAX
    base, offs0 = planted(offsets=())
    log2 = 14
    m0 = partition(base, offs0, 1, int(base.max()) + 1)
    limit = int(0.6 * (1 << log2))
    extra = limit - m0.init_pairs - sum(partition(base, offs0, member, int(base.max()) + 1).passes[0].new_pairs)
    ids, offs = with_filler_pairs(base, offs0, extra)
    fi = int(ids.max()) + 1
    K = 12 if SMALL else 24
    m = partition(ids, offs, K, fi)
    assert m.sizes[0] == BATCH_MAX and m.first_overflow(log2) == (0, member)
    wp, wc, wd = oracle.c_train(ids, offs, K, first_idx=fi)
    for host_batch in (1, 2, 3, 7):
        eng = _engine(host_batch)
        eng.set_option(E.OPT_TABLE_LOG2, log2)
        # up to the member before: no growth, and table_used is the model's count of reserved slots
        eng.load_ids(ids, offs)
        eng.train(member, first_idx=fi)
        tm = eng.timing()
        assert tm["table_slots"] == 1 << log2 and tm["table_used"] == partition(ids, offs, member, fi).used_after(1) == limit
        eng.load_ids(ids, offs)
        p, c, d = eng.train(K, first_idx=fi)
        tm = eng.timing()
        assert d == K and np.array_equal(p, wp) and np.array_equal(c, wc), host_batch
        assert tm["table_slots"] > 1 << log2 and tm["tokens_in"] == m.tokens_in
        assert eng.debug_table() == table_dict(*oracle.c_get_stats(m.final, m.final_offs))
        eng.close()


def _weighted_cases(taylorswift):
    ids, offs = planted(offsets=PLANTED_OFFSETS, byte_ids=True)
    yield "planted", ids, offs, weighted_entries(ids, offs, seed=1, big=True)
    data, toffs = oracle.split_to_stream(taylorswift[: 60000] if SMALL else taylorswift, GPT4)
    ub, uo, uw = oracle.c_dedup_chunks(data, toffs)
    yield "taylorswift", ub.astype(np.int32), uo, uw.astype(np.int64)
    w = uw.astype(np.int64).copy()
    w[:: 37] += 1 << 33
    yield "taylorswift_big", ub.astype(np.int32), uo, w


@pytest.mark.parametrize("case", ["planted", "taylorswift", "taylorswift_big"])
def test_weighted(case, taylorswift):
    """load_chunks_weighted: merges and counts are the oracle's weighted loop's (counts above 2^32 where the weights say
    so), tokens_in is the model's partition over the entry stream, and the table at the first cuts is the weighted
    recount."""
    name, ids, offs, w = next(x for x in _weighted_cases(taylorswift) if x[0] == case)
    K = 60 if SMALL else 160
    m = partition(ids, offs, K, weights=w)
    wp, wc, wd = oracle.c_train(ids, offs, K, weights=w)
    assert np.array_equal(m.merges, wp) and np.array_equal(m.counts, wc)
    assert max(m.sizes) == BATCH_MAX
    if case != "taylorswift":
        assert int(wc.max()) >= 1 << 33
    if case == "planted":
        for f in ("adj_fwd", "adj_rev", "adj_self", "adj_chunk_mark"):
            assert m.facts[f] > 0, (f, dict(m.facts))
    data = ids.astype(np.uint8)
    eng = _engine()
    eng.load_chunks_weighted(data, offs, w.astype(np.uint64))
    p, c, d = eng.train(K)
    assert d == wd and np.array_equal(p, wp) and np.array_equal(c, wc)
    assert eng.timing()["tokens_in"] == m.tokens_in
    assert eng.debug_table() == table_dict(*stats(m.final, _starts(m), w))
    for k in range(1, 2 * BATCH_MAX + 2):
        mk = partition(ids, offs, k, weights=w)
        eng.load_chunks_weighted(data, offs, w.astype(np.uint64))
        p, c, d = eng.train(k)
        assert d == k and np.array_equal(p, wp[:k]) and np.array_equal(c, wc[:k]), k
        assert eng.timing()["tokens_in"] == mk.tokens_in, k
        assert np.array_equal(eng.read_stream(), mk.final), k
        assert eng.debug_table() == table_dict(*stats(mk.final, _starts(mk), w)), k
    eng.close()
