"""GPU: the segment filter (BPE_OPT_SEG_FILTER; k_seg_filter.cuh, k_merge_seg<true>, k_sig_rebuild_cand) pinned to the host
model of tests/filter_model.py.  A segment the filter fails to list is a merge that silently never happens there, and a
segment it lists needlessly costs only time, so the tests check both sides exactly: every call's merges, counts, final
stream and pair table against the oracle, and filter_candidates / filter_segments (the sums of the list lengths and of
nseg over the filtered merges) against the model's candidate rule.

The corpora put the merged pair only across segment edges, next to segments of 1 and 2 tokens and across one and two
empty segments (an empty last segment included), a chunk-marked b after an a at an edge, pairs whose signature bit
collides with the merged pair's, ids above 2^16 with first_idx above 2^21, a pair (a,a) and re-packing between filtered
merges, table growth on a filtered merge, chained calls and a resumed byte stream."""
import os

import numpy as np
import pytest

import filter_model as F
import oracle
from batch_model import stats, table_dict

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs
CHAIN_MERGES = 512 + 1024 + 5                       # both chains, the two (Z,B) merges, (r,r), two filler merges
CHAIN_FACTS = ("pair_only_across_edges", "occurrence_across_empty_segment", "occurrence_across_two_empty_segments",
               "listed_segment_of_1", "listed_segment_of_2", "empty_last_segment", "marked_b_after_edge",
               "listed_by_colliding_bit", "aa_merge_while_filtering")


def _engine(mode, opt_batch=64, table_log2=0):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_SEG_FILTER, mode)
    eng.set_option(E.OPT_BATCH, opt_batch)
    eng.set_option(E.OPT_TABLE_LOG2, table_log2)
    return eng


def _check_call(eng, st, r, got, oracle_merges, oracle_counts):
    """One bpe_train call against the model's result `r` (state `st` after the call) and the oracle's merges."""
    p, c, d = got
    tm = eng.timing()
    assert d == r.n_done == len(oracle_merges)
    assert np.array_equal(r.merges, oracle_merges) and np.array_equal(r.counts, oracle_counts)
    assert np.array_equal(p, r.merges) and np.array_equal(c, r.counts)
    assert np.array_equal(eng.read_stream(), st.ids)
    assert eng.debug_table() == table_dict(*stats(st.ids, st.start))
    assert (tm["filter_candidates"], tm["filter_segments"]) == (r.candidates, r.segments), dict(r.facts)


def _run(ids, offs, K, first_idx, mode, opt_batch=64, table_log2=0, facts=()):
    wp, wc, wd, fin = oracle.c_train(ids, offs, K, first_idx=first_idx, want_final=True)
    st = F.State(ids, offs)
    r = F.train(st, K, first_idx, mode=mode, opt_batch=opt_batch, table_log2=table_log2)
    assert np.array_equal(st.ids, fin)
    for f in facts:
        assert r.facts[f] > 0, (f, dict(r.facts))
    eng = _engine(mode, opt_batch, table_log2)
    eng.load_ids(ids, offs)
    _check_call(eng, st, r, eng.train(K, first_idx=first_idx), wp, wc)
    eng.close()
    return r


@pytest.mark.parametrize("mode", [2, 1])
def test_chains_across_edges_and_empty_segments(mode):
    """Mode 2 filters all of it; mode 1 (100 segments of padding: the chains' 3 tokens per merge are below nseg / 32)
    switches on after the first host batch."""
    ids, offs = F.chains(pad_segments=100 if mode == 1 else 0)
    r = _run(ids, offs, CHAIN_MERGES, int(ids.max()) + 1, mode, opt_batch=16, facts=CHAIN_FACTS)
    if mode == 1:
        assert r.facts["switch_on"] == 1 and r.switch_at == 16


def test_large_ids():
    """Ids from 70,000 (above 2^16) and first_idx above 2^21: no batching (batch_fits is false), one delta vector of
    2V + 1 entries.  (On the emulator, which applies that vector thread by thread, only the first chain and a half.)"""
    ids, offs = F.chains(base=70000)
    first_idx = (1 << 21) + 1000
    _run(ids, offs, 800 if SMALL else CHAIN_MERGES, first_idx, 2,
         facts=("pair_only_across_edges", "listed_segment_of_1") if SMALL else CHAIN_FACTS)


def test_table_growth_on_a_filtered_merge():
    """A table that overflows in the middle of the chains: the merge whose update overflowed was performed and is counted
    (k_sig_rebuild_cand gated its statistics on the overflow flag before)."""
    ids, offs = F.chains(pad_segments=4)
    fi = int(ids.max()) + 1
    free = F.State(ids, offs)
    k = len(stats(free.ids, free.start)[1])
    F.train(free, CHAIN_MERGES, fi, mode=2)                  # in a table that never grows: slots at the start and the end
    end = free.used[1]
    # the first overflow lands between the two, and one doubling is enough for the rest
    log2 = next(L for L in range(10, 30) if int(0.6 * (1 << L)) > k + 64)
    assert int(0.6 * (1 << log2)) < end and int(0.6 * (2 << log2)) > end + 64, (k, end, log2)
    r = _run(ids, offs, CHAIN_MERGES, fi, 2, table_log2=log2, facts=("overflow_while_filtering",))
    assert (r.candidates_without_overflowed, r.segments_without_overflowed) != (r.candidates, r.segments)


def _repack_corpus():
    """64 segments of 3-token chunks (x y w) and three of filler with two copies of (p, q): after (x,y) and (z,w) the
    stream fills a third of its segments, maybe_repack packs it between host batches, and (p, q) merges on the packed
    layout."""
    s = F.Stream(5000)
    while len(s.ids) < 64 * F.SEG_TOKENS:
        s.put(10, True)
        s.put(11)
        s.put(12)
    for _ in range(2):
        s.filler(300)
        s.put(20)
        s.put(21)
    s.filler(700)
    return s.stream()


def test_repack_between_filtered_merges():
    ids, offs = _repack_corpus()
    _run(ids, offs, 6, int(ids.max()) + 1, 2, opt_batch=1, facts=("repack_while_filtering",))


def test_chained_calls():
    """Three calls continue one run: each call's counters are its own merges'; the layout, the table and its occupancy
    carry over."""
    ids, offs = F.chains()
    fi = int(ids.max()) + 1
    wp, wc, wd = oracle.c_train(ids, offs, CHAIN_MERGES, first_idx=fi)
    st = F.State(ids, offs)
    eng = _engine(2)
    eng.load_ids(ids, offs)
    at = 0
    for size in (300, 700, CHAIN_MERGES - 1000):
        r = F.train(st, size, fi + at, mode=2, opt_batch=64)
        _check_call(eng, st, r, eng.train(size, first_idx=fi + at), wp[at: at + size], wc[at: at + size])
        at += size
    eng.close()


def test_replay_then_filtered_training(taylorswift):
    """bpe_replay(k) on a byte stream, then train() with the filter on from the first merge."""
    data = np.frombuffer(taylorswift.encode()[: 60000 if SMALL else 120000], dtype=np.uint8)
    offs = np.arange(0, len(data), 997, dtype=np.uint64)
    k, more = 40, (60 if SMALL else 150)
    ids = data.astype(np.int32)
    wp, wc, wd = oracle.c_train(ids, offs, k + more)
    st = F.State(ids, offs, bytes_only=True)
    F.replay(st, wp[:k], opt_batch=8)
    r = F.train(st, more, 256 + k, mode=2, opt_batch=8)
    eng = _engine(2, opt_batch=8)
    eng.load_stream(data, offs)
    eng.replay(wp[:k])
    _check_call(eng, st, r, eng.train(more, first_idx=256 + k), wp[k:], wc[k:])
    eng.close()
