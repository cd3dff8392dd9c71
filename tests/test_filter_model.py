"""CPU: the host model of the filtered training loop (tests/filter_model.py) against the oracle, its candidate rule on hand-made
layouts, and the layouts the corpora of tests/test_gpu_zz_filter_exact.py were built to produce."""
import numpy as np

import filter_model as F
import oracle
from batch_model import SEG_TOKENS


def _state(segments, marks=()):
    """A State whose segments hold the given id lists (empty lists allowed); marks: stream positions of chunk starts."""
    ids = np.asarray([x for s in segments for x in s], dtype=np.int32)
    st = F.State(ids, np.asarray([0] + list(marks), dtype=np.uint64))
    st.seg = np.asarray([t for t, s in enumerate(segments) for _ in s], dtype=np.int64)
    st.nseg = len(segments)
    return st


def test_sig_bit_is_32_bit_arithmetic():
    x = np.asarray([0, 1, 0xfffff, 70000, (1 << 31) - 2], dtype=np.int64)
    y = np.asarray([0, 2, 3, 1 << 22, 5], dtype=np.int64)
    for xi, yi, got in zip(x.tolist(), y.tolist(), F.sig_bit(x, y).tolist()):
        h = ((xi * 0x9e3779b1) ^ (yi * 0x85ebca77)) & 0xffffffff
        h ^= h >> 15
        h = (h * 0x2c1b3c6d) & 0xffffffff
        h ^= h >> 12
        assert got == h >> (32 - F.SIG_LOG2) and 0 <= got < 1 << F.SIG_LOG2


def test_candidate_rule_on_hand_made_layouts():
    a, b = 7, 9
    # a ends segment 0, two empty segments, b starts segment 3: both ends listed, nothing else (filler ids 100+)
    st = _state([[100, 101, a], [], [], [b, 102], [103, 104]])
    got = set(np.flatnonzero(F.candidates(st, a, b)).tolist()) - set(_sig_only(st, a, b))
    assert got == {0, 3}
    # the same with b chunk-marked: no pair, neither edge branch lists it
    st = _state([[100, 101, a], [], [], [b, 102], [103, 104]], marks=[3])
    assert not set(np.flatnonzero(F.candidates(st, a, b)).tolist()) - set(_sig_only(st, a, b))
    # segments of one token: a alone, b alone
    st = _state([[100], [a], [b], [101]])
    assert {1, 2} <= set(np.flatnonzero(F.candidates(st, a, b)).tolist())
    # a pair inside a segment: listed by its own bit
    st = _state([[100, a, b, 101], [102]])
    assert F.candidates(st, a, b)[0]


def _sig_only(st, a, b):
    """Segments holding an inside pair whose bit collides with (a,b)'s (filler pairs may)."""
    out = []
    for t in range(st.nseg):
        s = st.ids[st.seg == t]
        if len(s) > 1 and (F.sig_bit(s[:-1], s[1:]) == F.sig_bit(a, b)).any():
            out.append(t)
    return out


def test_chains_model_equals_the_oracle_and_builds_its_layouts():
    ids, offs = F.chains()
    fi = int(ids.max()) + 1
    K = 512 + 1024 + 5
    st = F.State(ids, offs)
    r = F.train(st, K, fi, mode=2, opt_batch=16)
    wp, wc, wd, fin = oracle.c_train(ids, offs, K, first_idx=fi, want_final=True)
    assert r.n_done == wd == K and np.array_equal(r.merges, wp) and np.array_equal(r.counts, wc)
    assert np.array_equal(st.ids, fin)
    for f in ("pair_only_across_edges", "occurrence_across_empty_segment", "occurrence_across_two_empty_segments",
              "listed_segment_of_1", "listed_segment_of_2", "empty_last_segment", "marked_b_after_edge",
              "listed_by_colliding_bit", "aa_merge_while_filtering"):
        assert r.facts[f] > 0, (f, dict(r.facts))
    # every listed merge: the list holds every segment the merge changes (the model asserts it as it goes) and
    # filter_candidates is the sum of the list lengths
    assert r.candidates == sum(len(lst) for _, _, lst in r.lists) and r.facts["filtered_merges"] == len(r.lists)
    assert r.candidates < r.segments


def test_chain_offsets():
    """Chains start at the last offset of a segment; the stream ends with a full segment that the last chain drains."""
    ids, offs = F.chains()
    for c0 in (1000, 1600):
        pos = np.flatnonzero(ids == c0)
        assert len(pos) == 3 and (pos % SEG_TOKENS == SEG_TOKENS - 1).all()
    assert len(ids) % SEG_TOKENS == 0


def test_mode_1_switches_on_after_the_first_batch():
    ids, offs = F.chains(pad_segments=100)
    st = F.State(ids, offs)
    r = F.train(st, 40, int(ids.max()) + 1, mode=1, opt_batch=16)
    assert r.facts["switch_on"] == 1 and r.switch_at == 16 and r.facts["filtered_merges"] == 40 - 16


def test_table_growth_changes_the_counters_of_the_old_gate():
    """The overflowed merge is counted; leaving it out (k_sig_rebuild_cand's former gate) gives other sums."""
    ids, offs = F.chains(pad_segments=4)
    st = F.State(ids, offs)
    r = F.train(st, 512 + 1024 + 5, int(ids.max()) + 1, mode=2, table_log2=14)
    assert r.facts["overflow_while_filtering"] == 1
    assert r.candidates_without_overflowed < r.candidates and r.segments_without_overflowed < r.segments
