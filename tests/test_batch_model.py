"""CPU: the host model of bpe_train's pass partition (tests/batch_model.py) and the corpora built for it.  The model's
merges and counts must be the oracle's, a cap of one merge gives one merge per pass, and every generator must still
produce the layouts tests/test_gpu_zz_batch.py relies on."""
import numpy as np
import pytest

import oracle
from batch_model import BATCH_MAX, partition, planted, short_chunks, weighted_entries, with_filler_pairs


def _check_oracle(ids, offs, k, first_idx=256, weights=None):
    m = partition(ids, offs, k, first_idx, weights=weights)
    wp, wc, wd = oracle.c_train(ids, offs, k, first_idx=first_idx, weights=weights)
    assert np.array_equal(m.merges, wp) and np.array_equal(m.counts, wc) and len(m.merges) == wd
    assert sum(m.sizes) == wd and all(1 <= s <= BATCH_MAX for s in m.sizes)
    return m


def test_batch_max_is_the_library_constant():
    assert 2 <= BATCH_MAX <= 64


def test_planted_layouts():
    ids, offs = planted()
    fi = int(ids.max()) + 1
    m = _check_oracle(ids, offs, 40, fi)
    assert m.sizes[:3] == [BATCH_MAX] * 3
    for f in ("full_batch", "adj_fwd", "adj_rev", "adj_self", "adj_seg_edge", "adj_chunk_mark", "member_across_seg_edge"):
        assert m.facts[f] > 0, (f, dict(m.facts))
    # the planted pairs come first, in order, with counts strictly decreasing and well apart
    assert m.merges[:8].tolist() == [[1000 + 2 * i, 1001 + 2 * i] for i in range(8)]
    assert (np.diff(m.counts[:9]) < -4).all()


def test_one_merge_per_pass_with_cap_one():
    ids, offs = planted(offsets=range(510, 512))
    fi = int(ids.max()) + 1
    one = partition(ids, offs, 20, fi, cap=1)
    many = partition(ids, offs, 20, fi)
    assert one.sizes == [1] * 20 and np.array_equal(one.merges, many.merges) and np.array_equal(one.final, many.final)
    assert one.tokens_in > many.tokens_in
    # a call of k merges: the passes of the long call that start before merge k, the last one cut short
    for k in (1, 2, 3, 4, 5, 7, 9, 13):
        assert partition(ids, offs, k, fi).tokens_in == many.tokens_in_upto(k)


def test_byte_corpora():
    import regex
    from minbpe_b200.synth import generate
    text = generate(1337, 64 << 10).tobytes().decode("utf-8")
    GPT4 = regex.compile(r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
    data, offs = oracle.split_to_stream(text, GPT4)
    m = _check_oracle(np.asarray(data, dtype=np.int32), offs, 120)
    assert m.facts["full_batch"] > 0


def test_taylorswift_repacks(taylorswift):
    data, _ = oracle.split_to_stream(taylorswift)
    m = _check_oracle(np.asarray(data, dtype=np.int32), None, 320)
    assert m.facts["repack_possible"] > 0 and m.facts["full_batch"] > 0


def test_short_chunks():
    ids, offs = short_chunks(n_tokens=8000)
    m = _check_oracle(ids, offs, 120, 512)
    assert max(m.sizes) > 1 and m.facts["adj_chunk_mark"] > 0
    assert len(m.final) < 1.25 * len(offs)     # most chunks are one token


@pytest.mark.parametrize("big", [False, True])
def test_weighted_model(big):
    ids, offs = planted(offsets=range(510, 513), byte_ids=True)
    w = weighted_entries(ids, offs, seed=1, big=big)
    m = _check_oracle(ids, offs, 60, weights=w)
    assert max(m.sizes) == BATCH_MAX
    for f in ("adj_fwd", "adj_rev", "adj_self", "adj_chunk_mark"):
        assert m.facts[f] > 0, (f, dict(m.facts))
    if big:
        assert int(m.counts.max()) >= 1 << 33


@pytest.mark.parametrize("member", [1, 2, 3])
def test_first_overflow_placement(member):
    """The padding of test_table_growth_inside_a_batch puts the first overflow of a 2^14-slot table on `member`."""
    base, offs0 = planted(offsets=())
    limit = int(0.6 * (1 << 14))
    fi0 = int(base.max()) + 1
    pre = partition(base, offs0, member, fi0)
    extra = limit - pre.init_pairs - sum(pre.passes[0].new_pairs)
    ids, offs = with_filler_pairs(base, offs0, extra)
    m = partition(ids, offs, 12, int(ids.max()) + 1)
    assert m.init_pairs == pre.init_pairs + extra
    assert m.first_overflow(14) == (0, member)
    assert partition(ids, offs, member, int(ids.max()) + 1).used_after(1) == limit
