"""CPU: the rule by which bpe_train applies several merges in one pass (k_select_batch, DESIGN.md "Batched merges").

With the pairs of get_stats() sorted by count, p1 = the arg-max, the next k merges are exactly p1 .. pk when
c1 > c2 > ... > ck > c(k+1), every pj has two different ids and the 2k ids are all distinct.  At every step of the
oracle's restatement of the reference loop, the batch the rule predicts from the table (oracle.c_get_stats) must be the
oracle's next k merges, with their counts."""
import numpy as np
import pytest
import regex

import oracle

GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
CAP = 8   # the device carries at most BATCH_MAX (4) merges per pass; a correct batch of 8 has correct prefixes


def predict(pairs, counts, cap):
    """The batch the rule allows at this step: [(pair, count)], empty when the arg-max is tied."""
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


def merge(ids, start, pair, z):
    """base.py:25-41 over a stream whose chunk starts are marked in `start` (no pair spans two chunks)."""
    a, b = pair
    hit = (ids[:-1] == a) & (ids[1:] == b) & ~start[1:]
    pos = np.flatnonzero(hit)
    if a == b:   # runs: greedy from the left
        keep, last = [], -2
        for q in pos.tolist():
            if q != last + 1:
                keep.append(q)
                last = q
        pos = np.asarray(keep, dtype=np.int64)
    ids = ids.copy()
    ids[pos] = z
    drop = np.ones(len(ids), dtype=bool)
    drop[pos + 1] = False
    return ids[drop], start[drop]


def check(data, offs, merges):
    ids0 = np.frombuffer(data, dtype=np.uint8).astype(np.int32)
    want_pairs, want_counts, done, final = oracle.c_train(ids0, offs, merges, want_final=True)
    assert done == merges
    ids = ids0
    start = np.zeros(len(ids), dtype=bool)
    start[np.asarray(offs if offs is not None else [0], dtype=np.int64)] = True
    batched = 0
    for i in range(merges):
        pairs, counts = oracle.c_get_stats(ids, np.flatnonzero(start).astype(np.uint64))
        batch = predict(pairs, counts, min(CAP, merges - i))
        for j, (pair, count) in enumerate(batch):
            assert pair == tuple(want_pairs[i + j]) and count == want_counts[i + j], (i, j, batch)
        batched += len(batch) > 1
        ids, start = merge(ids, start, want_pairs[i], 256 + i)
    assert np.array_equal(ids, final)   # the stepping above is the oracle's loop
    return batched


@pytest.mark.parametrize("kind", ["basic", "regex"])
def test_rule_on_taylorswift(taylorswift, kind):
    data, offs = oracle.split_to_stream(taylorswift, GPT4 if kind == "regex" else None)
    assert check(bytes(data), offs, 256) >= 20


def test_rule_on_synthetic_corpus():
    from minbpe_b200.synth import generate
    text = generate(1337, 256 * 1024).tobytes().decode("utf-8")
    data, offs = oracle.split_to_stream(text, GPT4)
    assert check(bytes(data), offs, 256) >= 20


def test_rule_refuses_ties_and_shared_ids():
    p = np.array([[1, 2], [3, 4], [5, 6], [7, 8]])
    assert [x for x, _ in predict(p, np.array([9, 7, 5, 3]), 8)] == [(1, 2), (3, 4), (5, 6), (7, 8)]
    assert predict(p, np.array([9, 9, 5, 3]), 8) == []                            # the arg-max is tied
    assert [x for x, _ in predict(p, np.array([9, 7, 7, 3]), 8)] == [(1, 2)]       # c2 == c3: p2 is not certain
    q = np.array([[1, 2], [2, 4], [5, 6]])
    assert [x for x, _ in predict(q, np.array([9, 7, 5]), 8)] == [(1, 2)]          # p2 shares id 2 with p1
    r = np.array([[1, 2], [3, 3], [5, 6]])
    assert [x for x, _ in predict(r, np.array([9, 7, 5]), 8)] == [(1, 2)]          # a pair (a, a)
