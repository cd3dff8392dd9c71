"""CPU: the texts of tests/test_gpu_zz_beyond_32bit.py (tests/beyond32.py) at a small boundary B.  Their oracle, built from
the blocks alone, must equal `regex` + oracle.c_dedup_chunks on the real text, and every straddling case must
discriminate: a first position taken mod B, or read as signed, puts the entries in another order, and training on that
order gives other merges.  Without this a passing run past 2^32 would prove nothing."""
import numpy as np
import pytest
import regex

import beyond32 as T
import oracle
from batch_model import stats, table_dict

B = 1 << 20
K = 24
PATTERNS = ("GPT4_SPLIT_PATTERN", "GPT2_SPLIT_PATTERN", "O200K_SPLIT_PATTERN")


def _pattern(name):
    import minbpe_b200.tokenizer as M
    return getattr(M, name)


@pytest.fixture(scope="module")
def text():
    return T.Text(B, 4096)


def _real(t, pattern, specials=None):
    """The reference's chunks of the whole text (every part between specials split on its own) and their distinct entries."""
    s = t.array().tobytes().decode("utf-8")
    chunks = [c.encode("utf-8") for p in T.parts(s, specials) for c in regex.findall(pattern, p)]
    lens = np.fromiter(map(len, chunks), dtype=np.int64, count=len(chunks))
    offs = np.zeros(len(chunks), dtype=np.uint64)
    np.cumsum(lens[:-1], out=offs[1:].view(np.int64))
    data = np.frombuffer(b"".join(chunks), dtype=np.uint8)
    return data, offs, oracle.c_dedup_chunks(data, offs)


def test_layout(text):
    """Every block starts with a space and ends with an ASCII letter; the tail blocks sit where the construction says."""
    arr = text.array()
    assert arr.size == text.nbytes > B
    for raw, (_, r), s in zip(text.raw, text.blocks, text.starts):
        assert raw[:1] == b" " and chr(raw[-1]).isascii() and chr(raw[-1]).isalpha()
        assert arr[s: s + len(raw)].tobytes() == raw and arr[s + len(raw) * (r - 1): s + len(raw) * r].tobytes() == raw
    assert arr[text.x_first: text.x_first + 2].tobytes() == b"XY" and arr[text.u_first: text.u_first + 2].tobytes() == b"UV"
    assert b"XY" not in arr[: text.x_first].tobytes() and b"UV" not in arr[: text.u_first].tobytes()


def test_written_file_equals_the_array(text, tmp_path):
    path = tmp_path / "t.txt"
    text.write(str(path), slab=1 << 16)
    assert path.read_bytes() == text.array().tobytes()
    docs = list(text.documents())
    assert "".join(docs).encode("utf-8") == text.array().tobytes()


@pytest.mark.parametrize("name", PATTERNS)
@pytest.mark.parametrize("specials", [None, {T.EOT: 1000}], ids=["plain", "specials"])
def test_construction_equals_regex(text, name, specials):
    """Entries, weights and first positions from the blocks equal the oracle's distinct chunks of `regex` on the text;
    training on them equals training on every chunk (the plain loop)."""
    pattern = _pattern(name)
    data, offs, (ub, uo, uw) = _real(text, pattern, specials)
    d, o, w, first = T.entries(text, pattern, specials)
    assert np.array_equal(d, ub) and np.array_equal(o, uo) and np.array_equal(w, uw)
    raw = text.array().tobytes()
    ends = np.append(o[1:], np.uint64(d.size)).astype(np.int64)
    for i in range(len(o)):
        f = int(first[i])
        assert raw[f: f + ends[i] - int(o[i])] == d[int(o[i]): ends[i]].tobytes()
    assert np.all(np.diff(first.astype(np.int64)) > 0)
    wp, wc, _ = T.train(d, o, w, K)
    pp, pc, _ = oracle.c_train(data.astype(np.int32), offs, K)
    assert np.array_equal(wp, pp) and np.array_equal(wc, pc)


def test_ids_by_construction(text):
    """The per-block ids, repeated, equal the oracle's encode of the whole text, with and without specials."""
    pattern = _pattern("GPT4_SPLIT_PATTERN")
    d, o, w, _ = T.entries(text, pattern)
    merges, _, _ = T.train(d, o, w, K)
    s = text.array().tobytes().decode("utf-8")
    for specials in (None, {T.EOT: 1000}):
        want = np.concatenate([np.tile(T.encode_block(b, pattern, merges, specials), r) for b, r in text.blocks])
        got = []
        for i, p in enumerate(regex.split("(" + regex.escape(T.EOT) + ")", s) if specials else [s]):
            if i % 2:
                got.append(np.array([1000], dtype=np.int32))
                continue
            dd, oo = oracle.split_to_stream(p, regex.compile(pattern))
            got.append(oracle.c_encode(dd, oo, merges))
        assert np.array_equal(np.concatenate(got), want)


def test_stream_and_table_after_the_merges(text):
    """merged_entries: the weighted stream length and pair table after K merges equal those of the plain loop's final
    stream."""
    pattern = _pattern("GPT4_SPLIT_PATTERN")
    data, offs, _ = _real(text, pattern)
    d, o, w, _ = T.entries(text, pattern)
    pairs, _, _ = T.train(d, o, w, K)
    fin, start = T.merged_entries(d, o, w, pairs)
    _, _, _, full = oracle.c_train(data.astype(np.int32), offs, K, want_final=True)
    assert int(w[np.cumsum(start) - 1].sum()) == full.size
    lens = T.token_lengths(pairs)[full]
    fstart = np.isin(np.cumsum(lens) - lens, offs.astype(np.int64))
    assert table_dict(*stats(fin, start, w)) == table_dict(*stats(full, fstart))


@pytest.mark.parametrize("specials", [None, {T.EOT: 1000}], ids=["plain", "specials"])
def test_truncated_positions_give_other_merges(text, specials):
    """(X,Y) first occurs below B, (U,V) past it; every truncation of the positions puts (U,V) first, and the weighted
    loop on the entries in the truncated order picks (U,V) at the tie where the true order picks (X,Y)."""
    pattern = _pattern("GPT4_SPLIT_PATTERN")
    d, o, w, first = T.entries(text, pattern, specials)
    pairs, counts, _ = T.train(d, o, w, K)
    X, U = [ord("X"), ord("Y")], [ord("U"), ord("V")]
    assert pairs[:3].tolist() == [[90, 90], X, U] and counts[1] == counts[2]
    assert text.x_first < B <= text.u_first
    names = list(T.truncations(B))
    assert names == [f"mod 2^{B.bit_length() - 1}", f"signed at 2^{B.bit_length() - 1}"]
    for name, key in T.truncations(B).items():
        kx, ku = key(np.array([text.x_first, text.u_first], dtype=np.uint64))
        assert ku < kx, name                                        # the truncated order picks (U,V)
        order = np.argsort(key(first), kind="stable")
        assert not np.array_equal(order, np.arange(len(order)))
        tp, tc, _ = T.train(*T.reorder(d, o, w, order), K)
        assert tp[:3].tolist() == [[90, 90], U, X], name
        assert not np.array_equal(tp, pairs), name
    # the true order is text order: sorting by the full 64-bit position changes nothing
    assert np.array_equal(np.argsort(first, kind="stable"), np.arange(len(first)))


def test_truncations_at_the_real_boundaries():
    """At B = 2^31 and 2^32 the construction holds and every truncation of the first positions picks (U,V); the
    oracle's first merges are (Z,Z), (X,Y), (U,V)."""
    pattern = _pattern("GPT4_SPLIT_PATTERN")
    for b in (1 << 31, 1 << 32):
        t = T.Text(b, 65536)
        assert t.nbytes > b and t.nbytes - b < 300 << 20
        d, o, w, first = T.entries(t, pattern)
        pairs, counts, _ = T.train(d, o, w, 4)
        assert pairs[:3].tolist() == [[90, 90], [88, 89], [85, 86]] and counts[1] == counts[2]
        assert set(T.truncations(b)) == ({"mod 2^31", "signed at 2^31"} if b == 1 << 31 else {"mod 2^32"})
        for name, key in T.truncations(b).items():
            kx, ku = key(np.array([t.x_first, t.u_first], dtype=np.uint64))
            assert ku < kx, name
            tp, _, _ = T.train(*T.reorder(d, o, w, np.argsort(key(first), kind="stable")), 4)
            assert tp[1].tolist() == [85, 86], name
