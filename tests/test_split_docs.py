"""CPU: document boundaries of the counting session (bpe_dedup_add_docs, k_split.cuh).  Several documents are split in one
call of the rule code with one boundary byte of class SC_B between consecutive documents (the WITH_B rule of
split_logic.h), and the chunk starts are mapped back to gap-free positions.  That must equal `regex.findall` run on every
document on its own, for both patterns, any tiling of the scans and any value of the boundary byte.  Also the host path
of train_from_iterator for other patterns: one count across documents in first-occurrence order."""
import random

import numpy as np
import regex

import oracle

GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
GPT2 = regex.compile(r"""'(?:[sdmt]|ll|ve|re)| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+""")
ALPHABET = list("ab'sSdDmMtTlLvVeErR 12\t\n\r!.,' 　é日ſ½\x00") + ["  ", "\n\n", "'ll", "'ve", " '", "K", "\U0001f600", "'re", "'LL"]
CASES = [["", "ab", ""], ["   ", " \t ", "\n"], ["a  ", "  b"], ["x\r", "\ny"], ["'s", "'S'"], ["123", "4567 89"], ["12", "34"],
         ["ab ", "'ll"], ["\r\n", "\r\n"], ["a\x00", "\x00b"], ["", ""], ["日本 ", " 語"], ["! ", "!"], ["a", "b", "c"]]


def expected(docs, pat):
    offs, pos = [], 0
    for d in docs:
        for ch in pat.findall(d):
            offs.append(pos)
            pos += len(ch.encode("utf-8"))
    return np.asarray(offs, dtype=np.uint64)


def device_model(docs, pattern, tile, gap, cls, contr):
    """What bpe_dedup_add_docs does to one piece: empty documents dropped, the rest joined with one gap byte each and the
    gaps given class SC_B (k_split_classify<true>: one-byte boundaries), the chunk starts taken back to gap-free positions
    with a chunk start at every document start (k_flag_reduce<true> / k_flag_scatter<true>)."""
    parts = [d.encode("utf-8") for d in docs if d]
    if not parts:
        return np.zeros(0, dtype=np.uint64)
    starts = np.cumsum([0] + [len(p) for p in parts[:-1]])
    joined = gap.join(parts)
    hits = [(int(s) + j - 1, 1) for j, s in enumerate(starts) if j]
    if pattern == 0:
        got = oracle.split_logic_offsets_special(joined, cls, contr, hits, tile)
    else:
        got = oracle.split_logic_offsets_gpt2(joined, cls, contr, hits, tile)
    sflag = np.zeros(len(joined), dtype=bool)
    sflag[got.astype(np.int64)] = True
    m = sum(len(p) for p in parts)
    i = np.arange(m)
    d = np.searchsorted(starts, i, side="right") - 1
    flag = sflag[i + d]
    flag[starts] = True
    return np.flatnonzero(flag).astype(np.uint64)


def test_document_boundaries_equal_per_document_findall():
    from minbpe_b200.unicode_tables import tables
    cls, contr = tables()
    rnd = random.Random(4242)
    gaps = (b"\x00", b" ", b"'", b"a")
    n = 0
    for pattern, pat in ((0, GPT4), (1, GPT2)):
        for docs in CASES:
            for gap in gaps:
                for tile in (0, 1, 3):
                    got = device_model(docs, pattern, tile, gap, cls, contr)
                    assert np.array_equal(got, expected(docs, pat)), (docs, pattern, gap, tile)
        for _ in range(5000):
            docs = []
            for _ in range(rnd.randint(1, 6)):
                r = rnd.random()
                if r < 0.1:
                    docs.append("")
                elif r < 0.2:
                    docs.append("".join(rnd.choice(" \t\r\n") for _ in range(rnd.randint(1, 4))))
                else:
                    d = "".join(rnd.choice(ALPHABET) for _ in range(rnd.randint(1, 10)))
                    d = rnd.choice(("", "", "'s", "12", "123 ", "'LL")) + d + rnd.choice(("", "", " ", "  ", "\r", "\r\n"))
                    docs.append(d)
            gap, tile = rnd.choice(gaps), rnd.choice((0, rnd.randint(1, 9)))
            got = device_model(docs, pattern, tile, gap, cls, contr)
            assert np.array_equal(got, expected(docs, pat)), (docs, pattern, gap, tile)
            n += 1
    assert n == 10000


def test_boundaries_change_the_split():
    """The test above is not vacuous: joining the documents would split them differently."""
    docs = ["ab  ", "cd", "12", "34", "x'", "s y\r", "\nz"]
    for pat in (GPT4, GPT2):
        assert not np.array_equal(expected(docs, pat), expected(["".join(docs)], pat))


def test_host_path_for_other_patterns_loader(monkeypatch):
    """A pattern the device does not split: every document split with `regex` on its own, the chunks counted in one host
    Counter in first-occurrence order across documents; the weighted oracle loop on them gives the merges of the plain
    loop on the whole per-document chunk list.  The loader handed to _run_training is run against a stub engine that
    records what it loads."""
    from minbpe_b200 import RegexTokenizer
    pattern = r"\p{L}+|\s+|[^\s\p{L}]+"
    rnd = random.Random(8)
    docs = ["".join(rnd.choice(ALPHABET) for _ in range(rnd.randint(0, 30))) for _ in range(400)]
    got = {}

    class Loaded:     # the engine the loader puts the stream on: records what it received
        def load_chunks_weighted(self, data, offsets, weights):
            got.update(data=data, offsets=offsets, weights=weights)

    def capture(self, load, vocab_size, verbose, resume=False):
        load()
        got.update(resume=resume)
    monkeypatch.setattr(RegexTokenizer, "engine", property(lambda self: Loaded()))
    monkeypatch.setattr(RegexTokenizer, "_run_training", capture)
    RegexTokenizer(pattern).train_from_iterator(iter(docs), 300)
    chunks = [c.encode("utf-8") for d in docs for c in regex.findall(pattern, d)]
    data = np.frombuffer(b"".join(chunks), dtype=np.uint8)
    offs = np.zeros(len(chunks), dtype=np.uint64)
    offs[1:] = np.cumsum([len(c) for c in chunks[:-1]])
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    assert got["data"] == ub.tobytes() and np.array_equal(got["offsets"], uo) and np.array_equal(got["weights"], uw)
    assert got["resume"] is False
    wp, wc, wd = oracle.c_train(np.frombuffer(got["data"], dtype=np.uint8).astype(np.int32), got["offsets"], 44,
                                weights=got["weights"])
    pp, pc, pd = oracle.c_train(data.astype(np.int32), offs, 44)
    assert wd == pd == 44 and np.array_equal(wp, pp) and np.array_equal(wc, pc)


def test_non_str_documents_raise(monkeypatch):
    import pytest

    from minbpe_b200 import RegexTokenizer
    monkeypatch.setattr(RegexTokenizer, "_run_training", lambda *a, **k: None)
    with pytest.raises(TypeError):
        RegexTokenizer(r"\w+").train_from_iterator(["ok", b"bytes"], 300)
    with pytest.raises(UnicodeEncodeError):
        RegexTokenizer(r"\w+|\s+|.").train_from_iterator(["ok", "a\ud800"], 300)
