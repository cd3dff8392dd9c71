"""GPU: training from a stream of documents — the counting session (bpe_dedup_begin / _add_docs / _finish, document
boundaries in k_split_classify<true> / k_flag_reduce<true> / k_flag_scatter<true>, chunk counting in k_dedup.cuh) and RegexTokenizer.train_from_iterator.  Every document is split
on its own: the entries and weights must be the oracle's distinct chunks of the per-document `regex` chunks, in iteration
order, and training on them must give the oracle's merges and counts, whatever the batches, pieces, table size or other
work on the shared engine between two calls."""
import contextlib
import hashlib
import io
import os
import random

import numpy as np
import pytest
import regex

import oracle

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller corpus, fewer merges

GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
GPT2 = regex.compile(r"""'(?:[sdmt]|ll|ve|re)| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+""")
PATTERNS = {0: GPT4, 1: GPT2}
RUNS = " zz zz zzzz aaaa aaaa" + " " * 70 + "b" * 60 + " zz\r\n12345 's 'S"


def corpora(taylorswift):
    from minbpe_b200.synth import generate
    synth = generate(1337, (128 << 10) if SMALL else (2 << 20)).tobytes().decode("utf-8")
    return {"taylorswift": taylorswift + RUNS, "synth": synth + RUNS}


def letter_space_cuts(text, rng, mean):
    """Cut points where an ASCII letter is followed by a space (provable chunk boundaries of both patterns)."""
    pts = [i for i in range(1, len(text)) if text[i] == " " and text[i - 1].isascii() and text[i - 1].isalpha()]
    return sorted(rng.sample(pts, min(len(pts), max(1, len(text) // mean))))


def arbitrary_cuts(text, rng, mean):
    return sorted(set(rng.randrange(1, len(text)) for _ in range(max(1, len(text) // mean))))


def cut(text, points, rng=None, empties=0.0):
    docs, prev = [], 0
    for p in list(points) + [len(text)]:
        docs.append(text[prev:p])
        if rng is not None and rng.random() < empties:
            docs.append("")
        prev = p
    return docs


def doc_chunks(docs, pat):
    """The chunk list of the reference run on every document on its own: (bytes, chunk start offsets)."""
    chunks = [c.encode("utf-8") for d in docs for c in pat.findall(d)]
    lens = np.fromiter(map(len, chunks), dtype=np.int64, count=len(chunks))
    offs = np.zeros(len(chunks), dtype=np.uint64)
    if len(chunks) > 1:
        offs[1:] = np.cumsum(lens[:-1])
    return np.frombuffer(b"".join(chunks), dtype=np.uint8), offs


def _engine(pattern=0):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_SPLIT_PATTERN, pattern)
    return eng


def session(eng, docs, rng=None, max_docs=None):
    """begin, the documents in calls of random size (or all in one call), finish -> (chunks, entries, chunks per call)"""
    eng.dedup_begin()
    per_call, j = [], 0
    while j < len(docs) or not per_call:
        k = len(docs) - j if rng is None else rng.randint(1, max_docs)
        part = [d.encode("utf-8") for d in docs[j: j + k]]
        offs = np.zeros(len(part), dtype=np.uint64)
        if len(part) > 1:
            offs[1:] = np.cumsum([len(b) for b in part[:-1]])
        per_call.append(eng.dedup_add_docs(b"".join(part), offs))
        j += k
    nc, ne = eng.dedup_finish()
    return nc, ne, per_call


def check_entries(eng, docs, pat, nc=None, ne=None):
    data, offs = doc_chunks(docs, pat)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    b, o = eng.chunk_entries()
    assert np.array_equal(b, ub) and np.array_equal(o, uo)
    assert np.array_equal(eng.chunk_weights(), np.asarray(uw, dtype=np.uint64))
    if nc is not None:
        assert nc == len(offs) and ne == len(uo)
    return data, offs, ub, uo, uw


@pytest.mark.parametrize("how", ["letter_space", "arbitrary"])
@pytest.mark.parametrize("pattern", [0, 1])
@pytest.mark.parametrize("name", ["taylorswift", "synth"])
def test_session_equals_the_oracle(name, pattern, how, taylorswift):
    """Documents cut at letter+space points or at arbitrary characters, with empty documents among them, in one call and
    in many calls of random size: entries, weights and chunk counts are the oracle's of the per-document chunks."""
    text = corpora(taylorswift)[name]
    rng = random.Random(f"{name}/{pattern}/{how}")
    cuts = (letter_space_cuts if how == "letter_space" else arbitrary_cuts)(text, rng, 2000)
    docs = cut(text, cuts, rng, empties=0.05)
    eng = _engine(pattern)
    nc, ne, per_call = session(eng, docs)
    check_entries(eng, docs, PATTERNS[pattern], nc, ne)
    nc2, ne2, per_call2 = session(eng, docs, rng, max_docs=7)
    assert len(per_call2) > 10 and sum(per_call2) == nc2 == nc and ne2 == ne
    check_entries(eng, docs, PATTERNS[pattern])
    st = eng.dedup_stats()
    assert st["text_chunks"] == nc and st["entries"] == ne and st["pieces"] >= len(per_call2) - per_call2.count(0)
    if how == "arbitrary":          # the boundaries do change the split
        assert not np.array_equal(doc_chunks(docs, PATTERNS[pattern])[1], doc_chunks([text], PATTERNS[pattern])[1])
    eng.close()


@pytest.mark.parametrize("pattern", [0, 1])
def test_documents_longer_than_a_piece(pattern, taylorswift):
    """BPE_OPT_SPLIT_PIECE = 4096: short documents share pieces, a document longer than a piece is cut at letter+space
    points, and the result is still the oracle's."""
    from minbpe_b200 import engine as E
    text = taylorswift + RUNS
    rng = random.Random(5 + pattern)
    docs = cut(text[:20000], arbitrary_cuts(text[:20000], rng, 300)) + [text[20000:]] + cut(RUNS[:60] * 3, [5, 17, 40])   # chunks <= 48 bytes: all in the table
    assert len(docs[-5].encode("utf-8")) > 4096
    eng = _engine(pattern)
    eng.set_option(E.OPT_SPLIT_PIECE, 4096)
    try:
        nc, ne, _ = session(eng, docs, rng, max_docs=40)
    finally:
        eng.set_option(E.OPT_SPLIT_PIECE, 0)      # process-wide
    check_entries(eng, docs, PATTERNS[pattern], nc, ne)
    assert eng.dedup_stats()["pieces"] > 20
    eng.close()


@pytest.mark.parametrize("piece", [0, 4096])
@pytest.mark.parametrize("pattern", [0, 1])
def test_load_text_equals_a_one_document_session(pattern, piece, taylorswift):
    from minbpe_b200 import engine as E
    text = taylorswift + RUNS
    data = text.encode("utf-8")
    eng = _engine(pattern)
    eng.set_option(E.OPT_SPLIT_PIECE, piece)
    try:
        got = [eng.load_text_gpt4_dedup(data)]
        b1, o1 = eng.chunk_entries()
        w1, st1 = eng.chunk_weights(), eng.dedup_stats()
        got.append(session(eng, [text])[:2])
    finally:
        eng.set_option(E.OPT_SPLIT_PIECE, 0)
    b2, o2 = eng.chunk_entries()
    assert got[0] == got[1]
    assert np.array_equal(b1, b2) and np.array_equal(o1, o2) and np.array_equal(w1, eng.chunk_weights())
    assert st1 == eng.dedup_stats() and (st1["pieces"] > 10) == bool(piece)
    check_entries(eng, [text], PATTERNS[pattern])
    eng.close()


def test_training_equals_the_oracle(taylorswift):
    """Documents whose boundaries change the split: merges and counts are the oracle's weighted loop on the per-document
    chunks (the oracle's weighted loop is pinned to the plain loop by tests/test_oracle.py)."""
    text = corpora(taylorswift)["synth"]
    rng = random.Random(11)
    docs = cut(text, arbitrary_cuts(text, rng, 500))
    merges = 300 if SMALL else 1500
    for pattern in (0, 1):
        eng = _engine(pattern)
        session(eng, docs, rng, max_docs=50)
        data, offs, ub, uo, uw = check_entries(eng, docs, PATTERNS[pattern])
        wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges, weights=uw)
        p, c, d = eng.train(merges)
        assert d == wd == merges and np.array_equal(p, wp) and np.array_equal(c, wc)
        pp, pc, pd = oracle.c_train(data.astype(np.int32), offs, merges)      # the whole chunk list, unweighted
        assert np.array_equal(pp, p) and np.array_equal(pc, c)
        eng.close()


def test_small_table_over_many_batches(taylorswift):
    """A 32-slot table (BPE_OPT_DEDUP_LOG2) over hundreds of add_docs calls: most entries pass through, the weights still
    count every chunk once and the merges are the oracle's."""
    from minbpe_b200 import engine as E
    text = taylorswift + RUNS
    rng = random.Random(3)
    docs = cut(text, arbitrary_cuts(text, rng, 150))
    data, offs = doc_chunks(docs, GPT4)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    merges = 200 if SMALL else 800
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges, weights=uw)
    eng = _engine(0)
    eng.set_option(E.OPT_DEDUP_LOG2, 5)
    nc, ne, per_call = session(eng, docs, rng, max_docs=4)
    assert len(per_call) >= 200
    st, w = eng.dedup_stats(), eng.chunk_weights()
    assert nc == len(offs) == int(w.sum()) and ne == len(w) > len(uo)
    assert st["slots"] == 32 and st["slots_used"] <= 32 and st["passthrough_entries"] > 0
    p, c, d = eng.train(merges)
    assert d == wd == merges and np.array_equal(p, wp) and np.array_equal(c, wc)
    eng.close()


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def _train(tok, how, *args, **kw):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        getattr(tok, how)(*args, verbose=True, **kw)
    return tok.merges, buf.getvalue()


def test_train_from_iterator_golden_and_train(golden_train, taylorswift, tmp_path, monkeypatch):
    from minbpe_b200 import RegexTokenizer
    g = golden_train["taylorswift_regex_512"]
    tok = RegexTokenizer()
    m_it, v_it = _train(tok, "train_from_iterator", iter([taylorswift]), 512)
    assert [list(p) for p in m_it] == g["merges"]
    tok.save(str(tmp_path / "it"))
    assert _sha(str(tmp_path / "it.model")) == g["model_sha256"] and _sha(str(tmp_path / "it.vocab")) == g["vocab_sha256"]
    assert (m_it, v_it) == _train(RegexTokenizer(), "train", taylorswift, 512)
    assert (m_it, v_it) == _train(RegexTokenizer(), "train", taylorswift, 512, dedup=True)
    # letter+space pieces are provable chunk boundaries: the merges of the whole text
    rng = random.Random(1)
    pieces = cut(taylorswift, letter_space_cuts(taylorswift, rng, 700))
    assert len(pieces) > 100
    assert _train(RegexTokenizer(), "train_from_iterator", (p for p in pieces), 512) == (m_it, v_it)
    # the batch size changes nothing
    docs = cut(taylorswift, arbitrary_cuts(taylorswift, rng, 900))
    want = _train(RegexTokenizer(), "train_from_iterator", docs, 512)
    monkeypatch.setattr(RegexTokenizer, "ITERATOR_BATCH_BYTES", 4096)
    small = RegexTokenizer()
    assert _train(small, "train_from_iterator", docs, 512) == want != (m_it, v_it)
    assert small.engine.dedup_stats()["pieces"] > 30
    # resume: 384 -> save -> load -> 512
    a = RegexTokenizer()
    a.train_from_iterator(docs, 384)
    a.save(str(tmp_path / "part"))
    b = RegexTokenizer()
    b.load(str(tmp_path / "part.model"))
    b.train_from_iterator(iter(docs), 512, resume=True)
    assert b.merges == want[0]


def test_train_from_iterator_errors():
    from minbpe_b200 import RegexTokenizer
    tok = RegexTokenizer()
    tok.train_from_iterator(["hello world"] * 3, 258)
    before = dict(tok.merges)
    with pytest.raises(ValueError):
        tok.train_from_iterator(["a", "", "b", " "], 300)          # no pairs at all
    assert tok.merges == before

    def broken():
        yield "some text here " * 100
        raise KeyError("reader failed")
    with pytest.raises(KeyError):
        tok.train_from_iterator(broken(), 300)
    assert tok.merges == before
    with pytest.raises(TypeError):
        tok.train_from_iterator(["ok", b"bytes"], 300)
    with pytest.raises(UnicodeEncodeError):
        tok.train_from_iterator(["ok", "lone \ud800 surrogate"], 300)
    assert tok.merges == before
    tok.train_from_iterator(["hello world"] * 3, 258)                # the engine is usable afterwards
    assert tok.merges == before
    t = RegexTokenizer()
    t.train_from_iterator(iter(()), 256)
    assert t.merges == {}


def test_train_from_iterator_custom_pattern(taylorswift):
    """Any other pattern: every document split with `regex`, counted on the host in first-occurrence order."""
    from minbpe_b200 import RegexTokenizer
    pattern = r"\p{L}+|\s+|[^\s\p{L}]+"
    rng = random.Random(4)
    docs = cut(taylorswift, arbitrary_cuts(taylorswift, rng, 400))
    data, offs = doc_chunks(docs, regex.compile(pattern))
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    merges = 150 if SMALL else 400
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges, weights=uw)
    tok = RegexTokenizer(pattern)
    tok.train_from_iterator(docs, 256 + merges)
    assert [list(p) for p in tok.merges] == wp.tolist()


def test_session_isolation(taylorswift):
    """The user's iterator runs between two add_docs calls: another tokenizer's encode, a train on another text (plain
    and dedup, which load the shared engine) and a change of BPE_OPT_SPLIT_PATTERN leave the result unchanged."""
    from minbpe_b200 import RegexTokenizer, engine as E
    from minbpe_b200.tokenizer import GPT2_SPLIT_PATTERN
    rng = random.Random(9)
    docs = cut(taylorswift, arbitrary_cuts(taylorswift, rng, 3000))
    V = 256 + (100 if SMALL else 300)
    want = RegexTokenizer()
    want.train_from_iterator(docs, V)
    other = RegexTokenizer(GPT2_SPLIT_PATTERN)
    other.train(taylorswift[:70000], 300)
    side = RUNS * (420 if SMALL else 4000)                 # >= 64 KiB: the device paths

    def meddle(i):
        if i % 3 == 0:
            other.encode(side)                                   # >= 64 KiB: GPT-2 split + encode on the device
        elif i % 3 == 1:
            RegexTokenizer().train(side, 260, dedup=bool(i % 2))    # a load and a training run on the shared engine
        else:
            other.engine.set_option(E.OPT_SPLIT_PATTERN, 1)

    def interleaved():
        for i, d in enumerate(docs):
            yield d
            meddle(i)

    tok = RegexTokenizer()
    assert tok.engine is other.engine
    old = RegexTokenizer.ITERATOR_BATCH_BYTES
    RegexTokenizer.ITERATOR_BATCH_BYTES = 4096
    try:
        tok.train_from_iterator(interleaved(), V)
    finally:
        RegexTokenizer.ITERATOR_BATCH_BYTES = old
    assert tok.merges == want.merges
    assert tok.engine.dedup_stats()["pieces"] > 10


def test_session_state_and_arguments(taylorswift):
    from minbpe_b200 import engine as E
    eng = _engine(0)
    L, h = eng._lib, eng._h
    offs = np.zeros(1, dtype=np.uint64)
    data = np.frombuffer(b"some text", dtype=np.uint8)
    assert L.bpe_dedup_add_docs(h, data.ctypes.data, data.size, offs.ctypes.data, 1, None) == -3     # BPE_ERR_STATE
    assert L.bpe_dedup_finish(h, None, None) == -3
    # begin discards an unfinished session
    text = taylorswift[:30000]
    eng.dedup_begin()
    eng.dedup_add_docs(b"unrelated words that must not count", [0])
    nc, ne, _ = session(eng, [text[:10000], text[10000:]])
    check_entries(eng, [text[:10000], text[10000:]], GPT4, nc, ne)
    assert L.bpe_dedup_finish(h, None, None) == -3                                              # finish ended it
    eng.dedup_begin()
    for bad_offs, n_docs, n in (([1], 1, data.size), ([0, 5, 3], 3, data.size), ([0, data.size + 1], 2, data.size),
                                ([0], 0, data.size)):
        o = np.asarray(bad_offs, dtype=np.uint64)
        assert L.bpe_dedup_add_docs(h, data.ctypes.data, n, o.ctypes.data, n_docs, None) == -2      # BPE_ERR_ARG
    assert eng.dedup_add_docs(data, [0, 4, 4, 5]) == 3           # the session survives bad arguments; empty documents
    assert eng.dedup_add_docs(b"", []) == 0
    assert eng.dedup_finish() == (3, 3)
    b, o = eng.chunk_entries()
    assert b.tobytes() == b"some text" and o.tolist() == [0, 4, 5]
    with pytest.raises(E.EngineError):
        eng.get_stats()                                          # a weighted stream
    eng.dedup_begin()
    assert eng.dedup_finish() == (0, 0) and eng.stream_len() == 0
    eng.close()
