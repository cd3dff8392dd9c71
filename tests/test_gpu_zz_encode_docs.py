"""GPU: many documents encoded in one device call — bpe_encode_docs (documents in pieces, every one split on its own, special
tokens found inside a document only, the memo encode of every piece, the documents' first ids from k_enc_write<true>) and
RegexTokenizer.encode_batch / encode_ordinary_batch.  Ids must be bit-exact against oracle.c_encode on each document's own
`regex` chunks, or against the per-document class call where special tokens are involved."""
import os
import random

import numpy as np
import pytest
import regex

import oracle

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller texts, fewer merges

GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
GPT2 = regex.compile(r"""'(?:[sdmt]|ll|ve|re)| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+""")
PATTERNS = {0: GPT4, 1: GPT2}
# empty and whitespace-only documents, trailing spaces and \r, a leading 's, digit runs cut across two documents
EDGES = ["", " ", "   ", "\n", "word  ", "tail\r", "\r\n", "'s start", "'S", "12", "345 and 67", "89", "x", "", "  y  ", "!!", "?"]
SPECIALS = {"<|endoftext|>": 100257, "<|ab|>": 100258, "<|a": 100259, " <sp> ": 100260, "|>": 100261}


def letter_space_cuts(text, rng, mean):
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


def ref_doc(doc, pat, merges, perm=None, special=None):
    """encode(doc) of the reference (regex.py:111-164) with oracle.c_encode as encode_ordinary of every part"""
    out = []
    parts = regex.split("(" + "|".join(regex.escape(k) for k in special) + ")", doc) if special else [doc]
    for part in parts:
        if special and part in special:
            out.append(special[part])
        elif part:
            d, o = oracle.split_to_stream(part, pat)
            out.extend(oracle.c_encode(d, o, merges, perm).tolist())
    return out


def encode_docs(eng, docs, merges, perm=None, specials=None):
    """-> the ids of every document through Engine.encode_docs, plus the raw offsets"""
    data = [d.encode("utf-8") for d in docs]
    offs = np.zeros(len(data), dtype=np.uint64)
    if len(data) > 1:
        offs[1:] = np.cumsum([len(b) for b in data[:-1]])
    ids, o = eng.encode_docs(b"".join(data), offs, merges, perm, specials)
    assert o.size == len(docs) + 1 and o[0] == 0 and o[-1] == ids.size and np.all(np.diff(o.astype(np.int64)) >= 0)
    return [ids[o[j]: o[j + 1]].tolist() for j in range(len(docs))], o


def _engine(pattern=0):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_SPLIT_PATTERN, pattern)
    return eng


@pytest.fixture(scope="module")
def trained(taylorswift):
    from minbpe_b200 import RegexTokenizer
    tok = RegexTokenizer()
    tok.train(taylorswift, 256 + (150 if SMALL else 1000))
    return np.array(list(tok.merges.keys()), dtype=np.int32)


def corpora(taylorswift):
    from minbpe_b200.synth import generate
    synth = generate(1337, (96 << 10) if SMALL else (2 << 20)).tobytes().decode("utf-8")
    return {"taylorswift": taylorswift[: 60000 if SMALL else None], "synth": synth}


@pytest.mark.parametrize("how", ["letter_space", "arbitrary"])
@pytest.mark.parametrize("pattern", [0, 1])
@pytest.mark.parametrize("name", ["taylorswift", "synth"])
def test_documents_equal_the_oracle(name, pattern, how, taylorswift, trained):
    text = corpora(taylorswift)[name]
    rng = random.Random(f"{name}/{pattern}/{how}")
    docs = cut(text, (letter_space_cuts if how == "letter_space" else arbitrary_cuts)(text, rng, 1500), rng, empties=0.05)
    docs = EDGES + docs[: len(docs) // 2] + EDGES + docs[len(docs) // 2:] + EDGES
    eng = _engine(pattern)
    got, o = encode_docs(eng, docs, trained)
    for j, d in enumerate(docs):
        assert got[j] == ref_doc(d, PATTERNS[pattern], trained), (j, d[:80])
    st = eng.encode_stats()
    assert st["pieces"] == 1 and st["fallback_pieces"] == 0
    eng.close()


@pytest.mark.parametrize("pattern", [0, 1])
def test_documents_over_many_pieces(pattern, taylorswift, trained):
    """BPE_OPT_SPLIT_PIECE = 4096: short documents share pieces, one document longer than a piece is cut at letter+space
    points; with and without specials."""
    from minbpe_b200 import engine as E
    rng = random.Random(7 + pattern)
    head = taylorswift[:20000 if SMALL else 60000]
    long_doc = taylorswift[60000:60000 + (9000 if SMALL else 30000)]
    docs = cut(head, arbitrary_cuts(head, rng, 300), rng, 0.05) + [long_doc] + EDGES + ["<|endoftext|>" + long_doc[:5000] + "<|ab|>"]
    spec = [(k.encode(), v) for k, v in SPECIALS.items()]
    eng = _engine(pattern)
    eng.set_option(E.OPT_SPLIT_PIECE, 4096)
    try:
        plain, _ = encode_docs(eng, docs, trained)
        pieces = eng.encode_stats()["pieces"]
        with_sp, _ = encode_docs(eng, docs, trained, specials=spec)
    finally:
        eng.set_option(E.OPT_SPLIT_PIECE, 0)          # process-wide
    assert pieces > 10
    for j, d in enumerate(docs):
        assert plain[j] == ref_doc(d, PATTERNS[pattern], trained), j
        assert with_sp[j] == ref_doc(d, PATTERNS[pattern], trained, special=SPECIALS), j
    eng.close()


def test_tiny_memo_and_the_general_path(taylorswift, trained):
    """A 64-slot memo (BPE_OPT_ENC_MEMO_LOG2) and a document with one chunk of 12,000 letters: pieces of several documents
    take the general path one document at a time; the ids and the documents' boundaries stay the same."""
    from minbpe_b200 import engine as E
    rng = random.Random(21)
    text = taylorswift[: 30000 if SMALL else 180000]
    docs = cut(text, arbitrary_cuts(text, rng, 700)) + EDGES
    docs.insert(len(docs) // 2, "abc " + "lyiltumdya" * 1200 + " def")
    docs.insert(5, "x <|endoftext|>y<|a")
    want = [ref_doc(d, GPT4, trained) for d in docs]
    want_sp = [ref_doc(d, GPT4, trained, special=SPECIALS) for d in docs]
    spec = [(k.encode(), v) for k, v in SPECIALS.items()]
    eng = _engine(0)
    assert encode_docs(eng, docs, trained)[0] == want
    assert eng.encode_stats()["fallback_pieces"] == 1
    assert encode_docs(eng, docs, trained, specials=spec)[0] == want_sp
    assert eng.encode_stats()["fallback_pieces"] == 1
    try:
        eng.set_option(E.OPT_ENC_MEMO_LOG2, 6)
        big = docs * (1 if SMALL else 3)
        assert encode_docs(eng, big, trained)[0] == want * (1 if SMALL else 3)
        st = eng.encode_stats()
        assert st["fallback_pieces"] >= 1 and st["direct_chunks"] > 1000
        eng.set_option(E.OPT_SPLIT_PIECE, 1 << 14)
        assert encode_docs(eng, big, trained, specials=spec)[0] == want_sp * (1 if SMALL else 3)
        assert eng.encode_stats()["pieces"] >= 3
    finally:
        eng.set_option(E.OPT_ENC_MEMO_LOG2, 0)
        eng.set_option(E.OPT_SPLIT_PIECE, 0)
    eng.close()


def test_specials_inside_documents_only(trained):
    """Occurrences at document starts and ends, overlapping specials, and specials that exist only across a boundary:
    "<|endo" + "ftext|>" matches nothing, "...<|a" + "b|>" leaves the shorter special "<|a" in the first document."""
    body = "some words 123 and more 's text " * (20 if SMALL else 200)
    docs = ["<|endoftext|>" + body, body + "<|endoftext|>", body + "<|endo", "ftext|>" + body, "x<|a", "b|>y", "<|ab|>",
            "<|a", "b|> <sp> " + body, "|>|>", "<|ab|><|a<|ab", "|>", "", body + " <sp", "> <sp> ", "<|endoftext|>"]
    eng = _engine(0)
    res = {}
    for mode in ("all", "set", "none"):
        special = SPECIALS if mode == "all" else ({"<|a": 100259, "|>": 100261} if mode == "set" else {})
        spec = [(k.encode(), v) for k, v in special.items()] or None
        res[mode], _ = encode_docs(eng, docs, trained, specials=spec)
        for j, d in enumerate(docs):
            assert res[mode][j] == ref_doc(d, GPT4, trained, special=special), (mode, j, d[:40])
    got = res["all"]
    assert got[0][0] == got[1][-1] == 100257 and 100257 not in got[2] + got[3]
    assert got[4][-1] == 100259 and got[5][1] == 100261 and got[6] == [100258]
    eng.close()


def test_class_methods_equal_the_loop(taylorswift, trained, monkeypatch):
    """encode_batch / encode_ordinary_batch against [encode(t, allowed_special) for t in texts] of the same class, for every
    allowed_special mode, several device batches, a batch under 64 KiB, a non-device pattern; errors included."""
    from minbpe_b200 import RegexTokenizer
    tok = RegexTokenizer()
    tok.train(taylorswift[:40000], 256 + 100)
    tok.register_special_tokens(dict(SPECIALS))
    rng = random.Random(3)
    text = taylorswift[: 70000 if SMALL else 185000]
    docs = cut(text, arbitrary_cuts(text, rng, 900)) + EDGES
    sp_docs = list(docs)
    for i in range(0, len(sp_docs), 7):
        sp_docs[i] = rng.choice(list(SPECIALS)) + sp_docs[i] + rng.choice(list(SPECIALS))
    assert sum(len(d.encode()) for d in docs) >= tok.DEVICE_SPLIT_MIN_BYTES
    monkeypatch.setattr(RegexTokenizer, "ITERATOR_BATCH_BYTES", 1 << 14)
    assert tok.encode_ordinary_batch(docs) == [tok.encode_ordinary(d) for d in docs]
    assert tok.encode_ordinary_batch(iter(docs)) == [tok.encode_ordinary(d) for d in docs]
    assert tok.encode_batch(docs) == [tok.encode(d) for d in docs]
    for mode in ("all", "none", {"<|a", "|>"}, {"absent"}, set()):
        assert tok.encode_batch(sp_docs, allowed_special=mode) == [tok.encode(d, allowed_special=mode) for d in sp_docs], mode
    assert tok.encode_batch(sp_docs[:40], allowed_special="all") == [tok.encode(d, allowed_special="all") for d in sp_docs[:40]]
    assert tok.encode_batch([]) == [] and tok.encode_ordinary_batch([]) == []
    assert tok.encode_batch(["", "a", ""]) == [[], tok.encode("a"), []]
    # errors, before any device work
    eng = tok.engine
    tok.encode_ordinary_batch(docs)
    pieces_before = eng.encode_stats()["pieces"]
    with pytest.raises(AssertionError):
        tok.encode_batch(sp_docs)                                    # none_raise
    with pytest.raises(ValueError):
        tok.encode_batch(docs, allowed_special="some")
    with pytest.raises(TypeError):
        tok.encode_batch(docs + [b"bytes"])
    with pytest.raises(TypeError):
        tok.encode_ordinary_batch([1] + docs)
    with pytest.raises(UnicodeEncodeError):
        tok.encode_ordinary_batch(docs + ["lone \ud800 surrogate"])
    assert eng.encode_stats()["pieces"] == pieces_before
    # no merges / another pattern: the per-document loop
    assert RegexTokenizer().encode_ordinary_batch(docs[:50]) == [list(d.encode()) for d in docs[:50]]
    other = RegexTokenizer(r"\p{L}+|\s+|[^\s\p{L}]+")
    other.merges = tok.merges
    assert other.encode_ordinary_batch(docs) == [other.encode_ordinary(d) for d in docs]


def test_gpt4_tokenizer_byte_perm(taylorswift):
    from minbpe_b200 import GPT4Tokenizer
    from test_gpt4_host import synthetic_ranks
    ranks, merges, perm = synthetic_ranks(taylorswift[:30000], 120)
    if len(ranks) != 256 + len(merges):
        pytest.skip("degenerate synthetic table")
    tok = GPT4Tokenizer(mergeable_ranks=ranks)
    rng = random.Random(8)
    text = taylorswift[: 70000 if SMALL else 185000]
    docs = cut(text, arbitrary_cuts(text, rng, 1000)) + EDGES
    docs[3] = "<|endoftext|>" + docs[3] + "<|fim_prefix|>"
    m, p8 = np.asarray(merges, dtype=np.int32), perm.astype(np.uint8)
    got = tok.encode_batch(docs, allowed_special="all")
    assert got == [ref_doc(d, GPT4, m, p8, tok.special_tokens) for d in docs]
    assert got == [tok.encode(d, allowed_special="all") for d in docs]
    assert tok.encode_ordinary_batch(docs) == [ref_doc(d, GPT4, m, p8) for d in docs]


def test_no_merges_gives_the_bytes(taylorswift):
    from test_gpt4_host import synthetic_ranks
    _, _, perm = synthetic_ranks(taylorswift[:2000], 1)
    docs = ["héllo wörld", "", "12 34", "日本 語"]
    eng = _engine(0)
    none = np.zeros((0, 2), dtype=np.int32)
    assert encode_docs(eng, docs, none)[0] == [list(d.encode()) for d in docs]
    p8 = perm.astype(np.uint8)
    assert encode_docs(eng, docs, none, p8)[0] == [[int(p8[b]) for b in d.encode()] for d in docs]
    eng.close()


def test_capacity_and_arguments(trained):
    import ctypes
    eng = _engine(0)
    L, h = eng._lib, eng._h
    data = np.frombuffer(b"some words here and there", dtype=np.uint8)
    m = trained
    out = np.empty(data.size, dtype=np.int32)
    oo = np.empty(8, dtype=np.uint64)
    n = ctypes.c_uint64()

    def call(offs, n_docs, cap=data.size, out_offs=oo, nbytes=data.size):
        o = np.asarray(offs, dtype=np.uint64)
        return L.bpe_encode_docs(h, data.ctypes.data, nbytes, o.ctypes.data if o.size else None, n_docs, m.ctypes.data,
                                 m.shape[0], None, None, None, None, 0, out.ctypes.data, cap,
                                 out_offs.ctypes.data if out_offs is not None else None, ctypes.byref(n))
    eng.encode_docs(b"x", [0], m)                                   # the tables are loaded
    assert call([0, 10], 2) == 0 and oo[0] == 0 and oo[2] == n.value
    assert call([0, 10], 2, cap=2) == -4                             # BPE_ERR_CAPACITY
    for bad, nd in (([1, 10], 2), ([0, 10, 5], 3), ([0, data.size + 1], 2), ([0], 0)):
        assert call(bad, nd) == -2, bad                              # BPE_ERR_ARG
    assert call([0, 10], 2, out_offs=None) == -2
    assert call([0, 5, 5], 3) == 0 and oo[1] == oo[2]                # an empty document
    assert L.bpe_encode_docs(h, None, 0, None, 0, None, 0, None, None, None, None, 0, None, 0, oo.ctypes.data, ctypes.byref(n)) == 0
    assert n.value == 0 and oo[0] == 0
    eng.close()


def test_stream_and_session_unchanged(taylorswift, trained):
    """A stream loaded for training and an open counting session are left as they were by a call, and a second call with
    the same merges finds every chunk in the memo."""
    text = taylorswift[:30000]
    rng = random.Random(5)
    docs = cut(text, arbitrary_cuts(text, rng, 500))
    eng = _engine(0)
    d, o = oracle.split_to_stream(text[:20000], GPT4)
    eng.load_stream(d, o)
    before = eng.read_stream()
    first, _ = encode_docs(eng, docs, trained)
    assert np.array_equal(eng.read_stream(), before)
    # a session with an encode between two add_docs calls counts what one without it counts
    half = [x.encode() for x in docs[:40]], [x.encode() for x in docs[40:]]

    def offs(part):
        a = np.zeros(len(part), dtype=np.uint64)
        a[1:] = np.cumsum([len(b) for b in part[:-1]])
        return a
    eng.dedup_begin()
    eng.dedup_add_docs(b"".join(half[0]), offs(half[0]))
    again, _ = encode_docs(eng, docs, trained)
    assert again == first
    st = eng.encode_stats()
    assert st["new_chunks"] == 0 and st["pieces"] == 1                # warm memo
    eng.dedup_add_docs(b"".join(half[1]), offs(half[1]))
    got = eng.dedup_finish()
    b1, o1 = eng.chunk_entries()
    eng.dedup_begin()
    for part in half:
        eng.dedup_add_docs(b"".join(part), offs(part))
    assert eng.dedup_finish() == got
    b2, o2 = eng.chunk_entries()
    assert np.array_equal(b1, b2) and np.array_equal(o1, o2)
    eng.close()
