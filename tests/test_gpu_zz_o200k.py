"""GPU: the o200k (GPT-4o) split pattern on the device — BPE_OPT_SPLIT_PATTERN = 3 selects the o200k scans and rule of the
split kernels — through the C ABI and through RegexTokenizer(O200K_SPLIT_PATTERN): every training and encode path against
`regex.findall` and the oracle."""
import os
import random

import numpy as np
import pytest
import regex

import oracle
from minbpe_b200 import O200K_SPLIT_PATTERN, RegexTokenizer

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: shorter texts, fewer merges

O200K = regex.compile(O200K_SPLIT_PATTERN)
GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")

CASES = ["HelloWorld", "XMLHttpRequest", "中A", "A中B", "中AB!", "中Ab", "!\n/\n/\n/x", "x\n/\n/y", "!́abc", "1́", "áb",
         "don'tStop", "x's'll", " 'sfoo", "HTTPServer's", "  \n\n  x", "!!́a", "!́!́a", " !́a", "\t!a", "!\n/!x", "x's's's",
         "x's中Ab", "́AB", "a  1", "ǅungla ǅUNGLA", "ʰAʰb", "McDonald's iPhoneX", "a", " ", "\n"]
ALPHABET = (list("aAbBsStTdDmMlLvVeErR") + ["ǅ", "ʰ", "中", "あ", "́", "ः", "⃝", "/", "\r", "\n", "'", "ſ", "’", "0", "7",
            "½", " ", "\t", " ", "\u0085", " ", "　", "!", "."] + ["'s", "'ll", "'VE", "\n/", "/\n", "  ", "AB", "ab"])


def synth(n):
    from minbpe_b200.synth import generate
    return generate(1337, 1 << 20).tobytes().decode("utf-8")[:n]


def camel_text(n, seed=3):
    rnd = random.Random(seed)
    words = ["Hello", "World", "XMLHttp", "Request", "中文", "AB", "iPhone", "don't", "HTTPServer's", "x's", "12345", "!!",
             "/\n/", "́", "ǅa", "ʰB", " ", "\n", "  ", "\t", "McDonald's", "a/b", "'ll"]
    out, size = [], 0
    while size < n:
        w = rnd.choice(words)
        out.append(w)
        size += len(w)
    return "".join(out)


@pytest.fixture(scope="module")
def taylorswift(taylorswift):
    return taylorswift[:70000] if SMALL else taylorswift    # still above DEVICE_SPLIT_MIN_BYTES


@pytest.fixture(scope="module")
def eng():
    from minbpe_b200 import engine as E
    e = E.Engine(0)
    e.set_option(E.OPT_SPLIT_PATTERN, 3)
    yield e
    e.close()


def check_split(eng, text):
    data, offs = oracle.split_to_stream(text, O200K)
    got = eng.split_gpt4(data.tobytes())
    assert np.array_equal(got, offs), text[:80]


def test_split_offsets_vs_regex(eng, taylorswift):
    from minbpe_b200 import engine as E
    for t in CASES:
        check_split(eng, t)
    check_split(eng, taylorswift)
    check_split(eng, synth(100000 if SMALL else 1 << 20))
    check_split(eng, camel_text(30000 if SMALL else 300000))
    for t in ("x " + "中" * 3000 + "AB! next", "!" + "\n/" * 5000 + "x y", "a" * 5000 + "B" * 5000 + "́" + "C" * 4000 + " z",
              "!!" + "́" * 5000 + "A", "z" + "́" * 6000 + "Ab" + " '" * 3000 + "s"):
        check_split(eng, t)
    eng.set_option(E.OPT_SPLIT_PIECE, 1 << 15)      # several pieces, cut where a letter is followed by U+0020
    try:
        check_split(eng, taylorswift)
        check_split(eng, camel_text(80000 if SMALL else 200000, seed=8) + " end")
    finally:
        eng.set_option(E.OPT_SPLIT_PIECE, 0)
    with pytest.raises(E.EngineError):
        eng.set_option(E.OPT_SPLIT_PATTERN, 2)
    eng.set_option(E.OPT_SPLIT_PATTERN, 3)


def test_split_random_sizes(eng):
    rnd = random.Random(77)
    for size in (1, 2, 3, 17, 2047, 2048, 2049, 4097) + (() if SMALL else (60000, 300000)):
        check_split(eng, "".join(rnd.choice(ALPHABET) for _ in range(size)))


def test_load_text_train_counts(eng, taylorswift):
    """bpe_load_text_gpt4 under o200k (token words straight from the rule kernel) + bpe_train = the oracle on the regex chunks."""
    data, offs = oracle.split_to_stream(taylorswift, O200K)
    assert eng.load_text_gpt4(data.tobytes(), count_chunks=True) == offs.size
    pairs, counts, done = eng.train(64)
    wp, wc, wn = oracle.c_train(data.astype(np.int32), offs, 64)
    assert done == wn == 64 and np.array_equal(pairs, wp) and np.array_equal(counts, wc)
    eng.load_text_gpt4(data.tobytes())
    pairs2, counts2, _ = eng.train(64)
    assert np.array_equal(pairs2, wp) and np.array_equal(counts2, wc)


def want_merges(texts, k):
    ds, os_, base = [], [], 0
    for t in texts:
        d, o = oracle.split_to_stream(t, O200K)
        ds.append(d)
        os_.append(o + base)
        base += d.size
    data = np.concatenate(ds)
    wp, wc, wn = oracle.c_train(data.astype(np.int32), np.concatenate(os_), k)
    assert wn == k
    return wp.tolist()


def test_train_and_dedup(taylorswift):
    text = taylorswift + camel_text(60000)
    want = want_merges([text], 80)
    for dedup in (False, True):
        tok = RegexTokenizer(O200K_SPLIT_PATTERN)
        tok.train(text, 256 + 80, dedup=dedup)
        assert [list(p) for p in tok.merges] == want, dedup


def test_train_from_iterator(taylorswift):
    text = taylorswift + camel_text(40000, seed=5)
    rnd = random.Random(11)
    cuts = sorted(rnd.sample(range(1, len(text)), 300))
    docs = [text[a:b] for a, b in zip([0] + cuts, cuts + [len(text)])]
    tok = RegexTokenizer(O200K_SPLIT_PATTERN)
    tok.train_from_iterator(iter(docs), 256 + 60)
    assert [list(p) for p in tok.merges] == want_merges(docs, 60)


def test_train_from_file(tmp_path, taylorswift):
    text = taylorswift + camel_text(50000, seed=6)
    path = tmp_path / "corpus.txt"
    path.write_bytes(text.encode("utf-8"))
    a = RegexTokenizer(O200K_SPLIT_PATTERN)
    a.train(text, 256 + 60)
    for dedup in (False, True):
        b = RegexTokenizer(O200K_SPLIT_PATTERN)
        b.train_from_file(str(path), 256 + 60, dedup=dedup)
        assert b.merges == a.merges


SPECIALS = {"<|endoftext|>": 100257, "<|fim|>": 100258}


def trained(taylorswift):
    tok = RegexTokenizer(O200K_SPLIT_PATTERN)
    tok.train(taylorswift, 256 + 120)
    tok.register_special_tokens(SPECIALS)
    return tok


def want_ids(tok, text, specials):
    merges = np.asarray([list(p) for p in tok.merges], dtype=np.int32).reshape(-1, 2)
    pat = "(" + "|".join(regex.escape(k) for k in specials) + ")" if specials else None
    out = []
    for part in (regex.split(pat, text) if pat else [text]):
        if part in specials:
            out.append(specials[part])
        elif part:
            d, o = oracle.split_to_stream(part, O200K)
            out.extend(oracle.c_encode(d, o, merges).tolist())
    return out


def special_text(body):
    # specials inside a CamelCase word, after "/\n", at the edges of the text
    return ("<|endoftext|>" + body[:30000] + "Hello<|fim|>World !/\n<|endoftext|>/\nx" + body[30000:70000]
            + "XML<|endoftext|>Http中<|fim|>AB" + body[70000:] + "<|fim|>")


def test_encode_ordinary_and_special(taylorswift):
    tok = trained(taylorswift)
    body = taylorswift + camel_text(40000, seed=9)
    assert tok.encode_ordinary(body) == want_ids(tok, body, {})
    t = special_text(body)
    assert tok.encode(t, allowed_special="all") == want_ids(tok, t, SPECIALS)
    assert tok.encode(t, allowed_special={"<|fim|>"}) == want_ids(tok, t, {"<|fim|>": SPECIALS["<|fim|>"]})


def test_encode_batch(taylorswift):
    tok = trained(taylorswift)
    body = taylorswift + camel_text(60000, seed=10)
    rnd = random.Random(12)
    cuts = sorted(rnd.sample(range(1, len(body)), 120))
    docs = [body[a:b] for a, b in zip([0] + cuts, cuts + [len(body)])]
    docs[3] = "Hello<|fim|>World!/\n<|endoftext|>x"
    docs[7] = "<|endoftext|>" + docs[7] + "<|fim|>"
    docs.append("")
    for mode in ("all", "none", {"<|fim|>"}):
        assert tok.encode_batch(docs, allowed_special=mode) == [tok.encode(d, allowed_special=mode) for d in docs], mode
    plain = [d for d in docs if "<|" not in d]
    assert tok.encode_ordinary_batch(plain) == [want_ids(tok, d, {}) for d in plain]
    with pytest.raises(AssertionError):                 # as encode(d, "none_raise") on a document with a special
        tok.encode_batch(docs, allowed_special="none_raise")


def test_encode_file(tmp_path, taylorswift):
    tok = trained(taylorswift)
    t = special_text(taylorswift + camel_text(30000, seed=13))
    path = tmp_path / "t.txt"
    path.write_bytes(t.encode("utf-8"))
    assert np.asarray(tok.encode_file(str(path), allowed_special="all")).tolist() == tok.encode(t, allowed_special="all")
    plain = taylorswift + camel_text(30000, seed=14)
    path.write_bytes(plain.encode("utf-8"))
    assert np.asarray(tok.encode_file(str(path))).tolist() == want_ids(tok, plain, {})


def test_gpt4_and_o200k_interleaved(taylorswift):
    """Tokenizers of both patterns on the shared default engine, calls interleaved: each gets its own pattern's result."""
    text = taylorswift + camel_text(30000, seed=15)
    t4, to = RegexTokenizer(), RegexTokenizer(O200K_SPLIT_PATTERN)
    t4.train(text, 256 + 40)
    to.train(text, 256 + 40)
    d4, o4 = oracle.split_to_stream(text, GPT4)
    w4, _, _ = oracle.c_train(d4.astype(np.int32), o4, 40)
    assert [list(p) for p in t4.merges] == w4.tolist()
    assert [list(p) for p in to.merges] == want_merges([text], 40)
    camel = camel_text(80000, seed=16)                   # the two patterns split it differently
    assert O200K.findall(camel) != GPT4.findall(camel)
    dc, oc = oracle.split_to_stream(camel, GPT4)
    for _ in range(2):
        assert t4.encode_ordinary(text) == oracle.c_encode(d4, o4, w4).tolist()
        assert to.encode_ordinary(text) == want_ids(to, text, {})
        assert t4.encode_ordinary(camel) == oracle.c_encode(dc, oc, w4).tolist()
        assert to.encode_ordinary(camel) == want_ids(to, camel, {})
