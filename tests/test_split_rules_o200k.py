"""CPU: the o200k split rule of minbpe_b200/csrc/split_logic.h (spl_chunk_start_o200k and its two scans, evaluated tile by
tile as the kernels do) against `regex.findall` of the o200k (GPT-4o) pattern: the cases the rule is derived from, the
corpora, random strings over an adversarial alphabet, texts longer than a tile, and text boundaries (special tokens and
document gaps, the WITH_B form)."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest
import regex

from minbpe_b200 import O200K_SPLIT_PATTERN
from minbpe_b200.unicode_tables import o200k_table, tables

O200K = regex.compile(O200K_SPLIT_PATTERN)
TILE = 4096   # k_split.cuh SP_TILE

# (text, expected chunks), every one checked against `regex` as well
EXAMPLES = [
    ("HelloWorld", ["Hello", "World"]),
    ("XMLHttpRequest", ["XMLHttp", "Request"]),
    ("中A", ["中", "A"]),
    ("A中B", ["A中", "B"]),
    ("中AB!", ["中", "AB", "!"]),
    ("中Ab", ["中Ab"]),
    ("!\n/\n/\n/x", ["!\n/\n/\n/", "x"]),
    ("x\n/\n/y", ["x", "\n", "/\n/", "y"]),
    ("!́abc", ["!́abc"]),
    ("1́", ["1", "́"]),
    ("áb", ["áb"]),
    ("don'tStop", ["don't", "Stop"]),
    ("x's'll", ["x's", "'ll"]),
    (" 'sfoo", [" '", "sfoo"]),
    ("HTTPServer's", ["HTTPServer's"]),
    ("  \n\n  x", ["  \n\n", " ", " x"]),
]

MORE = [
    "", "a", " ", "\n", "hello world", "it's we'll I'VE you'Re 'tis x'llama", "!!́a", "!́!́a", " !́a",
    "\t!a", "\t́", "!\n/!x", "!\n/́!", "!!́\n", "á\n", "!́'s", "x's's's", "x's中Ab", "x'S中A",
    "中A's", "A中's", "́AB", " ́A", "!中A", "!ABc", "!AB", "a  1", "!\n !x", "x 's", "ǅungla ǅUNGLA aǅb",
    "ʰAʰb", "あいうエオABC", "12345 1 12 1234567", "a1b22c333", "x\r\n/\r\n/ y", "a/\n x", "//\n//", "/ /a", "http://a.b/c\n",
    "a b\u0085c　d", "　　x", "ſ's x'ſ X'S", "ÉCOLEécole", "iPhoneX", "McDonald's", "ABCdef", "aBCDef",
]


@pytest.fixture(scope="session")
def harness(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "split_harness_o200k.cpp")
    so = str(tmp_path_factory.mktemp("o200k") / "libsplitharness_o200k.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-Wall", "-Wextra", "-std=c++17", "-shared", "-o", so, src])
    L = ctypes.CDLL(so)
    L.split_logic_flags_o200k.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64,
                                          ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p]
    L.split_logic_flags_o200k.restype = ctypes.c_int
    cls, contr = tables()
    table = np.ascontiguousarray(cls | (o200k_table() << 5), dtype=np.uint8)   # what bpe_o200k_table uploads
    contr = np.ascontiguousarray(contr, dtype=np.uint8)

    def offsets(data, hits=(), tile=0):
        b = np.frombuffer(data, dtype=np.uint8)
        flags = np.zeros(b.size, dtype=np.uint8)
        h = np.asarray([(p << 8) | n for p, n in hits], dtype=np.uint64)
        if b.size:
            L.split_logic_flags_o200k(b.ctypes.data, b.size, table.ctypes.data, contr.ctypes.data, int(tile),
                                      h.ctypes.data if h.size else None, int(h.size), flags.ctypes.data)
        return np.flatnonzero(flags).tolist()
    return offsets


def regex_offsets(text):
    out, pos = [], 0
    for c in O200K.findall(text):
        out.append(pos)
        pos += len(c.encode("utf-8"))
    return out


def check(harness, text, tiles=(0,)):
    want = regex_offsets(text)
    data = text.encode("utf-8")
    for tile in tiles:
        got = harness(data, tile=tile)
        if got != want:
            cuts = got + [len(data)]
            chunks = [data[a:b].decode("utf-8", "replace") for a, b in zip(cuts, cuts[1:])]
            raise AssertionError((text, tile, chunks, O200K.findall(text)))


def test_pattern_is_tiktoken_o200k():
    assert O200K_SPLIT_PATTERN == "|".join([
        r"""[^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]*[\p{Ll}\p{Lm}\p{Lo}\p{M}]+(?i:'s|'t|'re|'ve|'m|'ll|'d)?""",
        r"""[^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]+[\p{Ll}\p{Lm}\p{Lo}\p{M}]*(?i:'s|'t|'re|'ve|'m|'ll|'d)?""",
        r"""\p{N}{1,3}""",
        r""" ?[^\s\p{L}\p{N}]+[\r\n/]*""",
        r"""\s*[\r\n]+""",
        r"""\s+(?!\S)""",
        r"""\s+""",
    ])


@pytest.mark.parametrize("text,chunks", EXAMPLES)
def test_examples(harness, text, chunks):
    assert O200K.findall(text) == chunks
    check(harness, text, tiles=(0, 1, 2, 3))


def test_more_cases(harness):
    for t in MORE:
        check(harness, t, tiles=(0, 1, 2, 5))


def test_corpora(harness, taylorswift):
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, "golden", "llama_text.txt"), encoding="utf-8") as f:
        llama = f.read()
    from minbpe_b200.synth import generate
    synth = generate(1337, 1 << 20).tobytes().decode("utf-8")
    for text in (taylorswift, llama, synth):
        check(harness, text, tiles=(0, TILE, 1000))


ALPHABET = (list("aAbBsStTdDmMlLvVeErR") + ["ǅ", "ʰ", "中", "あ", "́", "ः", "⃝", "/", "\r", "\n", "'", "ſ",
            "’", "0", "7", "½", "٣", " ", "\t", " ", "\u0085", "　", "!", ".", "-", "_"]
            + ["'s", "'ll", "'VE", "'Re", "\n/", "/\n", "  ", "\r\n", "AB", "ab"])


def test_random_adversarial(harness):
    rnd = random.Random(20261016)
    for _ in range(100_000):
        n = rnd.randint(1, 16)
        check(harness, "".join(rnd.choice(ALPHABET) for _ in range(n)), tiles=(0, rnd.randint(1, 8)))


def test_random_code_points(harness):
    rnd = random.Random(7)
    pools = [range(0x20, 0x7f), range(0xa0, 0x250), range(0x300, 0x370), range(0x370, 0x530), range(0x900, 0x980),
             range(0x1e00, 0x2070), range(0x3000, 0x3100), range(0x1f600, 0x1f650), range(0x10400, 0x10450),
             [0x9, 0xa, 0xd, 0x20, 0x27, 0x2f, 0x85, 0x1680, 0x2028, 0x2029, 0x202f, 0x205f]]
    for _ in range(5000):
        n = rnd.randint(1, 30)
        check(harness, "".join(chr(rnd.choice(rnd.choice(pools))) for _ in range(n)), tiles=(0, 3))


def test_longer_than_a_tile(harness):
    cases = [
        "x " + "中" * 3000 + "AB! next",          # case split 9 KB after the run started, across tiles
        "x " + "中" * 3000 + "ABc",
        "a" * 5000 + "B" * 5000 + "́" + "C" * 4000 + " z",
        "!" + "\n/" * 5000 + "x y",                # the tail of an O match across tiles
        "x" + "\n/" * 5000 + "y",
        "z" + "́" * 6000 + "Ab" + " '" * 3000 + "s",
        "1" * 10001 + "a",
        "!!" + "́" * 5000 + "A",
    ]
    for t in cases:
        check(harness, t, tiles=(0, TILE, 4099))


def expected_docs(docs):
    out, base = [], 0
    for d in docs:
        out += [base + o for o in regex_offsets(d)]
        base += len(d.encode("utf-8"))
    return out


def test_document_gaps(harness):
    """Documents back to back with one boundary byte between them (k_split_classify<true>): every document split on its
    own, as if alone."""
    rnd = random.Random(5)
    for _ in range(3000):
        docs = ["".join(rnd.choice(ALPHABET) for _ in range(rnd.randint(1, 10))) for _ in range(rnd.randint(2, 5))]
        joined, hits, pos = b"", [], 0
        for j, d in enumerate(docs):
            if j:
                hits.append((len(joined), 1))
                joined += b"\x00"
            joined += d.encode("utf-8")
        got = harness(joined, hits=hits, tile=rnd.choice((0, 2, 7)))
        gaps = [p for p, _ in hits]
        # take the gap bytes out as k_flag_scatter<true> does
        got = [o - sum(1 for g in gaps if g < o) for o in got if o not in gaps]
        assert got == expected_docs(docs), docs


def test_special_boundaries(harness):
    """Special-token occurrences are text boundaries: every one a chunk, the text on either side split on its own.  Here
    inside a CamelCase word, after "/\\n", at the edges and inside a contraction."""
    rnd = random.Random(9)
    special = "<|sp|>"
    texts = ["Hello" + special + "World", "ab" + special + "Cd", "!/\n" + special + "/\nx", special + "AB中" + special,
             "x'" + special + "s", "don" + special + "'t", "中中" + special + "AB", "!!" + special + "́a"]
    for _ in range(2000):
        parts = ["".join(rnd.choice(ALPHABET) for _ in range(rnd.randint(0, 8))) for _ in range(rnd.randint(1, 4))]
        texts.append(special.join(parts))
    for t in texts:
        parts = t.split(special)
        want, hits, pos = [], [], 0
        for j, p in enumerate(parts):
            if j:
                hits.append((pos, len(special)))
                want.append(pos)
                pos += len(special)
            want += [pos + o for o in regex_offsets(p)]
            pos += len(p.encode("utf-8"))
        got = harness(t.encode("utf-8"), hits=hits, tile=rnd.choice((0, 3)))
        assert got == want, t
