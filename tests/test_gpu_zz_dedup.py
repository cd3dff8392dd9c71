"""GPU: training on the distinct chunks of a text with their counts — device chunk counting (bpe_load_text_gpt4_dedup,
k_dedup.cuh), bpe_load_chunks_weighted, the weighted merge loop (k_weighted.cuh), RegexTokenizer.train(dedup=True) and
train_from_file(dedup=True).  A weighted stream must give the merges, counts and tie-breaks of
the whole text (the oracle's weighted loop, itself pinned to the plain loop by tests/test_oracle.py), whether every
distinct chunk is one entry or chunks are split over several entries; across batched merges, re-packing, pairs (a,a),
table growth and a second bpe_train call."""
import contextlib
import hashlib
import io
import os

import numpy as np
import pytest
import regex

import oracle

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller corpus, fewer merges

GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
GPT2 = regex.compile(r"""'(?:[sdmt]|ll|ve|re)| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+""")
RUNS = " zz zz zzzz aaaa aaaa" + " " * 70 + "b" * 60 + " zz"   # pairs (a,a), and chunks longer than 48 bytes


def corpora(taylorswift):
    from minbpe_b200.synth import generate
    synth = generate(1337, (256 << 10) if SMALL else (2 << 20)).tobytes().decode("utf-8")
    return {"taylorswift": taylorswift + RUNS, "synth": synth + RUNS}


def _engine():
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_BATCH, 64)                 # more batch boundaries: re-packing happens there
    return eng


def _check_entries(eng, ub, uo, uw):
    ids = eng.read_stream()
    assert np.array_equal(ids, np.frombuffer(ub, dtype=np.uint8).astype(np.int32))
    assert np.array_equal(eng.chunk_weights(), np.asarray(uw, dtype=np.uint64))


@pytest.mark.parametrize("name", ["taylorswift", "synth"])
def test_weighted_training_equals_the_oracle(name, taylorswift):
    text = corpora(taylorswift)[name]
    merges = 400 if SMALL else 1500
    data, offs = oracle.split_to_stream(text, GPT4)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges + 100, weights=uw)
    eng = _engine()
    eng.load_chunks_weighted(ub, uo, uw)
    _check_entries(eng, ub, uo, uw)
    p, c, d = eng.train(merges)
    assert d == merges and np.array_equal(p, wp[:merges]) and np.array_equal(c, wc[:merges])
    assert any(a == b for a, b in p.tolist())       # the (a,a) path ran
    p2, c2, d2 = eng.train(100, first_idx=256 + merges)    # continuing the run: the table is kept
    assert d2 == 100 and np.array_equal(p2, wp[merges:]) and np.array_equal(c2, wc[merges:])
    assert np.array_equal(eng.chunk_weights(), np.asarray(uw, dtype=np.uint64))
    table = eng.debug_table()
    # the table equals the one of the whole text trained to the same point
    eng.load_stream(data, offs)
    p3, c3, d3 = eng.train(merges + 100)
    assert d3 == merges + 100 and np.array_equal(p3, wp) and np.array_equal(c3, wc)
    assert eng.debug_table() == table
    eng.close()


def _split_entries(data, offs, rng, p_split):
    """Entries in which a distinct chunk may be split over several entries: each occurrence after the first becomes an
    entry of its own with probability p_split, otherwise it is counted by a random earlier entry with the same bytes."""
    raw = bytes(data)
    ends = list(offs[1:].tolist()) + [len(raw)]
    entries, weights, where = [], [], {}
    for s, e in zip(offs.tolist(), ends):
        ch = raw[s:e]
        mine = where.get(ch)
        if mine is None or rng.random() < p_split:
            where.setdefault(ch, []).append(len(entries))
            entries.append(ch)
            weights.append(1)
        else:
            weights[mine[int(rng.integers(len(mine)))]] += 1
    lens = np.fromiter(map(len, entries), dtype=np.int64, count=len(entries))
    eo = np.zeros(len(entries), dtype=np.uint64)
    eo[1:] = np.cumsum(lens[:-1])
    return b"".join(entries), eo, np.asarray(weights, dtype=np.uint64)


@pytest.mark.parametrize("p_split", [0.05, 0.5])
def test_chunks_split_over_several_entries(p_split, taylorswift):
    """The rule allows several entries per distinct chunk (a full table, chunks too long for it): merges and counts stay
    the oracle's."""
    text = taylorswift + RUNS
    merges = 300 if SMALL else 1000
    data, offs = oracle.split_to_stream(text, GPT4)
    eb, eo, ew = _split_entries(data, offs, np.random.default_rng(7), p_split)
    assert int(ew.sum()) == len(offs) and len(eo) < len(offs)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    assert len(eo) > len(uo)
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges, weights=uw)
    eng = _engine()
    eng.load_chunks_weighted(eb, eo, ew)
    _check_entries(eng, eb, eo, ew)
    p, c, d = eng.train(merges)
    assert d == wd == merges and np.array_equal(p, wp) and np.array_equal(c, wc)
    eng.close()


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def test_regex_tokenizer_dedup_taylorswift(golden_train, taylorswift, tmp_path):
    from minbpe_b200 import RegexTokenizer
    g = golden_train["taylorswift_regex_512"]
    out = {}
    for dedup in (False, True):
        tok = RegexTokenizer()
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            tok.train(taylorswift, 512, verbose=True, dedup=dedup)
        tok.save(str(tmp_path / f"d{int(dedup)}"))
        out[dedup] = (tok.merges, buf.getvalue())
    assert [list(p) for p in out[True][0]] == g["merges"]
    assert out[True] == out[False]
    assert RegexTokenizer().engine.dedup_stats()["entries"] > 0       # taylorswift (>= 64 KiB) took the device loader
    assert _sha(str(tmp_path / "d1.model")) == g["model_sha256"] and _sha(str(tmp_path / "d1.vocab")) == g["vocab_sha256"]
    # resume: 384 -> save -> load -> 512, all with dedup
    a = RegexTokenizer()
    a.train(taylorswift, 384, dedup=True)
    a.save(str(tmp_path / "part"))
    b = RegexTokenizer()
    b.load(str(tmp_path / "part.model"))
    b.train(taylorswift, 512, resume=True, dedup=True)
    assert [list(p) for p in b.merges] == g["merges"]


def test_regex_tokenizer_dedup_small_cases_and_patterns(golden_cases, taylorswift):
    from minbpe_b200 import RegexTokenizer
    from minbpe_b200.tokenizer import GPT2_SPLIT_PATTERN
    for c in golden_cases:
        if c["tokenizer"] != "regex":
            continue
        text, V = c["text"], c["vocab_size"]
        tok = RegexTokenizer()
        if "raises" in c:
            with pytest.raises(ValueError):
                tok.train(text, V, dedup=True)
            assert tok.merges == {}
            continue
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            tok.train(text, V, verbose=True, dedup=True)
        assert [list(p) for p in tok.merges] == c["merges"], text
        assert [int(x) for x in regex.findall(r"had (\d+) occurrences", buf.getvalue())] == c["counts"], text
    # the GPT-2 pattern (device split of a long text) and a custom pattern (host split)
    for pattern in (GPT2_SPLIT_PATTERN, r"\p{L}+|\s+|[^\s\p{L}]+"):
        merges = {}
        for dedup in (False, True):
            tok = RegexTokenizer(pattern)
            tok.train(taylorswift + RUNS, 256 + 200, dedup=dedup)
            merges[dedup] = tok.merges
        assert merges[True] == merges[False], pattern


def test_weighted_stream_refusals():
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    data = b"ab ab ab cd"
    offs = np.array([0, 2, 5, 8], dtype=np.uint64)
    with pytest.raises(E.EngineError):
        eng.load_chunks_weighted(data, offs, np.array([1, 0, 1, 1], dtype=np.uint64))   # zero weight
    with pytest.raises(E.EngineError):
        eng.load_chunks_weighted(data, None, np.zeros(0, dtype=np.uint64))              # no chunk offsets
    with pytest.raises(E.EngineError):
        eng.load_chunks_weighted(data, np.array([0, 5, 2], dtype=np.uint64), np.ones(3, dtype=np.uint64))   # unsorted
    eng.load_chunks_weighted(b"ab cd", np.array([0, 2], dtype=np.uint64), np.array([3, 1], dtype=np.uint64))
    with pytest.raises(E.EngineError):
        eng.get_stats()
    with pytest.raises(E.EngineError):
        eng.merge(97, 98, 256)
    dummy = np.zeros(65536, dtype=np.uint64)       # host memory: a refusal must come before any use of the pointer
    with pytest.raises(E.EngineError):
        eng.step_begin(dummy.ctypes.data)
    with pytest.raises(E.EngineError):
        eng.step_table(dummy.ctypes.data, 4)
    with pytest.raises(E.EngineError):
        eng.step_select(dummy.ctypes.data, 0)
    with pytest.raises(E.EngineError):
        eng.step_merge(dummy.ctypes.data, dummy.ctypes.data)
    with pytest.raises(E.EngineError):
        eng.step_apply(dummy.ctypes.data)
    with pytest.raises(E.EngineError):
        eng.step_fused(1)
    with pytest.raises(E.EngineError):
        eng.xchg_create(1, 0, 512)
    for opt in (E.OPT_RESCAN, E.OPT_SEG_FILTER):
        eng.set_option(opt, 1)
        with pytest.raises(E.EngineError):
            eng.train(2)
        eng.set_option(opt, 0)
    p, c, d = eng.train(2)                          # (a,b) x3 + (' ',c) x1 + (c,d) x1 ...
    assert d == 2 and p[0].tolist() == [97, 98] and int(c[0]) == 3
    # any other load makes the stream unweighted again
    eng.load_stream(data, offs)
    with pytest.raises(E.EngineError):
        eng.chunk_weights()
    assert len(eng.get_stats()[0]) > 0
    eng.close()


@pytest.mark.parametrize("pattern", [0, 1])
@pytest.mark.parametrize("name", ["taylorswift", "synth"])
def test_device_loader_equals_the_oracle(name, pattern, taylorswift):
    """bpe_load_text_gpt4_dedup: the entries are exactly the oracle's distinct chunks of the host `regex` split, with
    their counts, and training on them gives the oracle's merges and counts."""
    from minbpe_b200 import engine as E
    text = corpora(taylorswift)[name]
    data, offs = oracle.split_to_stream(text, GPT4 if pattern == 0 else GPT2)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    eng = _engine()
    eng.set_option(E.OPT_SPLIT_PATTERN, pattern)
    nc, ne = eng.load_text_gpt4_dedup(data)
    assert nc == len(offs) and ne == len(uo)
    _check_entries(eng, ub, uo, uw)
    st = eng.dedup_stats()
    assert st["text_chunks"] == len(offs) and st["entries"] == len(uo) and st["stream_bytes"] == len(ub)
    assert st["table_entries"] + st["passthrough_entries"] == st["entries"] and st["pieces"] == 1
    merges = 300 if SMALL else 1000
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges, weights=uw)
    p, c, d = eng.train(merges)
    assert d == wd == merges and np.array_equal(p, wp) and np.array_equal(c, wc)
    eng.close()


def test_device_loader_degraded_cases(taylorswift):
    """A chunk table that fills up, chunks longer than its 48-byte key and a text split into many pieces: entries may
    differ from the oracle's, but the weights still count every chunk of the text once and the merges are the oracle's."""
    from minbpe_b200 import engine as E
    text = taylorswift + RUNS + " " * 200 + "x" * 300 + RUNS
    data, offs = oracle.split_to_stream(text, GPT4)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    merges = 300 if SMALL else 800
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges, weights=uw)
    for log2, piece in ((5, 0), (0, 4096), (8, 8192)):
        eng = _engine()
        if log2:
            eng.set_option(E.OPT_DEDUP_LOG2, log2)
        eng.set_option(E.OPT_SPLIT_PIECE, piece)
        try:
            nc, ne = eng.load_text_gpt4_dedup(data)
        finally:
            eng.set_option(E.OPT_SPLIT_PIECE, 0)      # process-wide
        st = eng.dedup_stats()
        w = eng.chunk_weights()
        assert nc == len(offs) and int(w.sum()) == len(offs) and ne == len(w) >= len(uo)
        assert st["passthrough_entries"] > 0          # the long chunks, and with a small table the ones without room
        if log2:
            assert st["slots_used"] <= st["slots"] == 1 << log2 and ne > len(uo)
        if piece:
            assert st["pieces"] > 10
        p, c, d = eng.train(merges)
        assert d == wd == merges and np.array_equal(p, wp) and np.array_equal(c, wc), (log2, piece)
        eng.close()
    eng = E.Engine(0)
    with pytest.raises(E.EngineError):
        eng.set_option(E.OPT_DEDUP_LOG2, 3)
    eng.load_text_gpt4_dedup(b"")
    assert eng.stream_len() == 0 and len(eng.chunk_weights()) == 0
    with pytest.raises(E.EngineError):
        eng.get_stats()
    eng.close()


def test_train_from_file_dedup(taylorswift, tmp_path, monkeypatch):
    from minbpe_b200 import RegexTokenizer
    path = str(tmp_path / "corpus.txt")
    text = taylorswift + RUNS
    with open(path, "w", encoding="utf-8") as f:
        f.write(text)
    a = RegexTokenizer()
    a.train(text, 256 + 300)
    b = RegexTokenizer()
    b.train_from_file(path, 256 + 300, dedup=True)
    assert b.merges == a.merges and b.vocab == a.vocab
    assert b.engine.dedup_stats()["text_chunks"] > 0
    import torch.distributed as dist
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(ValueError):
        RegexTokenizer().train_from_file(path, 256 + 300, dedup=True)


@pytest.mark.skipif(SMALL, reason="1 GiB corpus")
def test_cfg3_dedup_all_merges_vs_oracle():
    """cfg3 (1 GiB synthetic, seed 1337, vocab 32,768) through the device loader: all 32,512 merges and counts equal
    to the oracle's weighted loop over the host `regex` split."""
    from minbpe_b200 import engine as E
    from minbpe_b200.presplit import chunk_offsets
    from minbpe_b200.synth import generate
    from minbpe_b200.tokenizer import GPT4_SPLIT_PATTERN
    raw = generate(1337, 1 << 30)
    eng = E.Engine(0)
    nc, ne = eng.load_text_gpt4_dedup(raw)
    p, c, d = eng.train(32512)
    offs = chunk_offsets(GPT4_SPLIT_PATTERN, raw, workers=min(16, len(os.sched_getaffinity(0))))
    ub, uo, uw = oracle.c_dedup_chunks(raw, offs)
    assert nc == offs.size and ne == len(uo)
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, 32512, weights=uw)
    assert d == wd == 32512
    bad = np.flatnonzero((p != wp).any(axis=1))
    assert bad.size == 0, f"first differing merge {int(bad[0])}"
    assert np.array_equal(c, wc)
    eng.close()
