"""GPU: training with special tokens (DESIGN.md §18) — a counting session with specials installed
(bpe_dedup_set_specials: spec_find on the session's own set, marks by k_special_meta<false>, k_dd_count<false, true>) and
the special_tokens argument of RegexTokenizer.train / train_from_iterator / train_from_file.  Only the parts between the
occurrences re.split reports are trained on, every part split on its own: the entries and weights must be the oracle's
distinct chunks of the per-part `regex` chunks, training on them must give the oracle's merges, and every entry point must
equal train_from_iterator over those parts followed by register_special_tokens."""
import bisect
import contextlib
import hashlib
import io
import os
import random
import socket
import sys

import numpy as np
import pytest
import regex

import oracle
from conftest import ROOT

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller corpus, fewer merges
MERGES = 40 if SMALL else 200

EOT, IMS = "<|endoftext|>", "<|im_start|>"
EDGE = "\n".join([
    EOT + "Once upon a time" + EOT + EOT + " there was." + EOT,           # at the start, adjacent, at the end
    "x<ab|cd>ef<|e and <|eot|> then <|eo",                                 # overlapping, prefix of another
    "a b<|x 1a b<|x2 q",                                                    # a special holding a letter+space
    "über <|ünïcødé|>☃☃ snow☃☃☃",                                          # multi-byte UTF-8 specials
])
EDGE_SPECIALS = {EOT: 0, "<ab|c": 1, "b|cd>e": 2, "<|e": 3, "<|eot|>": 4, "a b<|x": 5, "<|ünïcødé|>": 6, "☃☃": 7}
PATTERNS = {0: "GPT4_SPLIT_PATTERN", 1: "GPT2_SPLIT_PATTERN", 3: "O200K_SPLIT_PATTERN"}


def _pattern(which):
    import minbpe_b200.tokenizer as T
    return getattr(T, PATTERNS[which])


def parts(doc, specials):
    return regex.split("(" + "|".join(regex.escape(k) for k in specials) + ")", doc)[0::2]


def documents(text, rng, mean):
    """The text cut at letter+space points into documents of log-normal sizes around `mean` characters."""
    pts = [i for i in range(1, len(text)) if text[i] == " " and text[i - 1].isascii() and text[i - 1].isalpha()]
    docs, prev = [], 0
    while True:
        want = prev + max(1, int(rng.lognormvariate(np.log(mean), 0.8)))
        i = bisect.bisect_left(pts, want)
        if i == len(pts):
            docs.append(text[prev:])
            return docs
        docs.append(text[prev:pts[i]])
        prev = pts[i]


def corpus(taylorswift, seed=1):
    """Documents with EOT / IMS separators inside them, plus the edge cases (every one at least 64 KiB in all)."""
    from minbpe_b200.synth import generate
    synth = generate(1337, (96 << 10) if SMALL else (1 << 20)).tobytes().decode("utf-8")
    rng = random.Random(seed)
    docs = documents(taylorswift[: 40000 if SMALL else None] + synth, rng, 3000)
    out = []
    for d in docs:
        sub = documents(d, rng, 400)
        out.append("".join(s + rng.choice([EOT, EOT, IMS, "", EOT + IMS]) for s in sub))
    return out + [EDGE] * 3


def part_chunks(docs, specials, pat):
    """The chunk list of the reference loop on every part of every document: (bytes, chunk start offsets)."""
    chunks = [c.encode("utf-8") for d in docs for p in parts(d, specials) for c in pat.findall(p)]
    lens = np.fromiter(map(len, chunks), dtype=np.int64, count=len(chunks))
    offs = np.zeros(len(chunks), dtype=np.uint64)
    if len(chunks) > 1:
        offs[1:] = np.cumsum(lens[:-1])
    return np.frombuffer(b"".join(chunks), dtype=np.uint8), offs


def _engine(which=0):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_SPLIT_PATTERN, which)
    return eng


def session(eng, docs, specials, rng=None, between=None):
    """begin, specials, the documents in calls of random size (or all in one call), finish -> (chunks, entries, per call)"""
    eng.dedup_begin()
    eng.dedup_set_specials([k.encode("utf-8") for k in specials])
    per_call, j = [], 0
    while j < len(docs) or not per_call:
        k = len(docs) - j if rng is None else rng.randint(1, 9)
        part = [d.encode("utf-8") for d in docs[j: j + k]]
        offs = np.zeros(len(part), dtype=np.uint64)
        if len(part) > 1:
            offs[1:] = np.cumsum([len(b) for b in part[:-1]])
        per_call.append(eng.dedup_add_docs(b"".join(part), offs))
        if between is not None:
            between()
        j += k
    nc, ne = eng.dedup_finish()
    return nc, ne, per_call


def check_session(eng, docs, specials, pat, nc, ne, merges=0):
    data, offs = part_chunks(docs, specials, pat)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    b, o = eng.chunk_entries()
    assert np.array_equal(b, ub) and np.array_equal(o, uo)
    assert np.array_equal(eng.chunk_weights(), np.asarray(uw, dtype=np.uint64))
    assert nc == len(offs) and ne == len(uo)
    st = eng.dedup_stats()
    assert st["text_chunks"] == nc and st["entries"] == ne
    if merges:
        pairs, counts, done = eng.train(merges)
        wp, wc, wd = oracle.c_train(data.astype(np.int32), offs, merges)
        assert done == wd and np.array_equal(pairs, wp) and np.array_equal(counts, wc)


@pytest.mark.parametrize("which", [0, 1, 3])
def test_session_equals_the_oracle(which, taylorswift):
    """Entries, weights and chunk counts of a session with specials are the oracle's of the per-part chunks, in one call and
    in calls of random size; training on them gives the oracle's merges and counts."""
    docs = corpus(taylorswift)
    specials = {EOT: 0, IMS: 1, **EDGE_SPECIALS}
    pat = regex.compile(_pattern(which))
    eng = _engine(which)
    nc, ne, _ = session(eng, docs, specials)
    check_session(eng, docs, specials, pat, nc, ne, MERGES)
    nc2, ne2, per_call = session(eng, docs, specials, random.Random(which))
    assert len(per_call) > 3 and sum(per_call) == nc2 == nc and ne2 == ne
    check_session(eng, docs, specials, pat, nc2, ne2)
    eng.close()


def test_edge_cases_in_one_document_and_across_documents(taylorswift):
    """The edge cases as one long document and cut into documents; a special that only exists across two documents
    (\"<|endo\" + \"ftext|>\") never matches; dict order decides between overlapping specials and prefixes."""
    pat = regex.compile(_pattern(0))
    filler = taylorswift[:70000]
    text = EDGE + filler + "<|endo"
    docs = [text, "ftext|> more" + EOT, EDGE, "<|eo", "t|>" + EDGE]
    for specials in (EDGE_SPECIALS, dict(reversed(list(EDGE_SPECIALS.items())))):
        eng = _engine(0)
        nc, ne, _ = session(eng, docs, specials)
        check_session(eng, docs, specials, pat, nc, ne, MERGES)
        eng.close()
    assert parts("x<|eot|>", {"<|e": 0, "<|eot|>": 1}) == ["x", "ot|>"]


def test_special_across_a_piece_cut(taylorswift):
    """BPE_OPT_SPLIT_PIECE = 4096: a long document is cut at letter+space points, and never inside an occurrence, even
    where a special holds the only letter+space cut points for a while."""
    from minbpe_b200 import engine as E
    pat = regex.compile(_pattern(0))
    block = "1234567890-" * 60 + "a b<|x" + "0987654321+" * 60 + EOT          # no other letter+space for 1339 bytes
    text = "".join(taylorswift[i * 3000: (i + 1) * 3000] + block for i in range(12)) + EDGE
    specials = {"a b<|x": 0, EOT: 1}
    eng = _engine(0)
    eng.set_option(E.OPT_SPLIT_PIECE, 4096)
    try:
        nc, ne, _ = session(eng, [text, EDGE, text[:9000]], specials)
        check_session(eng, [text, EDGE, text[:9000]], specials, pat, nc, ne, MERGES)
        assert eng.dedup_stats()["pieces"] > 10
    finally:
        eng.set_option(E.OPT_SPLIT_PIECE, 0)      # process-wide
    eng.close()


def test_session_unchanged_by_encodes_with_other_specials(taylorswift):
    """An open session with specials keeps its own set: encode_text_gpt4 and encode_docs with other specials on the
    same engine between two calls change nothing."""
    docs = corpus(taylorswift, seed=2)
    specials = {EOT: 0, IMS: 1}
    eng = _engine(0)
    session(eng, docs, specials)
    want = eng.chunk_entries(), eng.chunk_weights()
    merges = np.array([[101, 32], [116, 104]], dtype=np.int32)
    other = [(b"Once", 5000), (b"<|im_start|", 5001), (b"e", 5002)]

    def between():
        eng.encode_text_gpt4(EDGE.encode() * 50, merges, specials=other)
        eng.encode_docs(("Once upon a time <|im_start|> there was e. " * 100).encode(), [0, 100, 2000], merges, specials=other)

    session(eng, docs, specials, random.Random(5), between)
    got = eng.chunk_entries(), eng.chunk_weights()
    assert all(np.array_equal(a, b) for a, b in zip(got[0], want[0])) and np.array_equal(got[1], want[1])
    eng.close()


def _trained(tok, fn, *args, **kw):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        fn(*args, verbose=True, **kw)
    return out.getvalue()


def _saved(tok, tmp_path, name):
    tok.save(str(tmp_path / name))
    return open(tmp_path / f"{name}.model", "rb").read(), open(tmp_path / f"{name}.vocab", "rb").read()


def _reference(pattern, docs, specials, V, tmp_path):
    """train_from_iterator over the parts, then register_special_tokens: the state every entry point must reach"""
    from minbpe_b200 import RegexTokenizer
    ref = RegexTokenizer(pattern)
    log = _trained(ref, ref.train_from_iterator, [p for d in docs for p in parts(d, specials)], V)
    ref.register_special_tokens(dict(specials))
    return ref, log, _saved(ref, tmp_path, "ref")


def _same(tok, log, ref, ref_log, ref_files, tmp_path, specials):
    assert tok.merges == ref.merges and tok.vocab == ref.vocab and log == ref_log
    assert tok.special_tokens == specials and tok.inverse_special_tokens == {v: k for k, v in specials.items()}
    assert not set(specials.values()) & set(tok.vocab)
    assert _saved(tok, tmp_path, "tok") == ref_files


@pytest.mark.parametrize("which", [0, 1, 3])
def test_train_equals_training_on_the_parts(which, taylorswift, tmp_path):
    """train(text, V, special_tokens=S) (device path, dedup either way) and train_from_iterator(docs, V, special_tokens=S)
    equal train_from_iterator over the parts + register_special_tokens: merges, vocab, verbose lines, .model / .vocab.
    The merges are the oracle's on the part chunks."""
    from minbpe_b200 import RegexTokenizer
    pattern = _pattern(which)
    docs = corpus(taylorswift)
    text = "".join(docs)
    V = 256 + MERGES
    specials = {EOT: V, IMS: V + 7, **{k: V + 10 + v for k, v in EDGE_SPECIALS.items()}}
    ref, ref_log, ref_files = _reference(pattern, [text], specials, V, tmp_path)
    data, offs = part_chunks([text], specials, regex.compile(pattern))
    wp, _, _ = oracle.c_train(data.astype(np.int32), offs, MERGES)
    assert [list(p) for p in ref.merges] == wp.tolist()
    for dedup in (False, True):
        tok = RegexTokenizer(pattern)
        assert len(text.encode()) >= tok.DEVICE_SPLIT_MIN_BYTES
        log = _trained(tok, tok.train, text, V, dedup=dedup, special_tokens=specials)
        _same(tok, log, ref, ref_log, ref_files, tmp_path, specials)
    ref, ref_log, ref_files = _reference(pattern, docs, specials, V, tmp_path)
    tok = RegexTokenizer(pattern)
    log = _trained(tok, tok.train_from_iterator, iter(docs), V, special_tokens=specials)
    _same(tok, log, ref, ref_log, ref_files, tmp_path, specials)


def test_host_fallback(taylorswift, tmp_path):
    """65 specials, a 49-byte special, a pattern the device does not split with, a short text: the host path, with the
    same result as training on the parts."""
    from minbpe_b200 import GPT4_SPLIT_PATTERN, RegexTokenizer
    V = 256 + MERGES
    text = "".join(corpus(taylorswift)[:40])
    many = {f"<|s{i}|>": V + i for i in range(65)}
    long = {EOT: V, "<|" + "x" * 45 + "|>": V + 1}
    cases = [(GPT4_SPLIT_PATTERN, text + "<|s64|>".join(["ab", "cd"]) * 50, many),
             (GPT4_SPLIT_PATTERN, text + "<|" + "x" * 45 + "|>" + text[:3000], long),
             (r"\p{L}+|\s+|[^\p{L}\s]+", text, {EOT: V, IMS: V + 1}),
             (GPT4_SPLIT_PATTERN, EDGE * 20 + text[:20000], {k: V + v for k, v in EDGE_SPECIALS.items()})]
    for pattern, t, specials in cases:
        ref, ref_log, ref_files = _reference(pattern, [t], specials, V, tmp_path)
        tok = RegexTokenizer(pattern)
        log = _trained(tok, tok.train, t, V, special_tokens=specials)
        _same(tok, log, ref, ref_log, ref_files, tmp_path, specials)
        tok = RegexTokenizer(pattern)
        log = _trained(tok, tok.train_from_iterator, [t[:5000], t[5000:]], V, special_tokens=specials)
        ref2, ref2_log, ref2_files = _reference(pattern, [t[:5000], t[5000:]], specials, V, tmp_path)
        _same(tok, log, ref2, ref2_log, ref2_files, tmp_path, specials)


def test_text_of_specials_only_and_argument_errors(taylorswift):
    """A text made only of specials has no pairs: ValueError for V > 256, state unchanged; V == 256 trains nothing and
    registers the specials.  Bad arguments raise ValueError before any work, state unchanged; {} is no argument."""
    from minbpe_b200 import RegexTokenizer
    text = taylorswift[:70000]
    V = 256 + MERGES
    tok = RegexTokenizer()
    tok.train(text, V, special_tokens={EOT: V})
    state = (dict(tok.merges), dict(tok.vocab), dict(tok.special_tokens))
    only = (EOT + IMS) * 4000
    for fn, arg in ((tok.train, only), (tok.train_from_iterator, [only, EOT])):
        with pytest.raises(ValueError):
            fn(arg, 300, special_tokens={EOT: 400, IMS: 401})
        assert (tok.merges, tok.vocab, tok.special_tokens) == state
    bad = [{"": V}, {1: V}, {EOT: V - 1}, {EOT: 2 ** 31}, {EOT: float(V)}, {EOT: True}, {EOT: V, IMS: V}, [(EOT, V)]]
    for special in bad:
        for fn, arg in ((tok.train, text), (tok.train_from_iterator, [text])):
            with pytest.raises(ValueError):
                fn(arg, V, special_tokens=special)
            assert (tok.merges, tok.vocab, tok.special_tokens) == state
    t2 = RegexTokenizer()
    t2.train(only, 256, special_tokens={EOT: 256, IMS: 257})
    assert t2.merges == {} and t2.special_tokens == {EOT: 256, IMS: 257}
    a, b = RegexTokenizer(), RegexTokenizer()
    a.train(text, V, special_tokens={})
    b.train(text, V)
    assert a.merges == b.merges and a.vocab == b.vocab and a.special_tokens == {} == b.special_tokens


def test_resume(taylorswift):
    """train(k, S); train(N, resume=True, S) == train(N, S); the ids must be at least the new vocab_size."""
    from minbpe_b200 import RegexTokenizer
    docs = corpus(taylorswift)
    text = "".join(docs)
    V1, V2 = 256 + MERGES // 2, 256 + MERGES
    specials = {EOT: V2, IMS: V2 + 1}
    full = RegexTokenizer()
    full.train(text, V2, special_tokens=specials)
    for fn, arg in (("train", text), ("train_from_iterator", docs)):
        part = RegexTokenizer()
        getattr(part, fn)(arg, V1, special_tokens=specials)
        with pytest.raises(ValueError):
            getattr(part, fn)(arg, V2, resume=True, special_tokens={EOT: V2 - 1})
        getattr(part, fn)(arg, V2, resume=True, special_tokens=specials)
        ref = full
        if fn == "train_from_iterator":
            ref = RegexTokenizer()
            ref.train_from_iterator(docs, V2, special_tokens=specials)
        assert part.merges == ref.merges and part.vocab == ref.vocab and part.special_tokens == specials


def _write(tmp_path, name, text):
    path = str(tmp_path / f"{name}.txt")
    with open(path, "wb") as f:
        f.write(text.encode("utf-8"))
    return path


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def straddling_text(taylorswift):
    """A text whose half-way cut point (the world = 2 shard boundary) has its first letter+space inside a special."""
    a = taylorswift[:30000 if SMALL else 80000]
    a = a.encode("ascii", "ignore").decode()
    mid = "1234<|q r|>"
    b = a[: len(a) - 7]
    text = a + mid + b
    assert len(text.encode()) // 2 == len(a) + 2
    return text


def test_train_from_file_one_gpu_and_shards(taylorswift, tmp_path):
    """train_from_file(special_tokens=S) equals train(text, S); every rank's range, played one after another, avoids the
    straddling special, and the merged shards give the single-GPU stream.  Specials the device does not take: ValueError."""
    from minbpe_b200 import RegexTokenizer, dist as D
    text = straddling_text(taylorswift)
    specials = {"<|q r|>": 1000, EOT: 1001}
    path = _write(tmp_path, "c", text)
    V = 256 + MERGES
    a, b = RegexTokenizer(), RegexTokenizer()
    a.train_from_file(path, V, special_tokens=specials)
    b.train(text, V, special_tokens=specials)
    assert a.merges == b.merges and a.vocab == b.vocab and a.special_tokens == specials
    raw = text.encode()
    lo, hi = D.shard_byte_range(len(raw), 0, 2, lambda x, y: np.frombuffer(raw[x:y], np.uint8), specials=[b"<|q r|>"])
    assert hi > raw.index(b"<|q r|>") + 7 and D.shard_byte_range(len(raw), 0, 2, lambda x, y: np.frombuffer(raw[x:y], np.uint8))[1] < hi
    eng = _engine(0)
    spec = [k.encode() for k in specials]
    parts_ = [D.count_file_shard(eng, path, r, 2, spec) for r in range(2)]
    D.load_merged_shards(eng, parts_)
    want = _engine(0)
    want.load_text_gpt4_dedup(raw, spec)
    for x, y in zip(eng.chunk_entries() + (eng.chunk_weights(),), want.chunk_entries() + (want.chunk_weights(),)):
        assert np.array_equal(x, y)
    assert sum(p[3] for p in parts_) == want.dedup_stats()["text_chunks"]
    eng.close()
    want.close()
    with pytest.raises(ValueError):
        RegexTokenizer().train_from_file(path, V, special_tokens={"<|" + "x" * 47 + "|>": 1000})


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(rank, world, port, path, V, specials, out_dir, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        from minbpe_b200 import RegexTokenizer
        tok = RegexTokenizer(device=0)
        tok.train_from_file(path, V, special_tokens=specials)
        prefix = os.path.join(out_dir, f"r{world}_{rank}")
        tok.save(prefix)
        q.put((rank, [list(p) for p in tok.merges], _sha(prefix + ".model"), _sha(prefix + ".vocab")))
        tok.engine.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_train_from_file_gloo_ranks(world, taylorswift, tmp_path):
    """`world` processes over gloo, every one on cuda:0, with a special straddling the natural cut: every rank's merges
    and files equal the single-GPU train_from_file."""
    import torch.multiprocessing as mp
    from minbpe_b200 import RegexTokenizer
    text = straddling_text(taylorswift)
    specials = {"<|q r|>": 1000, EOT: 1001}
    path = _write(tmp_path, "c", text)
    V = 256 + MERGES
    one = RegexTokenizer(device=0)
    one.train_from_file(path, V, special_tokens=specials)
    one.save(str(tmp_path / "one"))
    ref = ([list(p) for p in one.merges], _sha(str(tmp_path / "one.model")), _sha(str(tmp_path / "one.vocab")))
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, path, V, specials, str(tmp_path), q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        out = sorted(q.get(timeout=1800 if SMALL else 600) for _ in procs)
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0, p.exitcode
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)
    assert [o[0] for o in out] == list(range(world))
    for rank, merges, msha, vsha in out:
        assert (merges, msha, vsha) == ref, rank
