"""GPU: special-token sets of up to 65,536 specials on the device (DESIGN.md §19) — the trie matcher k_special_find, the
16-bit candidate index, the u32 `which` of every host path, the seeding of large sets into the encode memo, and the
cross-document re-pick and piece cuts through the host copy of the trie.  Every case is compared with the reference's
procedure: re.split at the specials (regex.py:152-163), then the oracle's encode or training on every part's chunks."""
import contextlib
import functools
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
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller texts, fewer merges
MERGES = 40 if SMALL else 200
PATTERNS = {0: "GPT4_SPLIT_PATTERN", 1: "GPT2_SPLIT_PATTERN", 3: "O200K_SPLIT_PATTERN"}


def _pattern(which):
    import minbpe_b200.tokenizer as T
    return getattr(T, PATTERNS[which])


@functools.lru_cache(maxsize=8)
def _splitter(names):
    return regex.compile("(" + "|".join(regex.escape(k) for k in names) + ")")


def parts(text, special):
    """regex.py:152-158: the text split at the specials, the occurrences at odd positions"""
    return _splitter(tuple(special)).split(text) if special else [text]


def ref_encode(text, special, merges, pattern):
    """regex.py:152-163 with oracle.c_encode as encode_ordinary"""
    pat = regex.compile(pattern)
    out = []
    for i, part in enumerate(parts(text, special)):
        if i % 2:
            out.append(special[part])
        elif part:
            d, o = oracle.split_to_stream(part, pat)
            out.extend(oracle.c_encode(d, o, merges).tolist())
    return out


def llama3_names():
    """The 256 special tokens of Llama 3, in id order"""
    r = [f"<|reserved_special_token_{i}|>" for i in range(251)]
    return (["<|begin_of_text|>", "<|end_of_text|>"] + r[0:4] + ["<|start_header_id|>", "<|end_header_id|>", r[4], "<|eot_id|>"]
            + r[5:])


def big_set(base, extra=44):
    """Llama 3's 256 specials followed by `extra` more, so that an index does not fit 8 bits: {name: base + index}"""
    names = llama3_names() + [f"<|extra_{i}|>" for i in range(extra)]
    return {k: base + i for i, k in enumerate(names)}


def body(n):
    from minbpe_b200.synth import generate
    return generate(1337, max(n * 2, 1 << 16)).tobytes().decode("utf-8", "ignore")[:n]


def with_specials(text, names, rng, every):
    """text with a special from `names` after roughly every `every` characters"""
    out = []
    for i in range(0, len(text), every):
        out.append(text[i:i + every])
        out.append(rng.choice(names))
    return "".join(out)


@pytest.fixture(scope="module")
def trained():
    """{pattern: (tokenizer, merges array)} trained on a synthetic text"""
    from minbpe_b200 import RegexTokenizer
    text = body(120000 if SMALL else 300000)
    out = {}
    for which in PATTERNS:
        t = RegexTokenizer(_pattern(which))
        t.train(text, 256 + MERGES)
        out[which] = (t, np.array(list(t.merges.keys()), dtype=np.int32).reshape(-1, 2))
    return out


def _engine(which=0):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_SPLIT_PATTERN, which)
    return eng


def _enc(eng, text, merges, special):
    spec = [(k.encode("utf-8"), v) for k, v in special.items()] if special else None
    return eng.encode_text_gpt4(text.encode("utf-8"), merges, specials=spec).tolist()


def _llama_text(n, sp, seed):
    """a text holding the specials of index 0, 63, 64, 255, 256 and the last one, and many others"""
    names = list(sp)
    rng = random.Random(seed)
    must = [names[i] for i in (0, 63, 64, 255, 256, len(names) - 1)]
    t = with_specials(body(n), names, rng, 700)
    return "".join(must) + t[: len(t) // 2] + " ".join(must) + t[len(t) // 2:] + must[3]


@pytest.mark.parametrize("which", [0, 1, 3])
def test_llama3_set_encode(which, trained, tmp_path):
    """300 specials (Llama 3's 256 and 44 more): encode with "all", a subset and "none", encode_batch, encode_file — the
    device path every time, equal to re.split + the oracle on every part."""
    tok, merges = trained[which]
    pattern = _pattern(which)
    sp = big_set(100000)
    tok.register_special_tokens(sp)
    text = _llama_text(90000 if SMALL else 250000, sp, which)
    assert len(text.encode()) >= tok.DEVICE_SPLIT_MIN_BYTES and tok._device_specials(sp)
    want = ref_encode(text, sp, merges, pattern)
    assert sum(1 for x in want if x >= 100000) > 100 and {100000, 100063, 100064, 100255, 100256, 100299} <= set(want)
    assert tok.encode(text, allowed_special="all") == want
    sub = {k for k, v in sp.items() if v in (100003, 100064, 100256, 100280)}
    assert tok.encode(text, allowed_special=sub) == ref_encode(text, {k: sp[k] for k in sp if k in sub}, merges, pattern)
    assert tok.encode(text, allowed_special="none") == ref_encode(text, {}, merges, pattern)
    docs = [text[i: i + 9000] for i in range(0, len(text), 9000)]
    assert tok.encode_batch(docs, allowed_special="all") == [ref_encode(d, sp, merges, pattern) for d in docs]
    path = str(tmp_path / "c.txt")
    with open(path, "wb") as f:
        f.write(text.encode())
    assert tok.encode_file(path, "all").tolist() == want
    tok.register_special_tokens({})


def _trained_log(fn, *args, **kw):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        fn(*args, verbose=True, **kw)
    return out.getvalue()


def _part_chunks(docs, special, pattern):
    pat = regex.compile(pattern)
    chunks = [c.encode("utf-8") for d in docs for p in parts(d, special)[0::2] for c in pat.findall(p)]
    offs = np.zeros(len(chunks), dtype=np.uint64)
    if len(chunks) > 1:
        offs[1:] = np.cumsum([len(c) for c in chunks[:-1]])
    return np.frombuffer(b"".join(chunks), dtype=np.uint8), offs


@pytest.mark.parametrize("which", [0, 1, 3])
def test_llama3_set_training(which, tmp_path):
    """train, train_from_iterator and train_from_file with the 300 specials give the merges of the oracle on the parts'
    chunks, and the state of train_from_iterator over the parts followed by register_special_tokens."""
    from minbpe_b200 import RegexTokenizer
    pattern = _pattern(which)
    V = 256 + MERGES
    sp = big_set(V)
    text = _llama_text(90000 if SMALL else 250000, sp, 10 + which)
    docs = [text[i: i + 7000] for i in range(0, len(text), 7000)]
    data, offs = _part_chunks([text], sp, pattern)
    wp, _, _ = oracle.c_train(data.astype(np.int32), offs, MERGES)
    ref = RegexTokenizer(pattern)
    ref_log = _trained_log(ref.train_from_iterator, parts(text, sp)[0::2], V)
    assert [list(p) for p in ref.merges] == wp.tolist()
    path = str(tmp_path / "c.txt")
    with open(path, "wb") as f:
        f.write(text.encode())
    for fn, arg in (("train", text), ("train_from_file", path)):
        tok = RegexTokenizer(pattern)
        log = _trained_log(getattr(tok, fn), arg, V, special_tokens=sp)
        assert tok.merges == ref.merges and tok.vocab == ref.vocab and log == ref_log and tok.special_tokens == sp, fn
    data, offs = _part_chunks(docs, sp, pattern)
    wp, _, _ = oracle.c_train(data.astype(np.int32), offs, MERGES)
    tok = RegexTokenizer(pattern)
    tok.train_from_iterator(iter(docs), V, special_tokens=sp)
    assert [list(p) for p in tok.merges] == wp.tolist() and tok.special_tokens == sp


def _session_entries(eng, docs, names):
    eng.dedup_begin()
    eng.dedup_set_specials([k.encode("utf-8") for k in names])
    b = [d.encode("utf-8") for d in docs]
    offs = np.zeros(len(b), dtype=np.uint64)
    if len(b) > 1:
        offs[1:] = np.cumsum([len(x) for x in b[:-1]])
    eng.dedup_add_docs(b"".join(b), offs)
    eng.dedup_finish()
    return eng.chunk_entries(), eng.chunk_weights()


def _counted(b, o, w):
    """{chunk: weight} in first-occurrence order; a chunk longer than the counting key is an entry per occurrence
    (DESIGN.md §14), so entries of equal bytes are summed"""
    ends = list(o[1:]) + [len(b)]
    out = {}
    for s, e, x in zip(o, ends, w):
        k = bytes(b[int(s):int(e)])
        out[k] = out.get(k, 0) + int(x)
    return list(out.items())


def _check_session(eng, docs, special, pattern):
    (b, o), w = _session_entries(eng, docs, special)
    assert _counted(b, o, w) == _counted(*oracle.c_dedup_chunks(*_part_chunks(docs, special, pattern)))


def _filler(n, base, tag="f"):
    return {f"<{tag}{i}>": base + i for i in range(n)}


def test_prefix_chains_beyond_64(trained):
    """Chains of specials where one is a prefix of the next, with the short one at an index above 64 and the long one
    below, and the reverse; every special sharing its first byte; a, aa, ... a*48 over runs of a.  The first special in
    dict order that matches wins, not the longest."""
    _, merges = trained[0]
    pattern = _pattern(0)
    chain = ["<|x" + "|>"[:j] + "y" * max(0, j - 2) for j in range(0, 12)]          # <|x, <|x|, <|x|>, <|x|>y, ...
    filler = list(_filler(70, 0))
    sets = [chain[6:][::-1] + filler + chain[:6], chain[:6] + filler + chain[6:][::-1],   # long ones low / short ones low
            chain[::-1] + filler, chain + filler]
    same_first = ["<" + chr(65 + (i % 26)) * (1 + i // 26) for i in range(300)]                      # one first byte
    runs = ["a" * n for n in range(1, 49)]
    sets += [same_first, same_first[::-1], runs, runs[::-1], filler + runs[::-1], filler + runs]
    rng = random.Random(3)
    text = body(70000)
    eng = _engine(0)
    for names in sets:
        special = {k: 50000 + i for i, k in enumerate(names)}
        t = "".join(text[i:i + 600] + rng.choice(names + chain) + rng.choice(["", "|>", "yy", "a" * rng.randint(1, 120)])
                    for i in range(0, len(text), 600))
        assert _enc(eng, t, merges, special) == ref_encode(t, special, merges, pattern), names[:3]
        docs = [t[i: i + 3000] for i in range(0, len(t), 3000)]
        _check_session(eng, docs, special, pattern)
    eng.close()


@functools.lru_cache(maxsize=1)
def _set_65536():
    rng = random.Random(65536)
    alpha = "abcdefghijklmnopqrstuvwxyz0123456789_|>"
    names = {}
    while len(names) < 65536 - 64:     # long ones first: a short one early would shadow every special it is a prefix of
        names.setdefault("<|" + "".join(rng.choice(alpha) for _ in range(rng.randint(6, 46))), None)
    while len(names) < 65535:
        names.setdefault("<|" + "".join(rng.choice(alpha) for _ in range(rng.randint(1, 5))), None)
    return list(names) + ["<|"]         # 2 bytes, last: it matches wherever no other special does


def test_65536_and_65537_specials(trained):
    """65,536 distinct specials of 2..48 bytes with the same first two bytes: the device path, equal to re.split.  One more
    is an error of the C ABI, and the class keeps the host split with the same answer."""
    from minbpe_b200 import engine as E
    tok, merges = trained[0]
    pattern = _pattern(0)
    names = _set_65536()
    sp = {k: 100000 + i for i, k in enumerate(names)}
    rng = random.Random(5)
    pick = [names[i] for i in (0, 1, 255, 256, 40000, 65535)] + [rng.choice(names) for _ in range(40)]
    text = with_specials(body(66000), pick + ["<|", "<|a", "<|zz"], rng, 1400)
    want = ref_encode(text, sp, merges, pattern)
    assert sum(1 for x in want if x >= 100000) > 30 and max(want) >= 100000 + 40000
    tok.register_special_tokens(sp)
    assert tok._device_specials(sp)
    eng = tok.engine
    import minbpe_b200.tokenizer as T
    real_split = T.re.split
    T.re.split = None                                # the host split would fail: the class must take the device path
    try:
        assert tok.encode(text, allowed_special="all") == want
    finally:
        T.re.split = real_split
    st = eng.encode_stats()
    assert st["pieces"] >= 1 and st["memo_chunks"] >= 65536
    more = dict(sp)
    more["<|one more|>"] = 99999
    text2 = text + "<|one more|>" + text[:100]
    with pytest.raises(E.EngineError):
        _enc(eng, text2, merges, more)
    tok.register_special_tokens(more)
    assert not tok._device_specials(more)
    assert tok.encode(text2, allowed_special="all") == ref_encode(text2, more, merges, pattern)
    tok.register_special_tokens({})


def test_general_path_with_a_high_index(trained):
    """A piece with a chunk too long for the memo encode takes the general path (encode_parts), which emits the ids of
    the occurrences itself: indices 256 and above must keep their ids there."""
    _, merges = trained[0]
    pattern = _pattern(0)
    sp = big_set(100000)
    names = list(sp)
    b = body(90000)
    t = (b[:30000] + names[299] + "lyiltumdya" * 1200 + " " + names[256] + b[30000:60000] + names[257] + names[1]
         + names[511 % len(names)] + b[60000:])
    eng = _engine(0)
    assert _enc(eng, t, merges, sp) == ref_encode(t, sp, merges, pattern)
    assert eng.encode_stats()["fallback_pieces"] == 1
    docs = [t[:20000], t[20000:-1000], t[-1000:]]
    raw = [d.encode() for d in docs]
    offs = np.cumsum([0] + [len(x) for x in raw[:-1]]).astype(np.uint64)
    ids, o = eng.encode_docs(b"".join(raw), offs, merges, specials=[(k.encode(), v) for k, v in sp.items()])
    assert eng.encode_stats()["fallback_pieces"] == 1
    assert [ids[o[j]:o[j + 1]].tolist() for j in range(3)] == [ref_encode(d, sp, merges, pattern) for d in docs]
    eng.close()


def test_piece_cuts_and_documents(trained):
    """BPE_OPT_SPLIT_PIECE: a special holding letter+space at index > 64 is never cut.  A special straddling two documents
    does not match; a shorter special of a higher index that matches inside the first document does."""
    from minbpe_b200 import engine as E
    _, merges = trained[0]
    pattern = _pattern(0)
    sp = {**_filler(100, 7000), "a b<|x": 8000, "<|q r|>": 8001, **_filler(100, 9000, "g"), "<|q": 9500}
    assert list(sp).index("<|q") > 200
    block = "1234567890-" * 60 + "a b<|x" + "0987654321+" * 60 + "<|q r|>"
    b = body(40000)
    text = "".join(b[i * 3000: (i + 1) * 3000] + block for i in range(12))
    eng = _engine(0)
    eng.set_option(E.OPT_SPLIT_PIECE, 4096)
    try:
        assert _enc(eng, text, merges, sp) == ref_encode(text, sp, merges, pattern)
        assert eng.encode_stats()["pieces"] > 10
        docs = [text, text[:9000]]
        _check_session(eng, docs, sp, pattern)
    finally:
        eng.set_option(E.OPT_SPLIT_PIECE, 0)      # process-wide
    # "<|q r|>" (index 101) straddles the start of the second document; "<|q" (index 201) matches inside the first
    docs = [b[:30000] + "<|q", " r|>" + b[30000:50000] + "<|q r|>", "<|q r|>" + b[50000:60000] + "<|q", " r|>" + b[:5000]]
    raw = [d.encode() for d in docs]
    offs = np.cumsum([0] + [len(x) for x in raw[:-1]]).astype(np.uint64)
    spec = [(k.encode(), v) for k, v in sp.items()]
    ids, o = eng.encode_docs(b"".join(raw), offs, merges, specials=spec)
    got = [ids[o[j]:o[j + 1]].tolist() for j in range(len(docs))]
    assert got == [ref_encode(d, sp, merges, pattern) for d in docs]
    assert got[0][-1] == 9500 and got[1][-1] == 8001
    _check_session(eng, docs, sp, pattern)
    eng.close()


def test_memo_sets_switched_and_memo_smaller_than_the_set(trained):
    """300 -> 5 -> none -> 300 specials on one engine: no set sees another's memo entries.  A memo of 256 slots cannot
    hold 300 specials: every piece takes the general path, with the right ids."""
    from minbpe_b200 import engine as E
    _, merges = trained[0]
    pattern = _pattern(0)
    big = big_set(100000)
    names = list(big)
    small = {names[i]: 200000 + i for i in (299, 256, 3, 0, 255)}
    text = _llama_text(70000, big, 7)
    eng = _engine(0)
    for special in (big, small, None, big, small):
        assert _enc(eng, text, merges, special) == ref_encode(text, special or {}, merges, pattern)
    eng.set_option(E.OPT_ENC_MEMO_LOG2, 8)
    try:
        for special in (big, small, big):
            assert _enc(eng, text, merges, special) == ref_encode(text, special, merges, pattern)
            st = eng.encode_stats()
            if special is big:
                assert st["fallback_pieces"] == st["pieces"] >= 1, st
    finally:
        eng.set_option(E.OPT_ENC_MEMO_LOG2, 0)
    eng.close()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(rank, world, port, path, V, specials, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        from minbpe_b200 import RegexTokenizer
        tok = RegexTokenizer(device=0)
        tok.train_from_file(path, V, special_tokens=specials)
        ids = tok.encode_file(path, "all", gather=True)
        q.put((rank, [list(p) for p in tok.merges], None if ids is None else ids.tolist()))
        tok.engine.close()
    finally:
        dist.destroy_process_group()


def test_gloo_ranks_with_a_straddling_special(tmp_path):
    """train_from_file and encode_file over 2 gloo ranks (both on cuda:0), 300 specials, one of index > 256 straddling the
    natural cut: every rank's merges and the gathered ids equal one GPU's."""
    import torch.multiprocessing as mp
    from minbpe_b200 import RegexTokenizer
    V = 256 + MERGES
    sp = big_set(V)
    sp["<|q r|>"] = V + 400
    a = body(30000 if SMALL else 80000).encode("ascii", "ignore").decode()
    text = a + "1234<|q r|>" + a[: len(a) - 7]
    assert len(text.encode()) // 2 == len(a) + 2
    path = str(tmp_path / "c.txt")
    with open(path, "wb") as f:
        f.write(text.encode())
    one = RegexTokenizer(device=0)
    one.train_from_file(path, V, special_tokens=sp)
    want_ids = one.encode_file(path, "all").tolist()
    assert want_ids == ref_encode(text, sp, np.array(list(one.merges), dtype=np.int32), _pattern(0))
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, 2, port, path, V, sp, q)) for r in range(2)]
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
    assert [o[0] for o in out] == [0, 1]
    for rank, merges, ids in out:
        assert merges == [list(p) for p in one.merges], rank
    assert out[0][2] == want_ids
