"""GPU: every hashed structure against crafted collisions (tests/hash_craft.py), compared with the oracle.

A — host caches, keyed on contents: merges, byte maps and special-token sets with the same 64-bit hash as the previous
call's must not reuse the rank table, the encode memo or the special set built for it.
B — device tables: memo tag collisions and full probe chains (k_encode2.cuh), exact key collisions and full probe chains
of the chunk table (k_dedup.cuh), shared-memory histogram overflow (k_stats.cuh) and rank-table clusters that wrap past
the last slot (k_encode.cuh).

Every case also asserts a path witness (a counter showing that the slow path ran), so that it fails rather than passes
vacuously if a hash changes and the crafted input stops colliding."""
import os
import random

import numpy as np
import pytest
import regex

import hash_craft as H
import oracle

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller texts
GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
MEMO_MIN = 1 << 16          # bpe_encode takes the memo path from this many bytes (ENC2_MIN_BYTES)


def _engine():
    from minbpe_b200 import engine as E
    return E.Engine(0)


@pytest.fixture(scope="module")
def corpus():
    from minbpe_b200.synth import generate
    text = generate(1337, (1 << 16) + 4096 if SMALL else 1 << 20).tobytes().decode("utf-8", "ignore")
    data, offs = oracle.split_to_stream(text, GPT4)
    merges, _, _ = oracle.c_train(data.astype(np.int32), offs, 120 if SMALL else 400)
    return text, data, offs, np.ascontiguousarray(merges, dtype=np.int32)


def _ref_text(text, merges, perm=None, specials=None):
    """encode(text) of the reference (regex.py:152-163) with oracle.c_encode for every part between special tokens"""
    out = []
    special = {t.decode("utf-8"): i for t, i in specials} if specials else None
    parts = regex.split("(" + "|".join(regex.escape(k) for k in special) + ")", text) if special else [text]
    for part in parts:
        if special and part in special:
            out.append(special[part])
        elif part:
            d, o = oracle.split_to_stream(part, GPT4)
            out.extend(oracle.c_encode(d, o, merges, perm).tolist())
    return out


def _docs(text, n):
    """text cut at n - 1 letter+space points into documents (the GPT-4 chunks of the documents are the text's)"""
    rng = random.Random(n)
    pts = [i for i in range(1, len(text)) if text[i] == " " and text[i - 1].isascii() and text[i - 1].isalpha()]
    cuts = sorted(rng.sample(pts, n - 1)) + [len(text)]
    docs, prev = [], 0
    for c in cuts:
        docs.append(text[prev:c])
        prev = c
    return docs


def _encode_docs(eng, docs, merges, perm=None, specials=None):
    data = [d.encode("utf-8") for d in docs]
    offs = np.zeros(len(data), dtype=np.uint64)
    offs[1:] = np.cumsum([len(b) for b in data[:-1]])
    ids, o = eng.encode_docs(b"".join(data), offs, merges, perm, specials)
    return ids.tolist(), o


# ---- A: host caches ----------------------------------------------------------------------------------------------------
PATHS = ["memo_offsets", "text_gpt4", "docs", "general_one_chunk"]


def _run_path(path, eng, text, data, offs, merges, perm=None):
    """-> (ids, what the oracle gives) of one call on `path`"""
    if path == "memo_offsets":
        assert data.size >= MEMO_MIN
        return eng.encode(data, offs, merges, perm).tolist(), oracle.c_encode(data, offs, merges, perm).tolist()
    if path == "text_gpt4":
        return eng.encode_text_gpt4(data.tobytes(), merges, perm).tolist(), oracle.c_encode(data, offs, merges, perm).tolist()
    if path == "docs":
        got, _ = _encode_docs(eng, _docs(text, 7), merges, perm)
        return got, oracle.c_encode(data, offs, merges, perm).tolist()
    raw = data[:3000]                               # one chunk: the general path (k_encode_long)
    return eng.encode(raw, None, merges, perm).tolist(), oracle.c_encode(raw, None, merges, perm).tolist()


@pytest.mark.parametrize("path", PATHS)
def test_a1_merges_with_equal_hash_rebuild_the_rank_table(path, corpus):
    text, data, offs, M = corpus
    M2 = H.merges_collision(M, 3, seed=5)
    assert H.hash_bytes(M2.tobytes()) == H.hash_bytes(M.tobytes()) and not np.array_equal(M, M2)
    eng = _engine()
    h2d = []
    for m in (M, M2, M, M):
        got, want = _run_path(path, eng, text, data, offs, m)
        assert got == want, path
        h2d.append(eng.timing()["h2d_bytes"])
    # the two tables give different ids on this text, or the case would prove nothing
    assert _run_path(path, eng, text, data, offs, M2)[1] != _run_path(path, eng, text, data, offs, M)[1]
    # witness: every switch rebuilt the rank table (8 bytes per merge uploaded); the repeated call did not
    assert h2d[1] - h2d[3] == 8 * len(M) and h2d[2] - h2d[3] == 8 * len(M), h2d
    eng.close()


@pytest.mark.parametrize("path", PATHS)
def test_a2_byte_maps_with_equal_hash_clear_the_memo(path, corpus):
    text, data, offs, M = corpus
    P = np.random.default_rng(11).permutation(256).astype(np.uint8)
    P2 = H.perm_collision(P, 12, seed=3)            # bytes 96..111: lower-case letters
    assert H.hash_bytes(P2.tobytes()) == H.hash_bytes(P.tobytes())
    eng = _engine()
    new = []
    for p in (P, P2, P, P):
        got, want = _run_path(path, eng, text, data, offs, M, p)
        assert got == want, path
        new.append(eng.encode_stats()["new_chunks"])
    assert _run_path(path, eng, text, data, offs, M, P2)[1] != _run_path(path, eng, text, data, offs, M, P)[1]
    if path != "general_one_chunk":                 # witness: the memo was cleared on every switch, kept on the repeat
        assert new[1] > 0 and new[2] > 0 and new[3] == 0, new
    eng.close()


SPEC_A = [(b"<|a|>", 100257), (b"<|b|>", 100258)]
SPEC_H = [(b"hello", 100300), (b"<|e|>", 100301)]       # a special that is an ordinary word


def _special_sets():
    B = H.specials_collision_search(SPEC_A, lambda t: [b"<|c%02d|>" % t, b"<|d|>"])
    H2 = H.specials_collision_search(SPEC_H, lambda t: [b"<|f%03d|>" % t, b"<|g|>"])
    for x, y in ((SPEC_A, B), (SPEC_H, H2)):
        assert H.spec_hash(x) == H.spec_hash(y) and x != y
    return B, H2


def _special_text(text):
    n = 4000 if SMALL else 40000
    words = text[:n].split(" ")
    rng = random.Random(5)
    ins = ["<|a|>", "<|b|>", "<|c00|>", "<|d|>", "\nhello", " hello", "hello ", "<|e|>", "<|g|>"]
    for j in range(0, len(words), 37):
        words[j] = words[j] + rng.choice(ins)
    return " ".join(words)


@pytest.mark.parametrize("how", ["text_gpt4", "docs"])
def test_a3_special_sets_with_equal_hash_are_told_apart(how, corpus):
    text, _, _, M = corpus
    B, H2 = _special_sets()
    t = _special_text(text)
    eng = _engine()
    for x, y in ((SPEC_A, B), (SPEC_H, H2)):
        for s in (x, y, x, y):
            want = _ref_text(t, M, specials=s)
            if how == "text_gpt4":
                got = eng.encode_text_gpt4(t.encode(), M, specials=s).tolist()
            else:
                got, _ = _encode_docs(eng, _docs(t, 5), M, specials=s)
            assert got == want, (how, s)
            fresh = _engine()
            assert fresh.encode_text_gpt4(t.encode(), M, specials=s).tolist() == want
            fresh.close()
        assert _ref_text(t, M, specials=x) != _ref_text(t, M, specials=y)
    eng.close()


def test_a3_two_tokenizers_on_the_default_engine(corpus):
    from minbpe_b200 import RegexTokenizer
    text, _, _, M = corpus
    B, H2 = _special_sets()
    t = _special_text(text)
    while len(t.encode()) < MEMO_MIN:               # the device front end takes texts of at least 64 KiB
        t = t + " " + t
    toks = []
    for s in (SPEC_H, H2, SPEC_A, B):
        tok = RegexTokenizer()
        tok.merges = {(int(a), int(b)): 256 + r for r, (a, b) in enumerate(M.tolist())}
        tok.register_special_tokens({k.decode(): v for k, v in s})
        toks.append((tok, s))
    for tok, s in toks + toks[::-1]:
        assert tok.encode(t, allowed_special="all") == _ref_text(t, M, specials=s), s


# ---- B: device tables ----------------------------------------------------------------------------------------------------
def _filler(rng, n_chunks, vocab=600):
    words = [b" " + bytes(rng.integers(97, 123, int(rng.integers(1, 10))).astype(np.uint8)) for _ in range(vocab)]
    return [words[int(i)] for i in rng.integers(0, vocab, n_chunks)]


def _join(chunks):
    blob = b"".join(chunks)
    o = np.zeros(len(chunks), dtype=np.uint64)
    o[1:] = np.cumsum([len(c) for c in chunks[:-1]])
    return np.frombuffer(blob, dtype=np.uint8), o


def _letters_merges(seed=0, n=300):
    rng = np.random.default_rng(seed)
    m = np.stack([rng.integers(0, 256 + i, 2) for i in range(n)]).astype(np.int32)
    m[:60] = np.stack([rng.integers(32, 123, 2) for _ in range(60)])
    return m


@pytest.mark.parametrize("order", ["ab", "ba"])
def test_b1_memo_tag_collision_in_one_piece(order):
    a = b"abcdefgh" * 2
    b = H.e2_collision(a, b"zzzzzzzz")
    assert H.e2_tag(a) == H.e2_tag(b)
    rng = np.random.default_rng(1)
    M = _letters_merges()
    pair = [a, b] if order == "ab" else [b, a]
    fill = _filler(rng, 12000)
    data, offs = _join(fill[:6000] + pair + fill[6000:] + pair)
    assert data.size >= MEMO_MIN
    eng = _engine()
    for _ in range(2):                              # cold, then warm memo
        assert np.array_equal(eng.encode(data, offs, M), oracle.c_encode(data, offs, M))
        st = eng.encode_stats()
        assert st["fallback_pieces"] + st["direct_chunks"] >= 1, st
    eng.close()


def test_b1_memo_tag_collision_across_calls():
    a = b" tokenize" + b"r-words" + b"!" * 8             # 24 bytes
    b = H.e2_collision(a, b"q" * 16)
    rng = np.random.default_rng(2)
    M = _letters_merges(1)
    fill = _filler(rng, 12000)
    d1, o1 = _join(fill[:6000] + [a] + fill[6000:])
    d2, o2 = _join(fill[:6000] + [b] + fill[6000:] + [a])
    eng = _engine()
    assert np.array_equal(eng.encode(d1, o1, M), oracle.c_encode(d1, o1, M))
    assert eng.encode_stats()["fallback_pieces"] == 0
    assert np.array_equal(eng.encode(d2, o2, M), oracle.c_encode(d2, o2, M))   # the memo holds a's tag already
    st = eng.encode_stats()
    assert st["fallback_pieces"] + st["direct_chunks"] >= 1, st
    eng.close()


def test_b1_memo_tag_collision_with_a_seeded_special(corpus):
    text, data, offs, M = corpus
    c = b" zebrasaurusxyzw"                            # a 16-byte GPT-4 chunk ...
    assert c.decode() not in text
    t = text + c.decode() + " and" + c.decode()
    special = H.e2_collision(c, b"<|spec|>")           # ... and a special (any bytes) with its memo tag
    assert H.e2_tag(special) == H.e2_tag(c) and special not in t.encode()
    d, o = oracle.split_to_stream(t, GPT4)
    eng = _engine()
    got = eng.encode_text_gpt4(t.encode(), M, specials=[(special, 100999)])
    assert np.array_equal(got, oracle.c_encode(d, o, M))
    st = eng.encode_stats()
    assert st["fallback_pieces"] + st["direct_chunks"] >= 1, st
    eng.close()


@pytest.mark.parametrize("log2", [12, 22])
def test_b2_memo_probe_exhaustion(log2):
    from minbpe_b200 import engine as E
    cluster = H.e2_cluster(40, log2, (1 << log2) - 1, prefix=b" cluster", seed=log2)   # home: the last slot, chains wrap
    rng = np.random.default_rng(3)
    M = _letters_merges(2)
    fill = _filler(rng, 12000, vocab=300)
    chunks = fill[:6000] + cluster + fill[6000:] + cluster[::-1]
    data, offs = _join(chunks)
    eng = _engine()
    eng.set_option(E.OPT_ENC_MEMO_LOG2, log2)
    assert np.array_equal(eng.encode(data, offs, M), oracle.c_encode(data, offs, M))
    st = eng.encode_stats()
    assert st["direct_chunks"] >= len(cluster) - H.E2_PROBES, st
    eng.close()


def _dedup_ref(data, offs):
    return oracle.c_dedup_chunks(data, offs, cap_chunks=max(len(offs), 1), cap_bytes=max(data.size, 1))


def test_b3_chunk_table_exact_key_collision():
    a, b = H.dd_collision(3, seed=0)
    assert H.dd_key(a) == H.dd_key(b) and a != b
    rng = np.random.default_rng(4)
    fill = _filler(rng, 3000, vocab=200)
    chunks = [a] + fill[:1500] + [b, a] + fill[1500:] + [b, b]
    data, offs = _join(chunks)
    ub, uo, uw = _dedup_ref(data, offs)
    eng = _engine()
    kept = eng.load_chunks_weighted_dedup(data, offs, np.ones(len(offs), dtype=np.uint64))
    eb, eo = eng.chunk_entries()
    assert kept == len(uo) and np.array_equal(eb, ub) and np.array_equal(eo, uo)
    assert np.array_equal(eng.chunk_weights(), uw.astype(np.uint64))
    ents = {bytes(ub[int(uo[j]): int(uo[j + 1]) if j + 1 < len(uo) else len(ub)]): int(uw[j]) for j in range(len(uo))}
    assert ents[a] == 2 and ents[b] == 3            # both entries keep their own slots
    n = 200
    wp, wc, _ = oracle.c_train(ub.astype(np.int32), uo, n, weights=uw)
    p, c, d = eng.train(n)
    assert d == len(wp) and np.array_equal(p, wp) and np.array_equal(c, wc)
    eng.close()


def test_b4_chunk_table_probe_exhaustion():
    from minbpe_b200 import engine as E
    log2 = 12

    def make(rng, k):
        return [b" " + bytes(rng.integers(97, 123, 6).astype(np.uint8)) for _ in range(k)]
    cluster = H.dd_cluster(H.DD_PROBES + 16, log2, 5, make, seed=1, batch=4096)
    rng = np.random.default_rng(5)
    chunks = [cluster[int(i)] for i in rng.integers(0, len(cluster), 4000)] + _filler(rng, 2000, vocab=100)
    text = b"".join(chunks).decode()
    data, offs = oracle.split_to_stream(text, GPT4)
    assert len(offs) == len(chunks)                 # the crafted chunks are GPT-4 chunks
    ub, uo, uw = _dedup_ref(data, offs)
    eng = _engine()
    eng.set_option(E.OPT_DEDUP_LOG2, log2)
    nc, ne = eng.load_text_gpt4_dedup(data)
    st = eng.dedup_stats()
    assert st["passthrough_entries"] > 0, st       # witness: chunks found no slot within DD_PROBES probes
    eb, eo = eng.chunk_entries()
    w = eng.chunk_weights()
    assert nc == len(offs) and int(w.sum()) == len(offs)
    got = {}
    for j in range(len(eo)):
        k = bytes(eb[int(eo[j]): int(eo[j + 1]) if j + 1 < len(eo) else len(eb)])
        got[k] = got.get(k, 0) + int(w[j])
    assert got == {bytes(ub[int(uo[j]): int(uo[j + 1]) if j + 1 < len(uo) else len(ub)]): int(uw[j]) for j in range(len(uo))}
    n = 150
    wp, wc, _ = oracle.c_train(ub.astype(np.int32), uo, n, weights=uw)
    p, c, d = eng.train(n)
    assert d == len(wp) and np.array_equal(p, wp) and np.array_equal(c, wc)
    eng.close()


def _stats_dict(pairs, counts):
    return {(int(a), int(b)): int(c) for (a, b), c in zip(pairs.tolist(), counts.tolist())}


def test_b5_pair_table_clusters_ties_and_growth():
    """Two-token chunks whose keys share the last two home slots of a 2^10-slot pair table (chains wrap to slot 0), every
    cluster pair equally often (ties across the cluster: k_find_first looks each one up), and three-token chunks whose
    merges insert new pairs until the table grows mid-run (k_rehash moves the wrapped clusters)."""
    from minbpe_b200 import engine as E
    log2 = 10
    mask = (1 << log2) - 1
    hi = H.pair_cluster(14, mask, mask, lo=256, hi=1 << 16, seed=1)
    lo = H.pair_cluster(14, mask, mask - 1, lo=256, hi=1 << 16, seed=2, exclude=hi)
    rng = np.random.default_rng(10)
    chunks = [list(p) for p in hi + lo] * 40
    tails = rng.integers(256, 256 + 300, len(chunks) // 2)
    chunks += [list(hi[j % len(hi)]) + [int(t)] for j, t in enumerate(tails)]
    order = rng.permutation(len(chunks))
    chunks = [chunks[int(j)] for j in order]
    ids = np.asarray([x for c in chunks for x in c], dtype=np.int32)
    offs = np.zeros(len(chunks), dtype=np.uint64)
    offs[1:] = np.cumsum([len(c) for c in chunks[:-1]])
    eng = _engine()
    eng.set_option(E.OPT_TABLE_LOG2, log2)
    eng.set_option(E.OPT_BATCH, 7)
    eng.load_ids(ids, offs)
    p, c = eng.get_stats()
    wp, wc = oracle.c_get_stats(ids, offs)
    assert np.array_equal(p, wp) and np.array_equal(c, wc)
    n, k = 60, 25
    first = 1 << 16
    wp, wc, _ = oracle.c_train(ids, offs, n, first_idx=first)
    p, c, d = eng.train(k, first_idx=first)
    assert d == k and np.array_equal(p, wp[:k]) and np.array_equal(c, wc[:k])
    _, _, _, fin_k = oracle.c_train(ids, offs, k, first_idx=first, want_final=True)
    fo = _final_offsets(chunks, wp[:k], first)
    assert eng.debug_table() == _stats_dict(*oracle.c_get_stats(fin_k, fo))
    p2, c2, d2 = eng.train(n - k, first_idx=first + k)
    assert d2 == n - k and np.array_equal(p2, wp[k:]) and np.array_equal(c2, wc[k:])
    assert eng.timing()["table_slots"] > (1 << log2)           # witness: the table grew mid-run
    eng.close()


def _final_offsets(chunks, merges, first):
    """chunk offsets of the stream after applying `merges` (ids first, first + 1, ...) to every chunk in rank order"""
    offs, pos = [], 0
    for c in chunks:
        c = list(c)
        for r, (a, b) in enumerate(merges.tolist()):
            out, i = [], 0
            while i < len(c):
                if i + 1 < len(c) and c[i] == a and c[i + 1] == b:
                    out.append(first + r)
                    i += 2
                else:
                    out.append(c[i])
                    i += 1
            c = out
        offs.append(pos)
        pos += len(c)
    return np.asarray(offs, dtype=np.uint64)


def test_b6_hist_hash_overflow():
    pairs = H.byte_pairs_in_slot(H.HH_SLOTS - 1, H.hist_hash_home)[:12]
    assert len(pairs) >= 8
    rng = np.random.default_rng(6)
    seq = [pairs[int(i)] for i in rng.integers(0, len(pairs), 40000 if SMALL else 400000)]
    ids = np.asarray(seq, dtype=np.int32).reshape(-1)
    offs = np.arange(0, ids.size, 2, dtype=np.uint64)
    eng = _engine()
    eng.load_ids(ids, offs)
    p, c = eng.get_stats()
    wp, wc = oracle.c_get_stats(ids, offs)
    assert np.array_equal(p, wp) and np.array_equal(c, wc)
    eng.close()


def _rank_cluster_merges(mask):
    """merges whose pairs share the last two home slots of a rank table of mask + 1 slots (chains wrap to slot 0), with
    duplicated pairs inside the cluster, then merges of the new ids"""
    c1 = H.byte_pairs_in_slot(mask, lambda a, b: H.table_home(a, b, mask))
    c0 = H.byte_pairs_in_slot(mask - 1, lambda a, b: H.table_home(a, b, mask))
    rng = random.Random(8)
    base = c1[:30] + c0[:20]
    rng.shuffle(base)
    merges = base + [base[3], base[10], base[17]]     # duplicates: the later rank wins
    n = len(merges)
    for r in range(n, 200):
        merges.append((rng.randrange(256, 256 + r), rng.randrange(0, 256 + r)))
    return np.asarray(merges, dtype=np.int32), sorted({x for p in base for x in p})


def test_b8_rank_table_clusters():
    mask = 1023                                     # next_pow2(max(1024, 4 * 200)) - 1
    M, alphabet = _rank_cluster_merges(mask)
    rng = np.random.default_rng(9)
    chunks = [bytes(rng.choice(alphabet, int(rng.integers(1, 12))).astype(np.uint8)) for _ in range(12000)]
    data, offs = _join(chunks)
    assert data.size >= MEMO_MIN
    eng = _engine()
    assert np.array_equal(eng.encode(data, offs, M), oracle.c_encode(data, offs, M))          # memo path
    k = int(np.searchsorted(offs, 8000))
    d, o = data[:int(offs[k])], offs[:k]
    assert np.array_equal(eng.encode(d, o, M), oracle.c_encode(d, o, M))                      # general path
    long = bytes(rng.choice(alphabet, 3000).astype(np.uint8))
    want = oracle.c_encode(np.frombuffer(long, dtype=np.uint8), None, M)
    assert want.size > 64                                                                     # long path
    assert np.array_equal(eng.encode(long, None, M), want)
    eng.close()


@pytest.mark.parametrize("kernel", [2, 1])
def test_b7_hist_dense_overflow(kernel):
    """Byte pairs sharing one home slot of k_hist_dense's shared table (8 probes, then the dense global counters), as
    2-byte chunks; kernel 1 is the packed histogram, which does not hash (same answer)."""
    from minbpe_b200 import engine as E
    pairs = H.byte_pairs_in_slot(100, H.hist_dense_home)[:12]
    assert len(pairs) >= 10
    rng = np.random.default_rng(7)
    weights = rng.integers(1, 6, len(pairs))
    seq = [pairs[int(i)] for i in rng.choice(len(pairs), 30000 if SMALL else 300000, p=weights / weights.sum())]
    data = np.asarray(seq, dtype=np.uint8).reshape(-1)
    offs = np.arange(0, data.size, 2, dtype=np.uint64)
    eng = _engine()
    eng.set_option(E.OPT_HIST_KERNEL, kernel)
    eng.load_stream(data, offs)
    p, c, d = eng.train(1)
    wp, wc, wd, fin = oracle.c_train(data.astype(np.int32), offs, 1, want_final=True)
    assert d == wd == 1 and np.array_equal(p, wp) and np.array_equal(c, wc)
    assert eng.timing()["hist_kernel"] == kernel
    fo = _final_offsets([tuple(x) for x in seq], wp, 256)
    assert eng.debug_table() == _stats_dict(*oracle.c_get_stats(fin, fo))
    eng.close()
