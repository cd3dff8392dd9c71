"""GPU: training on the distinct chunks of a file across the ranks of a process group (DESIGN.md §14) — every rank counts
the distinct chunks of its byte range (dist.count_file_shard), the ranks' entries are merged on the device
(bpe_load_chunks_weighted_dedup: k_dd_count<true>, k_dd_keep, k_dd_emit, k_dd_weights<true>) and read back
(bpe_read_chunk_entries).  The merged stream must equal the whole-file loader's, training on it must give the
oracle's merges, and RegexTokenizer.train_from_file(dedup=True) under a real gloo process group must give every rank the
single-process result.  Ranks are played one after another in this process wherever no collective is needed."""
import hashlib
import os
import socket
import sys

import numpy as np
import pytest
import regex

import oracle
from conftest import ROOT

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))      # set by the CPU SIMT emulator runs: smaller corpus, fewer merges

GPT4 = regex.compile(
    r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+""")
GPT2 = regex.compile(r"""'(?:[sdmt]|ll|ve|re)| ?\p{L}+| ?\p{N}+| ?[^\s\p{L}\p{N}]+|\s+(?!\S)|\s+""")
RUNS = " zz zz zzzz aaaa aaaa" + " " * 70 + "b" * 60 + " zz"   # pairs (a,a), and chunks longer than 48 bytes
KEY_MAX = 48                                                   # DD_KEY_MAX of k_dedup.cuh


def random_words(seed, pool, draws):
    """Lowercase words of 3..10 random letters drawn with replacement from a pool of `pool` words: about
    pool * (1 - exp(-draws / pool)) distinct chunks, most of them seen by several ranks."""
    rng = np.random.default_rng(seed)
    letters = rng.integers(97, 123, size=(pool, 10), dtype=np.uint8)
    lens = rng.integers(3, 11, size=pool)
    words = [letters[i, : lens[i]].tobytes().decode() for i in range(pool)]
    pick = rng.integers(0, pool, size=draws)
    return " ".join(words[i] for i in pick) + "\n"


def corpora(taylorswift):
    from minbpe_b200.synth import generate
    synth = generate(1337, (256 << 10) if SMALL else (2 << 20)).tobytes().decode("utf-8")
    words = random_words(11, 4000, 12000) if SMALL else random_words(11, 150000, 300000)
    return {"taylorswift": taylorswift + RUNS, "synth": synth + RUNS, "words": words}


def _engine(pattern=0):
    from minbpe_b200 import engine as E
    eng = E.Engine(0)
    eng.set_option(E.OPT_BATCH, 64)                 # more batch boundaries: re-packing happens there
    eng.set_option(E.OPT_SPLIT_PATTERN, pattern)
    return eng


def _write(tmp_path, name, text):
    path = str(tmp_path / f"{name}.txt")
    with open(path, "wb") as f:
        f.write(text.encode("utf-8"))
    return path


def _play_ranks(eng, path, world):
    """every rank's count_file_shard, one after another on one engine"""
    from minbpe_b200.dist import count_file_shard
    return [count_file_shard(eng, path, r, world) for r in range(world)]


def _state(eng):
    b, o = eng.chunk_entries()
    return eng.read_stream(), b, o, eng.chunk_weights(), eng.dedup_stats()


def _host_merge(data, offs, weights):
    """The merge as the host would do it with an unbounded table: every entry of <= 48 bytes folds into the first entry
    with its bytes; longer entries stay with their own weights."""
    raw = bytes(data)
    ends = list(np.asarray(offs, dtype=np.int64)[1:].tolist()) + [len(raw)]
    first, ents, wts = {}, [], []
    for s, e, w in zip(np.asarray(offs, dtype=np.int64).tolist(), ends, np.asarray(weights).tolist()):
        ch = raw[s:e]
        if len(ch) <= KEY_MAX:
            if ch in first:
                wts[first[ch]] += int(w)
                continue
            first[ch] = len(ents)
        ents.append(ch)
        wts.append(int(w))
    lens = np.fromiter(map(len, ents), dtype=np.int64, count=len(ents))
    eo = np.zeros(len(ents), dtype=np.uint64)
    eo[1:] = np.cumsum(lens[:-1])
    return np.frombuffer(b"".join(ents), dtype=np.uint8), eo, np.asarray(wts, dtype=np.uint64)


@pytest.mark.parametrize("pattern", [0, 1])
@pytest.mark.parametrize("name", ["taylorswift", "synth", "words"])
def test_merged_stream_equals_the_whole_file_loader(name, pattern, taylorswift, tmp_path):
    """count_file_shard on every rank + load_merged_shards == one load_text_gpt4_dedup of the whole file: same bytes, chunk
    marks, weights and chunk count, for world 2, 3 and 8."""
    from minbpe_b200.dist import load_merged_shards
    text = corpora(taylorswift)[name]
    path = _write(tmp_path, name, text)
    whole = _engine(pattern)
    nc, ne = whole.load_text_gpt4_dedup(np.fromfile(path, dtype=np.uint8))
    ids, wb, wo, ww, wst = _state(whole)
    assert wst["passthrough_entries"] == (wst["entries"] - wst["table_entries"])
    if name == "words":
        assert wst["entries"] >= (3000 if SMALL else 100000)       # high cardinality
    whole.close()
    eng = _engine(pattern)
    for world in (2, 3, 8):
        parts = _play_ranks(eng, path, world)
        assert sum(p[3] for p in parts) == nc
        assert sum(int(p[2].sum()) for p in parts) == nc
        n = load_merged_shards(eng, parts)
        got_ids, gb, go, gw, st = _state(eng)
        assert n == ne and st["entries"] == ne, world
        assert np.array_equal(got_ids, ids) and np.array_equal(gb, wb) and np.array_equal(go, wo), world
        assert np.array_equal(gw, ww), world
        assert st["text_chunks"] == nc and st["pieces"] == 0 and st["stream_bytes"] == len(wb)
        assert st["table_entries"] + st["passthrough_entries"] == ne
        assert st["slots_used"] == wst["slots_used"]
    eng.close()


def test_more_ranks_than_cut_points(tmp_path):
    """A text with two letter+space cut points over 8 ranks: most ranks get an empty range and empty arrays."""
    from minbpe_b200.dist import load_merged_shards
    text = "alpha beta gamma" + "!" * 40
    path = _write(tmp_path, "few", text)
    whole = _engine()
    nc, ne = whole.load_text_gpt4_dedup(text.encode())
    ref = _state(whole)
    whole.close()
    eng = _engine()
    parts = _play_ranks(eng, path, 8)
    empty = [p for p in parts if len(p[0]) == 0]
    assert len(empty) >= 5 and all(len(p[1]) == len(p[2]) == 0 and p[3] == 0 for p in empty)
    assert sum(p[3] for p in parts) == nc
    assert load_merged_shards(eng, parts) == ne
    got = _state(eng)
    for a, b in zip(ref[:4], got[:4]):
        assert np.array_equal(a, b)
    # an empty file: every rank empty, an empty weighted stream
    path = _write(tmp_path, "empty", "")
    parts = _play_ranks(eng, path, 3)
    assert load_merged_shards(eng, parts) == 0
    assert eng.stream_len() == 0 and len(eng.chunk_weights()) == 0 and eng.dedup_stats()["text_chunks"] == 0
    eng.close()


@pytest.mark.parametrize("name", ["taylorswift", "synth"])
def test_training_on_the_merged_stream_equals_the_oracle(name, taylorswift, tmp_path):
    """Batched passes, pairs (a,a), re-packing (OPT_BATCH 64) and a second train call on the merged stream of 3 ranks:
    merges and counts equal to the oracle's weighted loop on the whole text's distinct chunks."""
    from minbpe_b200.dist import load_merged_shards
    text = corpora(taylorswift)[name]
    path = _write(tmp_path, name, text)
    merges = 400 if SMALL else 1500
    data, offs = oracle.split_to_stream(text, GPT4)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges + 100, weights=uw)
    eng = _engine()
    load_merged_shards(eng, _play_ranks(eng, path, 3))
    _, gb, go, gw, _ = _state(eng)
    assert np.array_equal(gb, ub) and np.array_equal(go, uo) and np.array_equal(gw, np.asarray(uw, dtype=np.uint64))
    p, c, d = eng.train(merges)
    assert d == merges and np.array_equal(p, wp[:merges]) and np.array_equal(c, wc[:merges])
    assert any(a == b for a, b in p.tolist())       # the (a,a) path ran
    assert eng.timing()["tokens_in"] > 0
    p2, c2, d2 = eng.train(100, first_idx=256 + merges)
    assert d2 == 100 and np.array_equal(p2, wp[merges:]) and np.array_equal(c2, wc[merges:])
    eng.close()


def _split_entries(raw, offs, rng, p_split):
    """Entries obeying the rule in which a distinct chunk may be split over several entries (as in test_gpu_zz_dedup.py)."""
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
    return np.frombuffer(b"".join(entries), dtype=np.uint8), eo, np.asarray(weights, dtype=np.uint64)


def test_host_built_parts(taylorswift):
    """Parts in which chunks are split over several entries, inside one part and across parts; weights of 2^33 and more;
    and one part that is already distinct, which must round-trip unchanged."""
    from minbpe_b200.dist import load_merged_shards
    text = taylorswift + RUNS + " " * 200 + "x" * 300 + RUNS
    data, offs = oracle.split_to_stream(text, GPT4)
    raw = bytes(data)
    rng = np.random.default_rng(5)
    cuts = [0, len(offs) // 4, len(offs) // 2, len(offs)]
    parts = []
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        sub_end = int(offs[hi]) if hi < len(offs) else len(raw)
        sub = raw[int(offs[lo]):sub_end]
        b, o, w = _split_entries(sub, (offs[lo:hi] - offs[lo]).astype(np.uint64), rng, 0.3)
        parts.append((b, o, w, int(w.sum())))
    cat_b = np.concatenate([p[0] for p in parts])
    base = np.cumsum([0] + [len(p[0]) for p in parts[:-1]]).astype(np.uint64)
    cat_o = np.concatenate([p[1] + b for p, b in zip(parts, base)])
    cat_w = np.concatenate([p[2] for p in parts])
    hb, ho, hw = _host_merge(cat_b, cat_o, cat_w)
    eng = _engine()
    n = load_merged_shards(eng, parts)
    _, gb, go, gw, st = _state(eng)
    assert n == len(ho) < len(cat_o)
    assert np.array_equal(gb, hb) and np.array_equal(go, ho) and np.array_equal(gw, hw)
    assert int(gw.sum()) == st["text_chunks"] == len(offs)
    merges = 300 if SMALL else 1000
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges, weights=uw)
    p, c, d = eng.train(merges)
    assert d == wd == merges and np.array_equal(p, wp) and np.array_equal(c, wc)
    # weights of 2^33 and more sum exactly
    big = [(p[0], p[1], p[2] + np.uint64(1 << 33) * np.uint64(i + 1), 0) for i, p in enumerate(parts)]
    bw = np.concatenate([p[2] for p in big])
    hb2, ho2, hw2 = _host_merge(cat_b, cat_o, bw)
    load_merged_shards(eng, big)
    _, gb, go, gw, st = _state(eng)
    assert np.array_equal(go, ho2) and np.array_equal(gw, hw2) and int(gw.max()) > (1 << 34)
    assert st["text_chunks"] == int(sum(int(x) for x in bw.tolist())) == int(sum(int(x) for x in hw2.tolist()))
    # a single part that is already distinct
    ub8 = np.asarray(ub, dtype=np.uint8)
    uw64 = np.asarray(uw, dtype=np.uint64)
    assert load_merged_shards(eng, [(ub8, uo, uw64, int(uw64.sum()))]) == len(uo)
    _, gb, go, gw, st = _state(eng)
    assert np.array_equal(gb, ub8) and np.array_equal(go, uo) and np.array_equal(gw, uw64)
    assert st["text_chunks"] == len(offs)
    eng.close()


@pytest.mark.parametrize("log2", [4, 5])
def test_full_table(log2, taylorswift, tmp_path):
    """A merge table of 16 / 32 slots: most entries find no room and pass through with their own weights.  The entries
    differ from the oracle's distinct chunks, the weights still count every chunk once and the merges are the oracle's."""
    from minbpe_b200 import engine as E
    from minbpe_b200.dist import load_merged_shards
    text = taylorswift + RUNS
    path = _write(tmp_path, "ts", text)
    data, offs = oracle.split_to_stream(text, GPT4)
    ub, uo, uw = oracle.c_dedup_chunks(data, offs)
    merges = 300 if SMALL else 800
    wp, wc, wd = oracle.c_train(ub.astype(np.int32), uo, merges, weights=uw)
    eng = _engine()
    parts = _play_ranks(eng, path, 3)
    eng.set_option(E.OPT_DEDUP_LOG2, log2)
    n = load_merged_shards(eng, parts)
    st = eng.dedup_stats()
    w = eng.chunk_weights()
    assert n == len(w) > len(uo) and int(w.sum()) == len(offs) == st["text_chunks"]
    assert st["slots_used"] <= st["slots"] == 1 << log2 and st["passthrough_entries"] > 0
    p, c, d = eng.train(merges)
    assert d == wd == merges and np.array_equal(p, wp) and np.array_equal(c, wc)
    eng.close()


def _rc(fn):
    from minbpe_b200 import engine as E
    with pytest.raises(E.EngineError) as ex:
        fn()
    return regex.search(r"failed \((-?\d+)\)", str(ex.value)).group(1) if "failed (" in str(ex.value) else str(ex.value).split(":")[0]


def test_errors_and_empty_input():
    from minbpe_b200 import engine as E
    eng = _engine()
    data = b"ab ab ab cd"
    offs = np.array([0, 2, 5, 8], dtype=np.uint64)
    bad = [(offs, np.array([1, 0, 1, 1], dtype=np.uint64)),             # zero weight
           (np.array([0, 5, 2, 8], dtype=np.uint64), np.ones(4, dtype=np.uint64)),   # not increasing
           (np.array([0, 2, 2, 8], dtype=np.uint64), np.ones(4, dtype=np.uint64)),   # repeated
           (offs, np.ones(3, dtype=np.uint64)),                                       # lengths differ
           (None, np.zeros(0, dtype=np.uint64))]                                      # no offsets
    for o, w in bad:
        a = _rc(lambda: eng.load_chunks_weighted(data, o, w))
        b = _rc(lambda: eng.load_chunks_weighted_dedup(data, o, w))
        assert a == b.replace("_dedup", ""), (a, b)
    assert _rc(lambda: eng.load_chunks_weighted_dedup(b"", offs, np.ones(4, dtype=np.uint64))) == "-2"
    # chunk_entries: only on a weighted stream that no train / replay has touched
    eng.load_stream(data, offs)
    assert _rc(lambda: eng.chunk_entries()) == "-3"
    assert eng.load_chunks_weighted_dedup(data, offs, np.array([1, 2, 1, 1], dtype=np.uint64)) == 3
    b, o = eng.chunk_entries()
    assert b.tobytes() == b"ab ab cd" and o.tolist() == [0, 2, 5]
    assert eng.chunk_weights().tolist() == [1, 3, 1]
    p, c, d = eng.train(1)
    assert p.tolist() == [[97, 98]] and c.tolist() == [4]
    assert _rc(lambda: eng.chunk_entries()) == "-3"
    eng.load_chunks_weighted(data, offs, np.ones(4, dtype=np.uint64))   # bpe_load_chunks_weighted's stream reads back too
    assert eng.chunk_entries()[0].tobytes() == data
    eng.replay(np.array([[97, 98]], dtype=np.int32))
    assert _rc(lambda: eng.chunk_entries()) == "-3"
    # an empty input loads an empty weighted stream
    assert eng.load_chunks_weighted_dedup(b"", None, np.zeros(0, dtype=np.uint64)) == 0
    assert eng.stream_len() == 0 and len(eng.chunk_weights()) == 0
    b, o = eng.chunk_entries()
    assert len(b) == len(o) == 0
    st = eng.dedup_stats()
    assert st["text_chunks"] == st["entries"] == st["pieces"] == 0
    eng.close()


# ---- through RegexTokenizer under a real process group ----

def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def _rank_main(rank, world, port, backend, path, V, out_dir, q):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    device = rank if backend == "nccl" else 0
    kw = {}
    if backend == "nccl":
        torch.cuda.set_device(device)
        kw["device_id"] = torch.device("cuda", device)
    dist.init_process_group(backend, init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world, **kw)
    try:
        from minbpe_b200 import RegexTokenizer
        tok = RegexTokenizer(device=device)
        tok.train_from_file(path, V, dedup=True)
        prefix = os.path.join(out_dir, f"{backend}{world}_r{rank}")
        tok.save(prefix)
        q.put((rank, [list(p) for p in tok.merges], {k: v.hex() for k, v in tok.vocab.items()},
               _sha(prefix + ".model"), _sha(prefix + ".vocab")))
        tok.engine.close()
    finally:
        dist.destroy_process_group()


def _spawn_ranks(world, backend, path, V, out_dir):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, backend, path, V, out_dir, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        out = sorted(q.get(timeout=1800 if SMALL else 600) for _ in procs)
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0, p.exitcode
        return out
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=30)


def _single_process(path, text, V, tmp_path):
    from minbpe_b200 import RegexTokenizer
    a = RegexTokenizer(device=0)
    a.train_from_file(path, V, dedup=True)
    a.save(str(tmp_path / "single"))
    b = RegexTokenizer(device=0)
    b.train(text, V)
    assert b.merges == a.merges and b.vocab == a.vocab
    return ([list(p) for p in a.merges], {k: v.hex() for k, v in a.vocab.items()},
            _sha(str(tmp_path / "single.model")), _sha(str(tmp_path / "single.vocab")))


@pytest.mark.parametrize("world", [2, 3])
def test_train_from_file_dedup_gloo_ranks(world, taylorswift, tmp_path):
    """`world` processes over gloo, every one on cuda:0: every rank's merges, vocab and .model / .vocab files equal a
    single-process train_from_file(dedup=True) and a plain train(text)."""
    text = taylorswift + RUNS
    path = _write(tmp_path, "corpus", text)
    V = 256 + (100 if SMALL else 300)
    ref = _single_process(path, text, V, tmp_path)
    out = _spawn_ranks(world, "gloo", path, V, str(tmp_path))
    assert [o[0] for o in out] == list(range(world))
    for rank, merges, vocab, msha, vsha in out:
        assert (merges, vocab, msha, vsha) == ref, rank


def test_train_from_file_dedup_nccl_two_gpus(taylorswift, tmp_path):
    import torch
    if SMALL or not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    text = taylorswift + RUNS
    path = _write(tmp_path, "corpus", text)
    V = 256 + 300
    ref = _single_process(path, text, V, tmp_path)
    out = _spawn_ranks(2, "nccl", path, V, str(tmp_path))
    for rank, merges, vocab, msha, vsha in out:
        assert (merges, vocab, msha, vsha) == ref, rank
