"""GPU: training, encode and decode on texts just past B = 2^31 and B = 2^32 bytes, where positions, offsets and lengths
no longer fit in 32 bits (tests/beyond32.py builds the texts and their oracle from repeated blocks).  Every result is
compared exactly with the oracle: merges and counts of the plain loop (k_find_first on a tie straddling B, a pair (a,a)
packed while the stream holds more than B tokens, table growth), of the counting session (first positions of the
distinct chunks past B), with special tokens past B, the ids of encode_file block by block, the decoded text, and more
than 2^32 ids out of one encode.  Under BPE_TEST_SMALL (the SIMT emulator) B = 2^22: the plumbing and the oracle only.

Each test first checks free device memory, host memory and disk space, and skips naming the one that is short."""
import os
import shutil
import time

import numpy as np
import pytest

import beyond32 as T
from batch_model import stats, table_dict

pytestmark = pytest.mark.gpu
SMALL = bool(os.environ.get("BPE_TEST_SMALL"))
BS = [1 << 22] if SMALL else [1 << 31, 1 << 32]
P_BYTES = 4096 if SMALL else 65536
K = 64
GIB = 1 << 30


def _host_available():
    """/proc/meminfo MemAvailable, capped by the cgroup's limit - usage (as bench.py reads it)."""
    avail = None
    try:
        for ln in open("/proc/meminfo"):
            if ln.startswith("MemAvailable:"):
                avail = int(ln.split()[1]) * 1024
    except OSError:
        pass
    for lim, cur in (("/sys/fs/cgroup/memory.max", "/sys/fs/cgroup/memory.current"),
                     ("/sys/fs/cgroup/memory/memory.limit_in_bytes", "/sys/fs/cgroup/memory/memory.usage_in_bytes")):
        try:
            l = open(lim).read().strip()
            if l != "max" and int(l) < (1 << 60):
                room = int(l) - int(open(cur).read().strip())
                avail = room if avail is None else min(avail, room)
        except (OSError, ValueError):
            pass
    return avail


def _device_free():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def need(device=0, host=0, disk=0, path=None):
    """Skip (once, no retry) unless the GPU, the host and the disk under `path` have room."""
    if SMALL:
        return
    free = _device_free()
    if free < device:
        pytest.skip(f"device memory: {free / GIB:.1f} GiB free, {device / GIB:.1f} GiB needed")
    avail = _host_available()
    if avail is not None and avail < host:
        pytest.skip(f"host memory: {avail / GIB:.1f} GiB available, {host / GIB:.1f} GiB needed")
    if disk:
        d = shutil.disk_usage(path).free
        if d < disk:
            pytest.skip(f"disk space: {d / GIB:.1f} GiB free in {path}, {disk / GIB:.1f} GiB needed")


class Peak:
    """The largest device memory in use seen at the marks (cudaMemGetInfo, whatever allocates it), and the wall time."""

    def __init__(self, name):
        self.name, self.t0, self.base, self.peak = name, time.time(), 0 if SMALL else _device_free(), 0

    def mark(self):
        if not SMALL:
            self.peak = max(self.peak, self.base - _device_free())

    def report(self):
        print(f"\n[beyond32] {self.name}: peak device memory at the marks {self.peak / GIB:.2f} GiB, "
              f"wall {time.time() - self.t0:.1f} s")


@pytest.fixture(scope="module", params=BS, ids=lambda b: f"B2^{b.bit_length() - 1}")
def text(request):
    return T.Text(request.param, P_BYTES)


@pytest.fixture(scope="module")
def oracle_g4(text):
    """-> (entries, their first positions, pairs, counts) of the text under the GPT-4 pattern, no specials."""
    from minbpe_b200.tokenizer import GPT4_SPLIT_PATTERN
    d, o, w, first = T.entries(text, GPT4_SPLIT_PATTERN)
    pairs, counts, done = T.train(d, o, w, K)
    assert done == K and pairs[:3].tolist() == [[90, 90], [88, 89], [85, 86]]
    return (d, o, w), first, pairs, counts


def _file(text, tmp_path_factory):
    path = str(tmp_path_factory.getbasetemp() / f"beyond_{text.B}.txt")
    if not os.path.exists(path) or os.path.getsize(path) != text.nbytes:
        need(disk=text.nbytes + GIB, path=str(tmp_path_factory.getbasetemp()))
        text.write(path)
    return path


def _same(pairs, counts, want_pairs, want_counts):
    assert np.array_equal(np.asarray(pairs).reshape(-1, 2), want_pairs)
    if counts is not None:
        assert np.array_equal(counts, want_counts)


def test_engine_train_plain_loop(text, oracle_g4):
    """load_text_gpt4 + train(K) on the whole text with a small pair table: the merges and counts are the oracle's
    ((Z,Z) first, then (X,Y) over (U,V) by a first occurrence below B), the table grew, the stream length is the weighted
    length of the oracle's merged chunks and the pair table its weighted recount."""
    from minbpe_b200 import engine as E
    n = text.nbytes
    need(device=9 * n + 4 * GIB, host=n + 4 * GIB)
    pk = Peak("engine train")
    (d, o, w), _, pairs, counts = oracle_g4
    arr = text.array()
    eng = E.Engine(0)
    eng.set_option(E.OPT_TABLE_LOG2, 11)
    try:
        eng.load_text_gpt4(arr)
        pk.mark()
        del arr
        assert eng.stream_len() == n
        got_p, got_c, done = eng.train(K)
        pk.mark()
        tm = eng.timing()
    finally:
        eng.set_option(E.OPT_TABLE_LOG2, 0)
    assert done == K
    _same(got_p, got_c, pairs, counts)
    assert tm["table_slots"] > 1 << 11
    fin, start = T.merged_entries(d, o, w, pairs)
    assert eng.stream_len() == int(w[np.cumsum(start) - 1].sum())
    assert eng.debug_table() == table_dict(*stats(fin, start, w))
    eng.close()
    pk.report()


def test_train_from_file(text, oracle_g4, tmp_path_factory):
    """train_from_file on the text: the plain loop, dedup=True, special_tokens= (occurrences past B) and the o200k pattern
    with dedup=True all give the oracle's merges."""
    from minbpe_b200 import O200K_SPLIT_PATTERN, RegexTokenizer
    from minbpe_b200.tokenizer import GPT4_SPLIT_PATTERN
    n = text.nbytes
    need(device=9 * n + 4 * GIB, host=4 * GIB, disk=n + GIB, path=str(tmp_path_factory.getbasetemp()))
    path = _file(text, tmp_path_factory)
    pk = Peak("train_from_file")
    _, _, pairs, _ = oracle_g4
    V = 256 + K
    spec = {T.EOT: V + 5}
    d, o, w, _ = T.entries(text, GPT4_SPLIT_PATTERN, spec)
    spairs, _, _ = T.train(d, o, w, K)
    assert spairs[:3].tolist() == pairs[:3].tolist()
    d, o, w, _ = T.entries(text, O200K_SPLIT_PATTERN)
    opairs, _, _ = T.train(d, o, w, K)
    assert opairs[:3].tolist() == pairs[:3].tolist()
    for pattern, kw, want in ((None, {}, pairs), (None, {"dedup": True}, pairs), (None, {"special_tokens": spec}, spairs),
                              (O200K_SPLIT_PATTERN, {"dedup": True}, opairs)):
        tok = RegexTokenizer(pattern, device=0)
        tok.train_from_file(path, V, **kw)
        pk.mark()
        _same(list(tok.merges), None, want, None)
        assert tok.special_tokens == kw.get("special_tokens", {})
        tok.engine.close()
    pk.report()


def test_train_from_iterator(text, oracle_g4):
    """train_from_iterator with every repeat of every block as a document: the counting session's text positions pass
    B, and the merges are the oracle's, with and without special tokens."""
    from minbpe_b200 import RegexTokenizer
    from minbpe_b200.tokenizer import GPT4_SPLIT_PATTERN
    need(device=4 * GIB, host=4 * GIB)
    pk = Peak("train_from_iterator")
    _, _, pairs, _ = oracle_g4
    V = 256 + K
    spec = {T.EOT: V + 5}
    d, o, w, _ = T.entries(text, GPT4_SPLIT_PATTERN, spec)
    spairs, _, _ = T.train(d, o, w, K)
    for kw, want in (({}, pairs), ({"special_tokens": spec}, spairs)):
        tok = RegexTokenizer(device=0)
        tok.train_from_iterator(text.documents(), V, **kw)
        pk.mark()
        _same(list(tok.merges), None, want, None)
        tok.engine.close()
    pk.report()


def _check_ids(ids, text, per_block):
    """ids == every block's ids repeated, compared block by block in slabs of rows (no list, no full-size copy)."""
    pos = 0
    for want, (_, r) in zip(per_block, text.blocks):
        rows = ids[pos: pos + r * want.size].reshape(r, want.size)
        step = max(1, (1 << 26) // want.size)
        for i in range(0, r, step):
            assert (rows[i: i + step] == want).all(), (pos, i)
        pos += r * want.size
    assert pos == ids.size


def _tokenizer(pairs, specials):
    from minbpe_b200 import RegexTokenizer
    tok = RegexTokenizer(device=0)
    tok.merges = {(int(a), int(b)): 256 + i for i, (a, b) in enumerate(pairs)}
    tok.register_special_tokens(specials)
    tok.vocab = tok._build_vocab()
    return tok


def _decode_table(tok):
    table = dict(tok.vocab)
    top = max(table) + 1
    lens = np.full(top, 0xFFFFFFFF, dtype=np.uint32)
    starts = np.zeros(top, dtype=np.uint64)
    pos = 0
    for idx, b in table.items():
        starts[idx], lens[idx] = pos, len(b)
        pos += len(b)
    return np.frombuffer(b"".join(table.values()), dtype=np.uint8), starts, lens


def test_encode_file_and_decode(text, oracle_g4, tmp_path_factory):
    """encode_file with the trained merges, allowed_special "none" and "all": the ids are every block's oracle ids,
    repeated; Engine.decode of the "none" ids (more than 2^32 bytes at B = 2^32) gives the text back."""
    from minbpe_b200.tokenizer import GPT4_SPLIT_PATTERN
    n = text.nbytes
    need(device=9 * n + 4 * GIB, host=7 * n + 4 * GIB, disk=n + GIB, path=str(tmp_path_factory.getbasetemp()))
    path = _file(text, tmp_path_factory)
    pk = Peak("encode_file + decode")
    _, _, pairs, _ = oracle_g4
    spec = {T.EOT: 256 + K + 5}
    tok = _tokenizer(pairs, spec)
    ids = tok.encode_file(path, "none")
    pk.mark()
    _check_ids(ids, text, [T.encode_block(b, GPT4_SPLIT_PATTERN, pairs) for b, _ in text.blocks])
    out, bad = tok.engine.decode(ids, *_decode_table(tok))
    pk.mark()
    assert bad == -1 and len(out) == n
    del ids
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    got = np.frombuffer(out, dtype=np.uint8)
    for i in range(0, n, 1 << 30):
        assert np.array_equal(got[i: i + (1 << 30)], mm[i: i + (1 << 30)]), i
    del got, out, mm
    ids = tok.encode_file(path, "all")
    pk.mark()
    _check_ids(ids, text, [T.encode_block(b, GPT4_SPLIT_PATTERN, pairs, spec) for b, _ in text.blocks])
    del ids
    tok.engine.close()
    pk.report()


def test_more_than_2_32_ids(text):
    """encode_text_gpt4 with no merges on the whole text: one id per byte, more than 2^32 of them at B = 2^32, equal to
    the bytes."""
    from minbpe_b200 import engine as E
    n = text.nbytes
    need(device=5 * n + 6 * GIB, host=5 * n + 4 * GIB)
    pk = Peak("encode, no merges")
    arr = text.array()
    eng = E.Engine(0)
    ids = eng.encode_text_gpt4(arr, np.zeros((0, 2), dtype=np.int32))
    pk.mark()
    assert ids.size == n
    for i in range(0, n, 1 << 28):
        assert np.array_equal(ids[i: i + (1 << 28)], arr[i: i + (1 << 28)]), i
    del ids, arr
    eng.close()
    pk.report()
