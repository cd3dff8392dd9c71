"""
Sharded BPE training: one process per GPU, torch.distributed for the plumbing (NCCL over
NVLink/NVSwitch on GPUs, gloo in the CPU tests).

The corpus is cut into contiguous byte ranges at chunk starts (regex chunks never interact,
regex.py:51-54,60), rank r holding the r-th range, so rank order = text order.  Every rank keeps an
identical copy of the global pair-count table; per merge iteration the ranks exchange

  * one int64 reduced with MIN  — the arg-max candidate.  The max count is the same everywhere
    (same table); a tie is broken like the reference (first occurrence in the stream, basic.py:35)
    = the candidate of the lowest rank that sees one of the tied pairs, each rank offering the
    tied pair that occurs first in its own shard.  word = rank << 58 | p0 << 29 | p1.
  * the statistics delta vector (2V+1 uint64: L[x], R[x], ZZ — DESIGN.md) reduced with SUM.

`ShardedTrainer` only sequences these steps; the work is in the engine's step API
(include/b200bpe.h "step-wise training").  Tests drive the same class over gloo with a CPU
stand-in engine built on the oracle (tests/test_dist_gloo.py).
"""
import hashlib
import os

import numpy as np
import torch
import torch.distributed as dist

CAND_NONE = (1 << 63) - 1


def shard_chunks(n_bytes, offsets, rank, world):
    """Contiguous chunk range of rank `rank`: (byte_lo, byte_hi, chunk_lo, chunk_hi), balanced by
    bytes, cut only at chunk starts."""
    offsets = np.asarray(offsets, dtype=np.uint64)
    k = len(offsets)
    cuts = [int(np.searchsorted(offsets, n_bytes * r // world, side="left")) for r in range(world + 1)]
    cuts[0], cuts[-1] = 0, k
    lo, hi = cuts[rank], cuts[rank + 1]
    byte_lo = int(offsets[lo]) if lo < k else n_bytes
    byte_hi = int(offsets[hi]) if hi < k else n_bytes
    return byte_lo, byte_hi, lo, hi


def first_safe_cut(window):
    """Smallest p >= 1 with window[p-1] an ASCII letter and window[p] == U+0020, or -1.  Such a point is a chunk
    boundary of the GPT-2/GPT-4/o200k split patterns whatever surrounds it (SURVEY.md §8e, DESIGN.md §17): no alternative matches a
    letter followed by a space inside one chunk, and the patterns have no look-behind, so
    findall(left) + findall(right) == findall(whole)."""
    w = np.asarray(window, dtype=np.uint8)
    if w.size < 2:
        return -1
    prev = w[:-1]
    letter = ((prev >= 65) & (prev <= 90)) | ((prev >= 97) & (prev <= 122))
    hit = np.flatnonzero(letter & (w[1:] == 32))
    return int(hit[0]) + 1 if hit.size else -1


def shard_byte_range(n_bytes, rank, world, fetch, window=1 << 20, empty_tail=False, specials=None):
    """Byte range [lo, hi) of rank `rank`: the r-th of `world` equal parts of the text, both ends moved forward to
    the next provable chunk boundary (first_safe_cut).  fetch(lo, hi) returns the text bytes [lo, hi) as uint8
    (a slice of an mmap, a generated block, ...).  Rank order = text order.  empty_tail=True: a cut with no boundary
    between it and the end of the text moves to the end of the text (the end is a boundary too), so the ranks after it get
    empty ranges instead of a ValueError; for callers that handle an empty range (count_file_shard).  specials: [utf-8
    bytes, ...] of special tokens; a cut never falls strictly inside an occurrence of one, so every rank sees the
    occurrences re.split reports in the whole text."""
    by_len = {}                                         # length -> the specials of that length
    for t in specials or ():
        by_len.setdefault(len(t), set()).add(bytes(t))
    back = max(by_len, default=0)                       # an occurrence that covers a cut starts less than this before it

    def inside_special(raw, p):
        """does the cut between bytes p-1 and p fall strictly inside an occurrence of a special token?  One set lookup per
        (length, start), whatever the number of specials."""
        return any(raw[p - j: p - j + n] in toks for n, toks in by_len.items() for j in range(1, n) if p - j >= 0)

    def safe(window_bytes, base):
        """first letter+space cut at or after window_bytes[base] that does not lie inside an occurrence of a special token,
        or -1"""
        w = np.asarray(window_bytes, dtype=np.uint8)
        raw = w.tobytes()
        while True:
            p = first_safe_cut(w[base:])
            if p < 0:
                return -1
            p += base
            if not inside_special(raw, p):
                return p
            base = p

    def cut(r):
        if r <= 0:
            return 0
        if r >= world:
            return n_bytes
        lo = n_bytes * r // world
        w0 = max(0, lo - back)                          # the window starts early enough to see a special that straddles `lo`
        p = safe(fetch(w0, min(n_bytes, lo + window)), lo - w0)
        if p < 0 and empty_tail and lo + window >= n_bytes:
            return n_bytes
        if p < 0:
            raise ValueError(f"no letter+space cut point in the {window} bytes after offset {lo}: cannot shard this text")
        return w0 + p
    return cut(rank), cut(rank + 1)


class GpuStepEngine:
    """Adapter: minbpe_b200.engine.Engine step API over torch CUDA tensors on the current stream."""

    def __init__(self, engine, device):
        self.e = engine
        self.device = torch.device("cuda", device)
        # a dedicated torch stream shared by our kernels and (through torch's stream semantics) the
        # NCCL collectives: the legacy default stream has handle 0, which bpe_set_stream reads as
        # "use the handle's own stream" and which would leave kernels and collectives unordered
        self.stream = torch.cuda.Stream(device=self.device)
        self.e.set_stream(self.stream.cuda_stream)

    def stream_ctx(self):
        return torch.cuda.stream(self.stream)

    def new_i64(self, n):
        return torch.zeros(n, dtype=torch.int64, device=self.device)

    def begin(self, dense):
        self.e.step_begin(dense.data_ptr())

    def table(self, dense, num_merges, first_idx, poll_every):
        self.e.step_table(dense.data_ptr(), num_merges, first_idx, poll_every)
        return self.e.step_delta_len()

    def select(self, cand, rank):
        self.e.step_select(cand.data_ptr(), rank)

    def merge(self, cand, delta):
        self.e.step_merge(cand.data_ptr(), delta.data_ptr())

    def apply(self, delta):
        self.e.step_apply(delta.data_ptr())

    def poll(self):
        return self.e.step_poll()

    def result(self, cap):
        return self.e.step_result(cap)

    # ---- exchanges over NVLink peer memory (k_xchg.cuh): no host call per merge ----
    def xchg_setup(self, world, rank, vocab_cap, group=None):
        """Create this rank's exchange block (or keep the one of the same shape), all-gather the CUDA IPC handles
        through torch.distributed and map the peers' blocks.  Returns True when EVERY rank succeeded (the ranks agree
        on the answer: a local failure — no peer access, IPC refused — is exchanged, never raised between two
        collectives); on False the caller falls back to the collective exchange."""
        from .engine import EngineError
        key = (world, rank, vocab_cap)
        if getattr(self, "_xchg_key", None) == key:
            return True
        self._xchg_key = None
        if world > 1:
            try:
                self.e.xchg_detach()            # unmap the peers' old blocks ...
            except EngineError:
                pass
            torch.cuda.synchronize(self.device)
            dist.barrier(group=group)           # ... everywhere, before any rank frees its own
        ok, mine = 1, torch.zeros(64, dtype=torch.uint8, device=self.device)
        try:
            mine = torch.from_numpy(self.e.xchg_create(world, rank, vocab_cap)).to(self.device)
        except EngineError as ex:
            ok, self.xchg_error = 0, str(ex)
        if world > 1:
            parts = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(parts, mine, group=group)
            flag = torch.tensor([ok], device=self.device)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
            if int(flag.item()):
                try:
                    self.e.xchg_attach(torch.stack(parts).cpu().numpy())
                except EngineError as ex:
                    ok, self.xchg_error = 0, str(ex)
            else:
                ok = 0
            flag = torch.tensor([ok], device=self.device)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)   # also: every rank has mapped every block before the first flag is written
            ok = int(flag.item())
            if ok:      # handshake kernel: flags pushed to and magic words pulled from every peer, short timeout
                try:
                    ok = int(self.e.xchg_probe(3000))
                except EngineError as ex:
                    ok, self.xchg_error = 0, str(ex)
                if not ok and not getattr(self, "xchg_error", None):
                    self.xchg_error = "peer-memory handshake (bpe_xchg_probe) failed or timed out"
                flag = torch.tensor([ok], device=self.device)
                dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
                ok = int(flag.item())
        if ok:
            self._xchg_key = key
        return bool(ok)

    def sync_ranks(self, group=None):
        """Every rank's queued work is done (device sync), on every rank (barrier)."""
        torch.cuda.synchronize(self.device)
        dist.barrier(group=group)

    def fused(self, n_iters):
        self.e.step_fused(n_iters)


class ShardedTrainer:
    """regex.py:49-63 over `world` shards.  `eng` is a step engine whose stream already holds this
    rank's shard (Engine.load_stream)."""

    def __init__(self, eng, rank=None, world=None, group=None, poll_every=16, exchange=None):
        """exchange: "collective" = two torch.distributed all-reduces per merge (NCCL / gloo) — the default;
        "p2p" = our kernels over NVLink peer memory (k_xchg.cuh), opt-in (argument, or BPE_EXCHANGE=p2p) until it has run on
        multi-GPU hardware (DESIGN.md §5)."""
        self.eng, self.group = eng, group
        self.rank = dist.get_rank(group) if rank is None else rank
        self.world = dist.get_world_size(group) if world is None else world
        self.poll_every = poll_every
        want = exchange or os.environ.get("BPE_EXCHANGE", "collective")
        if want not in ("p2p", "collective"):
            raise ValueError(f"exchange must be 'p2p' or 'collective', not {want!r}")
        self.exchange = want if hasattr(eng, "xchg_setup") else "collective"

    def _allreduce(self, t, op):
        if self.world > 1:
            dist.all_reduce(t, op=op, group=self.group)

    def _ctx(self):
        import contextlib
        return self.eng.stream_ctx() if hasattr(self.eng, "stream_ctx") else contextlib.nullcontext()

    def prepare(self, num_merges, first_idx=256):
        """Iteration-0 statistics: local histograms, SUM across ranks, identical tables."""
        self.num_merges, self.first_idx = num_merges, first_idx
        with self._ctx():
            if self.exchange == "p2p" and not self.eng.xchg_setup(self.world, self.rank, first_idx + num_merges, self.group):
                self.exchange = "collective"     # agreed by all ranks (no peer access / IPC refused): NCCL all-reduces instead
                self.exchange_fallback = getattr(self.eng, "xchg_error", "a peer rank could not set up the exchange block")
            if self.exchange == "p2p" and self.world > 1:
                self.eng.sync_ranks(self.group)   # the previous run's last round may still be read by a slower peer
            dense = self.eng.new_i64(65536)
            self.eng.begin(dense)
            self._allreduce(dense, dist.ReduceOp.SUM)     # the one collective of the run (512 KB, iteration 0)
            n_delta = self.eng.table(dense, num_merges, first_idx, self.poll_every)
            if self.exchange != "p2p":
                self.cand = self.eng.new_i64(2)
                self.delta = self.eng.new_i64(n_delta)
        self.done = 0

    def run(self, num_steps=None):
        """Enqueue merge iterations (all of them by default); returns (iterations done, exhausted)."""
        target = self.num_merges if num_steps is None else min(self.num_merges, self.done + num_steps)
        exhausted = False
        with self._ctx():
            while self.done < target and not exhausted:
                k = min(self.poll_every, target - self.done)
                if self.exchange == "p2p":
                    self.eng.fused(k)
                    self.done, exhausted = self.eng.poll()
                    continue
                for _ in range(k):
                    self.eng.select(self.cand, self.rank)
                    self._allreduce(self.cand[:1], dist.ReduceOp.MIN)
                    self.eng.merge(self.cand, self.delta)
                    self._allreduce(self.delta, dist.ReduceOp.SUM)
                    self.eng.apply(self.delta)
                self.done, exhausted = self.eng.poll()
        return self.done, exhausted

    def result(self):
        return self.eng.result(self.num_merges)


def train_sharded(engine, device, data, offsets, num_merges, first_idx=256, group=None, poll_every=16, exchange=None):
    """Convenience: every rank passes the FULL corpus description (bytes + chunk offsets); the rank's
    shard is cut out, uploaded and trained.  Returns (pairs, counts, n_done)."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    raw = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    blo, bhi, clo, chi = shard_chunks(raw.size, offsets, rank, world)
    local_offs = (np.asarray(offsets[clo:chi], dtype=np.uint64) - np.uint64(blo))
    engine.load_stream(raw[blo:bhi], local_offs if len(local_offs) else None)
    tr = ShardedTrainer(GpuStepEngine(engine, device), rank, world, group, poll_every, exchange)
    tr.prepare(num_merges, first_idx)
    tr.run()
    return tr.result()


def train_file(engine, device, path, num_merges, first_idx=256, group=None, poll_every=16, exchange=None):
    """regex.py:36-66 for a text FILE that may be far larger than one GPU call: every rank maps the file, takes
    its byte range (shard_byte_range: cuts at letter+space), uploads it — bpe_load_text_gpt4 splits it on the device
    in pieces — and the ranks train together (ShardedTrainer).  Without an initialised process group (or with one
    rank) the whole file goes to this GPU and the device-driven loop (bpe_train) runs.  The split pattern is the engine's
    current one (BPE_OPT_SPLIT_PATTERN: GPT-4 by default, GPT-2 selectable).
    Returns (pairs, counts, n_done), identical on every rank."""
    size = os.path.getsize(path)
    mm = np.memmap(path, dtype=np.uint8, mode="r") if size else np.zeros(0, dtype=np.uint8)
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    if world == 1:
        engine.load_text_gpt4(mm)
        return engine.train(num_merges, first_idx)
    rank = dist.get_rank(group)
    lo, hi = shard_byte_range(size, rank, world, lambda a, b: mm[a:b])
    engine.load_text_gpt4(mm[lo:hi])
    tr = ShardedTrainer(GpuStepEngine(engine, device), rank, world, group, poll_every, exchange)
    tr.prepare(num_merges, first_idx)
    tr.run()
    return tr.result()


def count_file_shard(engine, path, rank, world, specials=None):
    """The distinct chunks of rank `rank`'s byte range of a text file (shard_byte_range), counted on this rank's GPU
    (Engine.load_text_gpt4_dedup, the engine's split pattern) and read back: -> (entry bytes uint8, entry offsets uint64,
    weights uint64, chunks of the range).  The entries obey DESIGN.md §14's rule for the range; an empty range gives empty
    arrays.  specials: [utf-8 bytes, ...] of special tokens whose occurrences are left out (DESIGN.md §18); the range
    never cuts one.  Needs no process group: a test can play every rank in one process."""
    size = os.path.getsize(path)
    mm = np.memmap(path, dtype=np.uint8, mode="r") if size else np.zeros(0, dtype=np.uint8)
    lo, hi = shard_byte_range(size, rank, world, lambda a, b: mm[a:b], empty_tail=True, specials=specials)
    if hi <= lo:
        return np.zeros(0, np.uint8), np.zeros(0, np.uint64), np.zeros(0, np.uint64), 0
    chunks, _ = engine.load_text_gpt4_dedup(mm[lo:hi], specials)
    del mm
    data, offsets = engine.chunk_entries()
    return data, offsets, engine.chunk_weights(), int(chunks)


def load_merged_shards(engine, parts):
    """Concatenate the ranks' count_file_shard results in rank order (= text order), rebase the offsets and merge the
    entries of equal bytes on the GPU (Engine.load_chunks_weighted_dedup): the weighted stream of the whole file is then
    loaded.  -> entries kept."""
    datas = [np.asarray(p[0], dtype=np.uint8) for p in parts]
    base = np.cumsum([0] + [d.size for d in datas[:-1]], dtype=np.uint64)
    offsets = np.concatenate([np.asarray(p[1], dtype=np.uint64) + b for p, b in zip(parts, base)] or [np.zeros(0, np.uint64)])
    weights = np.concatenate([np.asarray(p[2], dtype=np.uint64) for p in parts] or [np.zeros(0, np.uint64)])
    data = np.concatenate(datas) if datas else np.zeros(0, np.uint8)
    return engine.load_chunks_weighted_dedup(data, offsets, weights)


def _run_digest(pairs, counts, done):
    h = hashlib.sha256(np.ascontiguousarray(pairs, dtype=np.int32).tobytes() + np.ascontiguousarray(counts, dtype=np.int64).tobytes()
                       + int(done).to_bytes(8, "little"))
    return int.from_bytes(h.digest()[:8], "little") & ((1 << 63) - 1)


def train_file_dedup(engine, path, num_merges, first_idx=256, group=None, specials=None):
    """regex.py:36-66 for a text FILE on every rank of a process group, trained on its distinct chunks: every rank counts
    the distinct chunks of its byte range (count_file_shard), the ranks exchange their entries once (one all-gather), every
    rank merges them into the weighted stream of the whole file on its GPU (load_merged_shards) and runs the weighted loop
    there.  No exchange per merge.  Afterwards the ranks compare a 63-bit digest of their merges and counts (all-reduce MIN
    and MAX) and raise RuntimeError if they differ.  Works over gloo and NCCL groups.  specials: as count_file_shard.
    Returns (pairs, counts, n_done), identical on every rank."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    part = count_file_shard(engine, path, rank, world, specials)
    parts = [None] * world
    dist.all_gather_object(parts, part, group=group)
    load_merged_shards(engine, parts)
    del parts, part
    pairs, counts, done = engine.train(num_merges, first_idx)
    dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    d = _run_digest(pairs, counts, done)
    lo = torch.tensor([d], dtype=torch.int64, device=dev)
    hi = lo.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=group)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=group)
    if int(lo.item()) != d or int(hi.item()) != d:
        raise RuntimeError(f"train_file_dedup: rank {rank} trained different merges than another rank")
    return pairs, counts, done


def encode_sharded(engine, data, offsets, merges, byte_perm=None, group=None, gather=False, rank=None, world=None):
    """regex.py:111-121 over `world` GPUs: chunks are independent, so encode needs no exchange at all —
    every rank encodes its contiguous chunk range (replicas over byte-range shards).  Returns this
    rank's ids; with gather=True rank 0 also gets the concatenation in text order (others: None).
    rank / world default to the process group's."""
    rank = dist.get_rank(group) if rank is None else rank
    world = dist.get_world_size(group) if world is None else world
    raw = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    blo, bhi, clo, chi = shard_chunks(raw.size, offsets, rank, world)
    local_offs = np.asarray(offsets[clo:chi], dtype=np.uint64) - np.uint64(blo)
    ids = engine.encode(raw[blo:bhi], local_offs if len(local_offs) else None, merges, byte_perm) if bhi > blo else np.zeros(0, np.int32)
    if not gather:
        return ids
    parts = [None] * world if rank == 0 else None
    dist.gather_object(ids, parts, dst=0, group=group)
    return np.concatenate(parts) if rank == 0 else None


def encode_file(engine, path, merges, byte_perm=None, specials=None, group=None, gather=False, rank=None, world=None):
    """regex.py:111-121 (with `specials`: regex.py:152-163) for a text FILE over `world` GPUs: every rank maps the file,
    takes its byte range (shard_byte_range: cut where a letter is followed by a space — a chunk boundary whatever
    surrounds it — and never inside a special token) and runs the fused split + encode on it
    (Engine.encode_text_gpt4); chunks are independent, so there is no exchange.  Returns this rank's ids; with
    gather=True rank 0 also gets the concatenation in text order (others: None).  The split pattern is the engine's
    current one (BPE_OPT_SPLIT_PATTERN: GPT-4 by default)."""
    if rank is None or world is None:
        if dist.is_available() and dist.is_initialized():
            rank, world = dist.get_rank(group), dist.get_world_size(group)
        else:
            rank, world = 0, 1
    size = os.path.getsize(path)
    mm = np.memmap(path, dtype=np.uint8, mode="r") if size else np.zeros(0, dtype=np.uint8)
    lo, hi = shard_byte_range(size, rank, world, lambda a, b: mm[a:b], specials=[t for t, _ in (specials or [])])
    ids = engine.encode_text_gpt4(mm[lo:hi], merges, byte_perm, specials=specials) if hi > lo else np.zeros(0, np.int32)
    if not gather:
        return ids
    parts = [None] * world if rank == 0 else None
    dist.gather_object(ids, parts, dst=0, group=group)
    return np.concatenate(parts) if rank == 0 else None
