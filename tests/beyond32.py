"""Texts longer than a boundary B (2^31, 2^32) whose training and encoding results are known by construction.

A text is a concatenation of repeated blocks, block_1^r_1 ‖ block_2^r_2 ‖ ...  Every block starts with U+0020 and ends
with an ASCII letter, so every block boundary is a letter followed by a space: a chunk boundary of the GPT-2, GPT-4 and
o200k patterns (DESIGN.md §5, §17; dist.shard_byte_range cuts there).  The chunks of the text are therefore the chunks of
every block, r_i times each, and the distinct chunks in first-occurrence order, their counts and their first text
positions follow from the blocks' own `regex` split, which is a few KiB per block.  No gigabyte is ever split on the host.

The blocks are chosen so that a position or a length truncated to 32 bits (or read as signed) changes the answer:

* P^r: lowercase words, digits, punctuation, newlines and non-ASCII letters; it fills the text up to just below B.
* X^m = (" " + "XY" * 64)^m starts just below B and ends past it; U^m = (" " + "UV" * 64)^m follows at B + p.  (X,Y) and
  (U,V) have equal counts, above every other pair but (Z,Z), and the alphabets are disjoint from P's.  The first
  occurrence of (X,Y) is at B - eps, the first of (U,V) at B + p with p < B - eps: (X,Y) wins the tie, and a position
  taken mod B or read as signed at B = 2^31 would pick (U,V).
* Z^mz = (" " + "Z" * 1025)^mz after U: (Z,Z) has the largest count, so the first merge is a pair (a,a), applied while
  the stream holds more than B tokens, with runs that cross 512-word segments.
* S^rs = (" stop<|endoftext|> go")^rs at the end: special-token occurrences past B.
"""
import numpy as np
import regex

import oracle

EOT = "<|endoftext|>"
XY_REPS, Z_RUN = 64, 1025


def p_block(nbytes, seed=7):
    """About `nbytes` of lowercase words with digits, punctuation, newlines and non-ASCII lowercase letters; starts with
    a space, ends with an ASCII letter.  Many distinct words keep every pair's count low."""
    rng = np.random.default_rng(seed)
    letters = "abcdefghijklmnopqrstuvwxyz"
    out, size = [], 0
    while size < nbytes:
        r = rng.random()
        if r < 0.04:
            w = " " + str(int(rng.integers(0, 100000)))
        elif r < 0.07:
            w = "," if rng.random() < 0.5 else "."
        elif r < 0.08:
            w = ".\n"
        elif r < 0.10:
            w = " " + "".join(rng.choice(list(letters), int(rng.integers(1, 4)))) + rng.choice(list("éøßçñü")) + "a"
        else:
            w = " " + "".join(rng.choice(list(letters), int(rng.integers(1, 10))))
        out.append(w)
        size += len(w.encode("utf-8"))
    out.append(" end")
    return "".join(out)


def _block_counts(text):
    """Byte-pair counts of one block without chunk marks: an upper bound for every pattern's chunked count."""
    b = np.frombuffer(text.encode("utf-8"), dtype=np.uint8).astype(np.int64)
    return np.bincount((b[:-1] << 8) | b[1:], minlength=1 << 16)


class Text:
    """The blocks, their repeats and their start offsets in the text, with the construction's facts."""

    def __init__(self, B, p_bytes):
        self.B = B
        P = p_block(p_bytes)
        x_blk, u_blk = " " + "XY" * XY_REPS, " " + "UV" * XY_REPS
        z_blk, s_blk = " " + "Z" * Z_RUN, " stop" + EOT + " go"
        LP = len(P.encode("utf-8"))
        r_p_max = B // LP + 1
        # the tie count: above every pair count of P^r (and of S, which is short)
        tie = int(1.25 * int(_block_counts(P).max()) * r_p_max) + 1
        m = -(-tie // XY_REPS)
        tx = m * len(x_blk)
        r_p = (B - tx // 2) // LP                  # X starts about half its length below B
        mz = -(-m * XY_REPS * 5 // 4 // (Z_RUN - 1)) + 1
        self.blocks = [(P, r_p), (x_blk, m), (u_blk, m), (z_blk, mz), (s_blk, 1000)]
        self.raw = [b.encode("utf-8") for b, _ in self.blocks]
        starts, pos = [], 0
        for raw, (_, r) in zip(self.raw, self.blocks):
            starts.append(pos)
            pos += len(raw) * r
        self.starts, self.nbytes = starts, pos
        self.x_first, self.u_first = starts[1] + 1, starts[2] + 1      # the first (X,Y) and (U,V): after the space
        assert self.x_first < B <= self.u_first < self.starts[2] + len(self.raw[2]) * m
        assert self.u_first - B < B - self.x_first
        assert self.starts[3] >= B and self.starts[4] >= B
        counts = m * XY_REPS
        assert counts > _block_counts(P).max() * r_p and (Z_RUN - 1) * mz > counts > (Z_RUN // 2 - 1) * mz

    def array(self):
        """The text as one uint8 array, built by tiling (no str of the whole text is ever made)."""
        out = np.empty(self.nbytes, dtype=np.uint8)
        for raw, (_, r), s in zip(self.raw, self.blocks, self.starts):
            out[s: s + len(raw) * r].reshape(r, len(raw))[:] = np.frombuffer(raw, dtype=np.uint8)
        return out

    def write(self, path, slab=1 << 28):
        with open(path, "wb") as f:
            for raw, (_, r) in zip(self.raw, self.blocks):
                per = max(1, slab // len(raw))
                chunk = raw * min(per, r)
                left = r
                while left >= per:
                    f.write(chunk)
                    left -= per
                if left:
                    f.write(raw * left)

    def documents(self):
        """Every repeat of every block as one document (the same str objects, repeated)."""
        for b, r in self.blocks:
            for _ in range(r):
                yield b


def parts(text, specials):
    if not specials:
        return [text]
    return regex.split("(" + "|".join(regex.escape(k) for k in specials) + ")", text)[0::2]


def block_chunks(block, pattern, specials=None):
    """-> [(chunk bytes, byte offset in the block)] of the block's parts, split on their own."""
    out, base = [], 0
    pieces = regex.split("(" + "|".join(regex.escape(k) for k in specials) + ")", block) if specials else [block]
    for i, piece in enumerate(pieces):
        if i % 2 == 0:
            at = np.zeros(len(piece) + 1, dtype=np.int64)          # byte offset of every character
            np.cumsum([len(ch.encode("utf-8")) for ch in piece], out=at[1:])
            out += [(mt.group().encode("utf-8"), base + int(at[mt.start()])) for mt in pattern.finditer(piece)]
        base += len(piece.encode("utf-8"))
    return out


def entries(t, pattern, specials=None):
    """The distinct chunks of the text in first-occurrence order -> (bytes uint8, offsets uint64, weights int64,
    first text position uint64 of every entry), from the blocks alone."""
    pat = regex.compile(pattern)
    index, chunks, weights, first = {}, [], [], []
    for (block, r), s in zip(t.blocks, t.starts):
        for c, off in block_chunks(block, pat, specials):
            k = index.get(c)
            if k is None:
                index[c] = len(chunks)
                chunks.append(c)
                weights.append(r)
                first.append(s + off)
            else:
                weights[k] += r
    lens = np.fromiter(map(len, chunks), dtype=np.int64, count=len(chunks))
    offs = np.zeros(len(chunks), dtype=np.uint64)
    np.cumsum(lens[:-1], out=offs[1:].view(np.int64))
    return (np.frombuffer(b"".join(chunks), dtype=np.uint8), offs, np.asarray(weights, dtype=np.int64),
            np.asarray(first, dtype=np.uint64))


def reorder(data, offs, weights, order):
    """The entries in another order (a permutation of their indices)."""
    ends = np.append(offs[1:], np.uint64(data.size)).astype(np.int64)
    chunks = [data[int(offs[i]): ends[i]] for i in order]
    lens = np.fromiter((c.size for c in chunks), dtype=np.int64, count=len(chunks))
    o = np.zeros(len(chunks), dtype=np.uint64)
    np.cumsum(lens[:-1], out=o[1:].view(np.int64))
    return np.concatenate(chunks), o, weights[order]


def truncations(B):
    """How a 32-bit position could go wrong at boundary B: name -> the key a truncated position would sort by."""
    e = B.bit_length() - 1
    out = {f"mod 2^{e}": lambda p: p % B}
    if B <= 1 << 31:                               # an int32 (or, at a small B, a signed e+1-bit) position
        out[f"signed at 2^{e}"] = lambda p: ((p + B) % (2 * B)).astype(np.int64) - B
    return out


def train(data, offs, weights, K):
    return oracle.c_train(data.astype(np.int32), offs, K, weights=weights)


def token_lengths(pairs):
    L = np.ones(256 + len(pairs), dtype=np.int64)
    for i, (a, b) in enumerate(pairs):
        L[256 + i] = L[a] + L[b]
    return L


def merged_entries(data, offs, weights, pairs):
    """The entries after the merges: (final ids, chunk-start flags); stream_len = sum of the weights over the tokens."""
    _, _, _, fin = oracle.c_train(data.astype(np.int32), offs, len(pairs), weights=weights, want_final=True)
    lens = token_lengths(pairs)[fin]
    return fin, np.isin(np.cumsum(lens) - lens, offs.astype(np.int64))


def encode_block(block, pattern, merges, specials=None):
    """The ids of one block (allowed_special="all" when `specials` is given): the oracle's encode of every part."""
    pat = regex.compile(pattern)
    pieces = regex.split("(" + "|".join(regex.escape(k) for k in specials) + ")", block) if specials else [block]
    out = []
    for i, piece in enumerate(pieces):
        if i % 2:
            out.append(np.array([specials[piece]], dtype=np.int32))
            continue
        chunks = [c.encode("utf-8") for c in pat.findall(piece)]
        if not chunks:
            continue
        lens = np.fromiter(map(len, chunks), dtype=np.int64, count=len(chunks))
        o = np.zeros(len(chunks), dtype=np.uint64)
        np.cumsum(lens[:-1], out=o[1:].view(np.int64))
        out.append(oracle.c_encode(np.frombuffer(b"".join(chunks), dtype=np.uint8), o, merges))
    return np.concatenate(out)
