"""Exact collisions for every hash the library keys a table or a cache on.

The hashes are restated here in Python / numpy, with the inverses that make collisions cheap to build:

- hash64 (common.cuh, the murmur3 finaliser) is a bijection of 64-bit words: un-xorshift, multiply by the modular inverse.
- hash_bytes, the 8-bytes-per-step hash the host caches were keyed on before they compared contents (step
  h = (h ^ w) * odd, h ^= h >> 29): every step is a bijection in h ^ w, so one changed word is repaired by the next one.
- e2_tag (k_encode2.cuh): the memo tag of a chunk, hash64 chained over 8-byte words; the last word of a chunk whose
  length is a multiple of 8 is free to hit any tag.
- dd_key (k_dedup.cuh): the chunk-table key, hash64 chained over 32-bit *additive* steps; two prefixes whose states
  differ by less than 2^32 (birthday search on the high half) are made equal by their last words.
- the home slots of k_hist_dense, k_hist_hash and Table / RankTable.

The tests use these to reach the slow paths of the tables (bounded probes that spill, tag matches whose bytes differ,
linear probes that wrap past the end) on purpose, and to pin that the host caches compare contents, not hashes.
"""
import numpy as np

M64 = (1 << 64) - 1
GOLD = 0x9e3779b97f4a7c15
HB_SEED = 0x243f6a8885a308d3
_F1, _F2 = 0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53
_F1I, _F2I, _GOLDI = pow(_F1, -1, 1 << 64), pow(_F2, -1, 1 << 64), pow(GOLD, -1, 1 << 64)

E2_PROBES = 24          # k_encode2.cuh
DD_PROBES = 64          # k_dedup.cuh
HH_SLOTS = 2048         # k_stats.cuh, k_hist_hash shared-memory slots
HD_LOG2 = 12            # k_stats.cuh, k_hist_dense shared-memory slots (log2)


# ---- hash64 and its inverse ------------------------------------------------------------------------------------------
def _unxorshift(y, s):
    x = y
    for _ in range(64 // s + 1):
        x = y ^ (x >> s)
    return x & M64


def hash64(x):
    x &= M64
    x ^= x >> 33; x = (x * _F1) & M64
    x ^= x >> 33; x = (x * _F2) & M64
    return x ^ (x >> 33)


def hash64_inv(y):
    x = _unxorshift(y & M64, 33); x = (x * _F2I) & M64
    x = _unxorshift(x, 33); x = (x * _F1I) & M64
    return _unxorshift(x, 33)


def hash64_np(x):
    """hash64 of a uint64 array (wrapping arithmetic)."""
    x = np.asarray(x, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(33); x *= np.uint64(_F1)
        x ^= x >> np.uint64(33); x *= np.uint64(_F2)
        x ^= x >> np.uint64(33)
    return x


def pack_pair(a, b):
    return ((int(a) & 0xffffffff) << 32) | (int(b) & 0xffffffff)


# ---- hash_bytes ----------------------------------------------------------------------------------------------------------
def hb_step(h, w):
    h = ((h ^ w) * GOLD) & M64
    return h ^ (h >> 29)


def hb_step_inv(h_next):
    """-> h ^ w of the step that produced h_next."""
    return (_unxorshift(h_next, 29) * _GOLDI) & M64


def hash_bytes(b, seed=HB_SEED):
    b = bytes(b)
    h = seed ^ len(b)
    for i in range(0, len(b) - len(b) % 8, 8):
        h = hb_step(h, int.from_bytes(b[i:i + 8], "little"))
    if len(b) % 8:
        h = hb_step(h, int.from_bytes(b[len(b) - len(b) % 8:] + bytes(8 - len(b) % 8), "little"))
    return h


def _hb_states(b, seed=HB_SEED):
    """states[i] = the hash state before word i (whole words only)."""
    h = seed ^ len(b)
    out = [h]
    for i in range(0, len(b) - 7, 8):
        h = hb_step(h, int.from_bytes(b[i:i + 8], "little"))
        out.append(h)
    return out


def _repair(b, r, new_word, seed=HB_SEED):
    """-> the word r+1 that makes b with word r = new_word hash as b does."""
    s = _hb_states(b, seed)
    old_next = int.from_bytes(b[8 * (r + 1): 8 * (r + 2)], "little")
    return hb_step(s[r], new_word) ^ s[r + 1] ^ old_next


def merges_collision(merges, r, seed=0, tries=4096):
    """-> merges' != merges, same shape, equal hash_bytes: pair r is changed to a random pair of ids < 256 + r and pair
    r + 1 repaired; retried until both halves of the repaired word are in [0, 2^31) (about 1 try in 4).  The repaired pair
    holds ids no text produces, so it never applies."""
    m = np.ascontiguousarray(merges, dtype=np.int32)
    assert m.ndim == 2 and m.shape[1] == 2 and 0 <= r < m.shape[0] - 1
    b = m.astype("<i4").tobytes()
    rng = np.random.default_rng(seed)
    for _ in range(tries):
        pr = rng.integers(0, 256 + r, 2).astype(np.int32)
        if np.array_equal(pr, m[r]):
            continue
        w = _repair(b, r, int.from_bytes(pr.astype("<i4").tobytes(), "little"))
        lo, hi = w & 0xffffffff, w >> 32
        if lo < (1 << 31) and hi < (1 << 31):
            out = m.copy()
            out[r] = pr
            out[r + 1] = (lo, hi)
            return out
    raise RuntimeError("merges_collision: no repair in range")


def perm_collision(perm, r, seed=0):
    """-> a 256-byte map != perm with equal hash_bytes: word r (bytes 8r..8r+7) set to random bytes, word r+1 repaired."""
    p = bytes(np.ascontiguousarray(perm, dtype=np.uint8))
    assert len(p) == 256 and 0 <= r < 31
    rng = np.random.default_rng(seed)
    while True:
        new = bytes(rng.integers(0, 256, 8).astype(np.uint8))
        if new != p[8 * r: 8 * r + 8]:
            break
    w = _repair(p, r, int.from_bytes(new, "little"))
    out = p[:8 * r] + new + w.to_bytes(8, "little") + p[8 * r + 16:]
    return np.frombuffer(out, dtype=np.uint8).copy()


def spec_hash(specials):
    """The chained hash of a special set [(bytes, id), ...]: blob, then uint32 offsets, then int32 ids, | 1."""
    if not specials:
        return 0
    blob = b"".join(t for t, _ in specials)
    offs = np.zeros(len(specials) + 1, dtype="<u4")
    offs[1:] = np.cumsum([len(t) for t, _ in specials])
    h = hash_bytes(blob)
    h = hash_bytes(offs.tobytes(), h)
    return hash_bytes(np.asarray([i for _, i in specials], dtype="<i4").tobytes(), h) | 1


def specials_collision(specials, tokens):
    """-> [(tokens[0], id0), (tokens[1], id1)] with the spec_hash and the count of `specials` (two specials): the ids word
    is solved for; `| 1` gives two targets, and the ids must both land in [0, 2^31).  None when neither target does."""
    assert len(specials) == 2 and len(tokens) == 2
    target = spec_hash(specials)
    blob = b"".join(tokens)
    offs = np.asarray([0, len(tokens[0]), len(blob)], dtype="<u4")
    s = hash_bytes(offs.tobytes(), hash_bytes(blob)) ^ 8      # state before the ids word (8 bytes of ids)
    for t in (target & ~1, target | 1):
        w = hb_step_inv(t) ^ s
        lo, hi = w & 0xffffffff, w >> 32
        if lo < (1 << 31) and hi < (1 << 31):
            return [(tokens[0], lo), (tokens[1], hi)]
    return None


def specials_collision_search(specials, make_tokens, limit=4096):
    """specials_collision over make_tokens(0), make_tokens(1), ... until one solves."""
    for t in range(limit):
        got = specials_collision(specials, make_tokens(t))
        if got is not None:
            return got
    raise RuntimeError("specials_collision_search: nothing found")


# ---- e2_tag (memo of the chunk encode) -----------------------------------------------------------------------------
E2_LMAX = 48


def e2_tag(chunk):
    chunk = bytes(chunk)
    n = len(chunk)
    assert 1 <= n <= E2_LMAX
    kw = chunk + bytes(E2_LMAX - n)
    words = [int.from_bytes(kw[8 * j: 8 * j + 8], "little") for j in range(E2_LMAX // 8)]
    h = GOLD ^ (n << 56)
    h = hash64(h ^ words[0])
    for j in range(1, E2_LMAX // 8):
        if n > 8 * j:
            h = hash64(h ^ words[j])
    return h | 1


def e2_state(prefix, n):
    """the e2_tag state after the whole words of `prefix`, for a chunk of n bytes"""
    h = GOLD ^ (n << 56)
    for j in range(len(prefix) // 8):
        h = hash64(h ^ int.from_bytes(prefix[8 * j: 8 * j + 8], "little"))
    return h


def e2_home(tag, log2):
    return (tag >> 1) & ((1 << log2) - 1)


def e2_chunk_for_tag(prefix, target):
    """-> prefix + 8 bytes whose e2_tag is target | 1 (len(prefix) a multiple of 8, the chunk at most 48 bytes)."""
    prefix = bytes(prefix)
    assert len(prefix) % 8 == 0 and len(prefix) + 8 <= E2_LMAX
    n = len(prefix) + 8
    last = hash64_inv(target) ^ e2_state(prefix, n)
    return prefix + last.to_bytes(8, "little")


def e2_collision(a, prefix):
    """-> a chunk b != a with e2_tag(b) == e2_tag(a): len(a) = len(prefix) + 8, a multiple of 8."""
    a, prefix = bytes(a), bytes(prefix)
    assert len(a) == len(prefix) + 8
    b = e2_chunk_for_tag(prefix, e2_tag(a) & ~1)
    assert b != a
    return b


def e2_cluster(count, log2, slot, prefix=b"", seed=0):
    """-> `count` distinct chunks (prefix + 8 bytes) whose memo home slot under a 2^log2-slot memo is `slot`."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        hi = int(rng.integers(0, 1 << 62)) >> log2
        c = e2_chunk_for_tag(prefix, (hi << (log2 + 1)) | (slot << 1))
        if c not in out:
            out.append(c)
    return out


# ---- dd_key (chunk table of the counting session) -------------------------------------------------------------------
DD_KEY_MAX = 48


def dd_words(b):
    b = bytes(b)
    pad = b + bytes((-len(b)) % 4)
    return [int.from_bytes(pad[4 * i: 4 * i + 4], "little") for i in range(len(pad) // 4)]


def dd_key(b):
    b = bytes(b)
    h = GOLD ^ len(b)
    for i, w in enumerate(dd_words(b)):
        h = hash64((h + w + (i << 40)) & M64)
    return h


def dd_tag(key):
    return (key >> 32) | 2


def dd_home(key, log2):
    return key & ((1 << log2) - 1)


def dd_collision(nwords=3, seed=0, batch=1 << 17):
    """-> two distinct byte strings of 4 * nwords bytes with equal dd_key: a birthday search on the high 32 bits of the
    state after nwords - 1 random words (about 2^17 samples), then last words that absorb the difference (< 2^32)."""
    assert 2 <= nwords <= DD_KEY_MAX // 4
    rng = np.random.default_rng(seed)
    n = 4 * nwords
    while True:
        pre = rng.integers(0, 1 << 32, size=(batch, nwords - 1), dtype=np.uint64)
        h = np.full(batch, GOLD ^ n, dtype=np.uint64)
        with np.errstate(over="ignore"):
            for i in range(nwords - 1):
                h = hash64_np(h + pre[:, i] + np.uint64(i << 40))
        hi = h >> np.uint64(32)
        order = np.argsort(hi, kind="stable")
        same = np.nonzero(hi[order][1:] == hi[order][:-1])[0]
        for j in same:
            x, y = int(order[j]), int(order[j + 1])
            if np.array_equal(pre[x], pre[y]):
                continue
            sx, sy = int(h[x]), int(h[y])
            if sx < sy:
                x, y, sx, sy = y, x, sy, sx
            d = sx - sy                                  # 0 <= d < 2^32: sx + wx == sy + wy with wx = 0, wy = d
            a = b"".join(int(v).to_bytes(4, "little") for v in pre[x]) + (0).to_bytes(4, "little")
            b = b"".join(int(v).to_bytes(4, "little") for v in pre[y]) + d.to_bytes(4, "little")
            if a != b:
                return a, b


def dd_cluster(count, log2, slot, make, seed=0, batch=1 << 16):
    """-> `count` distinct byte strings from make(rng, batch) (a list of candidates) whose chunk-table home slot under a
    2^log2-slot table is `slot`."""
    rng = np.random.default_rng(seed)
    out, seen = [], set()
    while len(out) < count:
        for c in make(rng, batch):
            if c not in seen and dd_home(dd_key(c), log2) == slot:
                seen.add(c)
                out.append(c)
                if len(out) == count:
                    break
    return out


# ---- home slots of the pair tables ----------------------------------------------------------------------------------
def hist_dense_home(a, b):
    """k_hist_dense: key = a << 8 | b of a byte pair, (key * 2654435761) >> 20 (32-bit)."""
    key = (int(a) << 8) | int(b)
    return ((key * 2654435761) & 0xffffffff) >> (32 - HD_LOG2)


def hist_hash_home(a, b):
    """k_hist_hash: hash64(pack_pair(a, b)) & 2047."""
    return hash64(pack_pair(a, b)) & (HH_SLOTS - 1)


def table_home(a, b, mask):
    """Table / RankTable: hash64(pack_pair(a, b)) & mask (linear probing, wrapping to slot 0)."""
    return hash64(pack_pair(a, b)) & mask


def pair_homes(a, b, mask):
    """table_home of arrays of ids a, b (vectorised)."""
    key = (np.asarray(a, dtype=np.uint64) << np.uint64(32)) | np.asarray(b, dtype=np.uint64)
    return hash64_np(key) & np.uint64(mask)


def pair_cluster(count, mask, slot, lo=0, hi=1 << 16, seed=0, exclude=()):
    """-> `count` distinct pairs (a, b) with lo <= a, b < hi whose home slot in a table of mask + 1 slots is `slot`."""
    rng = np.random.default_rng(seed)
    out, seen = [], set(exclude)
    while len(out) < count:
        a = rng.integers(lo, hi, 1 << 16)
        b = rng.integers(lo, hi, 1 << 16)
        for j in np.nonzero(pair_homes(a, b, mask) == np.uint64(slot))[0]:
            p = (int(a[j]), int(b[j]))
            if p not in seen:
                seen.add(p)
                out.append(p)
                if len(out) == count:
                    break
    return out


def byte_pairs_in_slot(slot, home):
    """every byte pair (a, b) whose home(a, b) is `slot`"""
    return [(a, b) for a in range(256) for b in range(256) if home(a, b) == slot]
