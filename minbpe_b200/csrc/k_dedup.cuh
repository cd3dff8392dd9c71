// k_dedup.cuh — counting the distinct chunks of a text on the device (bpe_load_text_gpt4_dedup, dedup_host.inl).
//
// Per piece of the text (the splitter's pieces), with the chunk starts of the piece compacted to offsets:
//   k_dd_count<false>  every chunk of <= DD_KEY_MAX bytes claims or finds a slot of the chunk table (exact byte compare;
//               a slot's key is published before its tag, so nobody compares against a half-written key), adds 1 to the
//               slot's count and atomicMin's its text position into the slot's first position
//   k_dd_keep   an occurrence is kept as an entry when it is its slot's first occurrence, or when it has no slot
//               (longer than the key, or no free slot within DD_PROBES probes): the rule of DESIGN.md §14
//   k_dd_lens / k_dd_scan_u64 / k_dd_emit   the kept chunks' bytes, offsets and slots appended to the output, in text order
// A slot's first position is final once its piece is counted (later pieces hold larger positions), so every piece is
// emitted and dropped before the next one is split.  After the last piece k_dd_weights<false> reads every entry's weight:
// the slot's count, or 1 for an entry without a slot.
// With special tokens (a counting session's set, DESIGN.md §18) every accepted occurrence is one chunk of the piece, and
// mark[p] != 0 on the bytes of the occurrences (k_special_meta<false> on a cleared array): k_dd_count<false, true> gives the
// chunk of an occurrence no slot and no count but the table's guard slot (index mask + 1, never probed, first position ~0),
// so k_dd_keep never keeps it.  The text position still runs over the occurrences' bytes, so first occurrences and
// tie-breaks stay those of the text.
// bpe_load_chunks_weighted_dedup merges entries that are already weighted (the ranks' streams, back to back) the same way,
// in one pass over one buffer: k_dd_count<true> adds the entry's weight instead of 1, and k_dd_weights<true> gives an entry
// without a slot its own weight instead of 1.  The weights are the kernels' last parameters, which the <false>
// instantiations do not read.
#pragma once
#include "common.cuh"

#define DD_KEY_MAX 48
#define DD_KW (DD_KEY_MAX / 4)
#define DD_PROBES 64
#define DD_EMPTY 0u
#define DD_BUSY 1u
#define DD_NONE 0xffffffffu

struct DdSlot {
    u32 tag;          // DD_EMPTY, DD_BUSY (being written), else the key's hash tag (>= 2), published after the key
    u32 len;
    u32 key[DD_KW];   // the chunk's bytes, zero padded
    ull count;        // occurrences counted so far
    ull first;        // smallest text position of an occurrence
};
struct DdTable { DdSlot *s; u64 mask; ull *used; };

__device__ __forceinline__ u64 dd_key(const unsigned char *b, u32 len, u32 (&kw)[DD_KW]) {
#pragma unroll
    for (int i = 0; i < DD_KW; ++i) kw[i] = 0;
    for (u32 j = 0; j < len; ++j) kw[j >> 2] |= (u32)b[j] << (8u * (j & 3u));
    u64 h = 0x9e3779b97f4a7c15ull ^ len;
    for (u32 i = 0; i < (len + 3u) / 4u; ++i) h = hash64(h + kw[i] + ((u64)i << 40));
    return h;
}

// the slot of a chunk of len <= DD_KEY_MAX bytes, claimed if it is new (exact byte compare; a slot's key is published
// before its tag, so nobody compares against a half-written key); adds `add` to the slot's count and atomicMin's `pos`
// (= base + off) into its first position.  DD_NONE when no slot with these bytes or free was found within DD_PROBES probes.
__device__ __forceinline__ u32 dd_count_one(const unsigned char *b, u32 len, DdTable T, ull add, u64 base, u64 off) {
    u32 kw[DD_KW];
    const u64 h = dd_key(b, len, kw);
    const u32 tag = (u32)(h >> 32) | 2u;
    u64 slot = h & T.mask;
#pragma unroll 1
    for (int probe = 0; probe < DD_PROBES; ++probe) {
        DdSlot *S = &T.s[slot];
        u32 t = ld_volatile_u32(&S->tag);
        if (t == DD_EMPTY) {
            const u32 old = atomicCAS(&S->tag, DD_EMPTY, DD_BUSY);
            if (old == DD_EMPTY) {        // claimed: key first, then the tag that makes it visible
                S->len = len;
#pragma unroll
                for (int i = 0; i < DD_KW; ++i) S->key[i] = kw[i];
                S->first = ~0ull;
                __threadfence();
                atomicCAS(&S->tag, DD_BUSY, tag);   // only the claimer holds DD_BUSY
                atomicAdd(T.used, 1ull);
                t = tag;
            } else {
                t = old;
            }
        }
        while (t == DD_BUSY) t = ld_volatile_u32(&S->tag);
        __threadfence();
        bool same = t == tag && ld_volatile_u32(&S->len) == len;
        for (int i = 0; same && i < DD_KW; ++i) same = ld_volatile_u32(&S->key[i]) == kw[i];
        if (same) {                       // equal tags with different bytes keep probing
            atomicAdd(&S->count, add);
            atomicMin(&S->first, (ull)(base + off));
            return (u32)slot;
        }
        slot = (slot + 1) & T.mask;
    }
    return DD_NONE;
}

// WEIGHTED (bpe_load_chunks_weighted_dedup): the chunks are weighted entries, w[j] is added instead of 1 (text_pos is 0,
// so an entry's position is its byte offset and a slot's first position is its smallest-index entry)
template <bool WEIGHTED>
__global__ void __launch_bounds__(256) k_dd_count(const unsigned char *__restrict__ text, u64 m, const u64 *__restrict__ offs,
                                                  u64 k, u64 text_pos, DdTable T, u32 *__restrict__ slot_of,
                                                  const u64 *__restrict__ w) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < k; j += (u64)gridDim.x * blockDim.x) {
        const u64 start = offs[j], end = j + 1 < k ? offs[j + 1] : m;
        const u64 len = end - start;
        const ull add = WEIGHTED ? (ull)w[j] : 1ull;
        slot_of[j] = len <= DD_KEY_MAX ? dd_count_one(text + start, (u32)len, T, add, text_pos, start) : DD_NONE;
    }
}

__global__ void __launch_bounds__(256) k_dd_keep(const u64 *__restrict__ offs, u64 k, u64 text_pos, DdTable T,
                                                 const u32 *__restrict__ slot_of, unsigned char *__restrict__ keep) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < k; j += (u64)gridDim.x * blockDim.x) {
        const u32 s = slot_of[j];
        keep[j] = (s == DD_NONE || T.s[s].first == text_pos + offs[j]) ? 1 : 0;
    }
}

// SPEC: chunk j is a special-token occurrence when mark[offs[j]] != 0; its slot is the guard slot T.mask + 1, it adds no
// count, and *skipped counts it
template <bool WEIGHTED, bool SPEC>
__global__ void __launch_bounds__(256) k_dd_count(const unsigned char *__restrict__ text, u64 m, const u64 *__restrict__ offs,
                                                  u64 k, u64 text_pos, DdTable T, u32 *__restrict__ slot_of,
                                                  const u64 *__restrict__ w, const unsigned char *__restrict__ mark,
                                                  ull *__restrict__ skipped) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < k; j += (u64)gridDim.x * blockDim.x) {
        const u64 start = offs[j], end = j + 1 < k ? offs[j + 1] : m;
        const u64 len = end - start;
        const ull add = WEIGHTED ? (ull)w[j] : 1ull;
        if (SPEC && mark[start]) {
            slot_of[j] = (u32)(T.mask + 1);
            atomicAdd(skipped, 1ull);
            continue;
        }
        slot_of[j] = len <= DD_KEY_MAX ? dd_count_one(text + start, (u32)len, T, add, text_pos, start) : DD_NONE;
    }
}

// byte length of every kept chunk (idx = the kept chunks' indices, ascending)
__global__ void __launch_bounds__(256) k_dd_lens(const u64 *__restrict__ offs, u64 k, u64 m, const u64 *__restrict__ idx, u64 nk,
                                                 u64 *__restrict__ lens) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < nk; e += (u64)gridDim.x * blockDim.x) {
        const u64 j = idx[e];
        lens[e] = (j + 1 < k ? offs[j + 1] : m) - offs[j];
    }
}

// exclusive prefix sum of n u64 values and their total (one block of 1024 threads, one slice per warp)
__global__ void __launch_bounds__(1024) k_dd_scan_u64(const u64 *__restrict__ in, u64 n, u64 *__restrict__ excl, u64 *total) {
    const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u64 per = ((n + 31) / 32 + 31) & ~31ull;
    const u64 lo = min(n, (u64)warp * per), hi = min(n, lo + per);
    u64 sum = 0;
    for (u64 t = lo + lane; t < hi; t += 32) sum += in[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __shared__ u64 s_w[32];
    if (lane == 0) s_w[warp] = sum;
    __syncthreads();
    u64 run = 0;
    for (u32 q = 0; q < warp; ++q) run += s_w[q];
    if (warp == 31 && lane == 0) *total = run + sum;
    for (u64 t0 = lo; t0 < hi; t0 += 32) {
        const u64 t = t0 + lane;
        const u64 c = (t < hi) ? in[t] : 0ull;
        u64 incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const u64 v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += v; }
        if (t < hi) excl[t] = run + (incl - c);
        run += __shfl_sync(0xffffffffu, incl, 31);
    }
}

// append the kept chunks: bytes at out_bytes + excl[e], offset bytes_done + excl[e], slot
__global__ void __launch_bounds__(256) k_dd_emit(const unsigned char *__restrict__ text, const u64 *__restrict__ offs,
                                                 const u64 *__restrict__ idx, u64 nk, const u64 *__restrict__ lens,
                                                 const u64 *__restrict__ excl, const u32 *__restrict__ slot_of, u64 bytes_done,
                                                 unsigned char *__restrict__ out_bytes, u64 *__restrict__ out_offs,
                                                 u32 *__restrict__ out_slot) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < nk; e += (u64)gridDim.x * blockDim.x) {
        const u64 j = idx[e], s = offs[j], len = lens[e], o = excl[e];
        for (u64 b = 0; b < len; ++b) out_bytes[o + b] = text[s + b];
        out_offs[e] = bytes_done + o;
        out_slot[e] = slot_of[j];
    }
}

// weights of the entries: the slot's count, 1 without a slot; stats[0] += entries that have a slot.  WEIGHTED: an entry
// without a slot keeps its own weight w_in[idx[e]] (idx = the kept entries' input indices)
template <bool WEIGHTED>
__global__ void __launch_bounds__(256) k_dd_weights(const u32 *__restrict__ slot, u64 n, DdTable T, u64 *__restrict__ wts,
                                                    ull *__restrict__ from_table, const u64 *__restrict__ idx,
                                                    const u64 *__restrict__ w_in) {
    u32 mine = 0;
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (u64)gridDim.x * blockDim.x) {
        const u32 s = slot[e];
        wts[e] = s == DD_NONE ? (WEIGHTED ? w_in[idx[e]] : 1ull) : T.s[s].count;
        mine += s != DD_NONE;
    }
    if (mine) atomicAdd(from_table, (ull)mine);
}
