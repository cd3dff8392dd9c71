// k_encode.cuh — per-chunk encode (regex.py:92-109 `_encode_chunk`, applied to every chunk of
// regex.py:111-121 `encode_ordinary`): while the chunk has >= 2 tokens, find the present pair with
// the lowest merge rank (min(stats, key=merges.get)), stop if none is mergeable, else replace its
// occurrences greedily left to right (base.py:25-41).
//
// Chunks are independent and tiny (mean ~5 bytes for the GPT-4 split), so the natural mapping is
//   k_encode_chunks  one THREAD per chunk (<= ENC_LOCAL tokens), tokens in a per-thread array,
//                    merge ranks from an open-addressing table that lives in L2/L1 (encode_chunk_thread, which
//                    the memoised path's one-thread kernels run as well)
//   k_encode_long    one CTA per long chunk (<= ENC_LONG_MAX tokens), tokens in shared memory
// Ids are written at the chunk's own byte offset in a buffer of n words, unused tail slots get
// ENC_HOLE; k_compact_holes then squeezes every 512-word segment in place and leaves segment
// counts in the edge records, so the ordinary pack (k_scan_counts + k_gather) produces the
// contiguous id list.
#pragma once
#include "common.cuh"
#include "k_seg.cuh"

#define ENC_LOCAL 64
#define ENC_LONG_MAX 8192
#define ENC_HOLE 0xffffffffu
#define RANK_NONE 0xffffffffu

struct RankTable {
    const u64 *keys;   // packed pair or KEY_EMPTY
    const u32 *ranks;
    u64 mask;
};

__device__ __forceinline__ u32 rank_of(const RankTable &t, u32 a, u32 b) {
    const u64 key = pack_pair(a, b);
    u64 slot = hash64(key) & t.mask;
    for (;;) {
        const u64 k = __ldg(&t.keys[slot]);
        if (k == key) return __ldg(&t.ranks[slot]);
        if (k == KEY_EMPTY) return RANK_NONE;
        slot = (slot + 1) & t.mask;
    }
}

// merges[2r], merges[2r+1] -> table (later duplicates of a pair overwrite earlier ones, like the
// dict built by base.py:159-165)
__global__ void k_rank_table_build(const int *__restrict__ merges, int n_merges, u64 *keys, u32 *ranks, u64 mask) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_merges) return;
    const u64 key = pack_pair((u32)merges[2 * r], (u32)merges[2 * r + 1]);
    u64 slot = hash64(key) & mask;
    for (;;) {
        const u64 k = keys[slot];
        if (k == key) break;
        if (k == KEY_EMPTY) {
            const u64 old = atomicCAS((ull *)&keys[slot], (ull)KEY_EMPTY, (ull)key);
            if (old == KEY_EMPTY || old == key) break;
        }
        slot = (slot + 1) & mask;
    }
    atomicMax(&ranks[slot], (u32)r);
}

// regex.py:92-109 on a short token list held by one thread: tok[0, len) in/out, returns the new length
__device__ __forceinline__ u32 encode_chunk_thread(u32 *tok, u32 len, const RankTable &rt) {
    while (len >= 2) {
        u32 best = RANK_NONE, ba = 0, bb = 0;
        for (u32 i = 0; i + 1 < len; ++i) {
            const u32 r = rank_of(rt, tok[i], tok[i + 1]);
            if (r < best) { best = r; ba = tok[i]; bb = tok[i + 1]; }
        }
        if (best == RANK_NONE) break;
        const u32 z = 256u + best;
        u32 j = 0;
        for (u32 i = 0; i < len;) {
            if (i + 1 < len && tok[i] == ba && tok[i + 1] == bb) { tok[j++] = z; i += 2; }
            else tok[j++] = tok[i++];
        }
        len = j;
    }
    return len;
}

__global__ void __launch_bounds__(128) k_encode_chunks(const unsigned char *__restrict__ bytes, const u64 *__restrict__ offs,
                                                       u64 n_chunks, u64 n, RankTable rt,
                                                       const unsigned char *__restrict__ perm, u32 *__restrict__ out,
                                                       u64 *__restrict__ long_list, ull *__restrict__ long_count) {
    const u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chunks) return;
    const u64 lo = offs[c], hi = (c + 1 < n_chunks) ? offs[c + 1] : n;
    const u64 len64 = hi - lo;
    if (len64 > ENC_LOCAL) {        // k_encode_long owns this chunk
        if (len64 > ENC_LONG_MAX) atomicAdd(&long_count[1], 1ull);   // too long even for that: host falls back
        else long_list[atomicAdd(&long_count[0], 1ull)] = c;
        return;
    }
    const u32 len0 = (u32)len64;
    u32 tok[ENC_LOCAL];
    for (u32 i = 0; i < len0; ++i) {
        const u32 b = bytes[lo + i];
        tok[i] = perm ? perm[b] : b;
    }
    const u32 len = encode_chunk_thread(tok, len0, rt);
    for (u32 i = 0; i < len0; ++i) out[lo + i] = (i < len) ? tok[i] : ENC_HOLE;
}

// one CTA per long chunk; list[k] = chunk index
__global__ void __launch_bounds__(256) k_encode_long(const unsigned char *__restrict__ bytes, const u64 *__restrict__ offs,
                                                     u64 n_chunks, u64 n, const u64 *__restrict__ list, u64 n_list,
                                                     RankTable rt, const unsigned char *__restrict__ perm,
                                                     u32 *__restrict__ out) {
    extern __shared__ u32 sm[];
    u32 *tk = sm, *tk2 = sm + ENC_LONG_MAX;
    __shared__ u32 s_scan[256];
    __shared__ u32 s_best, s_a, s_b, s_len;
    const u32 tid = threadIdx.x;
    for (u64 q = blockIdx.x; q < n_list; q += gridDim.x) {
        const u64 c = list[q];
        const u64 lo = offs[c], hi = (c + 1 < n_chunks) ? offs[c + 1] : n;
        const u32 len0 = (u32)(hi - lo);
        for (u32 i = tid; i < len0; i += 256) { const u32 b = bytes[lo + i]; tk[i] = perm ? perm[b] : b; }
        u32 len = len0;
        __syncthreads();
        for (;;) {
            if (len < 2) break;
            if (tid == 0) s_best = RANK_NONE;
            __syncthreads();
            u32 best = RANK_NONE;
            for (u32 i = tid; i + 1 < len; i += 256) { const u32 r = rank_of(rt, tk[i], tk[i + 1]); best = r < best ? r : best; }
            if (best != RANK_NONE) atomicMin(&s_best, best);
            __syncthreads();
            best = s_best;
            if (best == RANK_NONE) break;
            // the pair of that rank: any position holding it (all lookups of one rank agree)
            for (u32 i = tid; i + 1 < len; i += 256)
                if (rank_of(rt, tk[i], tk[i + 1]) == best) { s_a = tk[i]; s_b = tk[i + 1]; }
            __syncthreads();
            const u32 a = s_a, b = s_b, z = 256u + best;
            // mark merge starts into tk2 (1 = start, 2 = tail), greedy left to right
            if (a != b) {
                for (u32 i = tid; i < len; i += 256) {
                    const bool st = (i + 1 < len) && tk[i] == a && tk[i + 1] == b;
                    const bool tail = (i >= 1) && tk[i - 1] == a && tk[i] == b;
                    tk2[i] = st ? 1u : (tail ? 2u : 0u);
                }
            } else if (tid == 0) {
                for (u32 i = 0; i < len;) {
                    if (i + 1 < len && tk[i] == a && tk[i + 1] == a) { tk2[i] = 1u; tk2[i + 1] = 2u; i += 2; }
                    else { tk2[i] = 0u; i += 1; }
                }
            }
            __syncthreads();
            // compaction: each thread owns a contiguous slice
            const u32 per = (len + 255) / 256;
            const u32 s0 = min(len, tid * per), s1 = min(len, s0 + per);
            u32 kept = 0;
            for (u32 i = s0; i < s1; ++i) kept += (tk2[i] != 2u);
            s_scan[tid] = kept;
            __syncthreads();
            for (int o = 1; o < 256; o <<= 1) {
                const u32 v = (tid >= (u32)o) ? s_scan[tid - o] : 0;
                __syncthreads();
                s_scan[tid] += v;
                __syncthreads();
            }
            u32 dst = s_scan[tid] - kept;
            if (tid == 255) s_len = s_scan[255];
            // write compacted tokens over the mark array is unsafe (slices interleave): stage in registers
            // by re-reading tk/tk2 and writing into the upper half only after everyone has read its marks
            __syncthreads();
            u32 outv[32];   // per <= 32 for len <= 8192
            u32 m = 0;
            for (u32 i = s0; i < s1; ++i) {
                const u32 f = tk2[i];
                if (f != 2u) outv[m++] = (f == 1u) ? z : tk[i];
            }
            __syncthreads();
            for (u32 k = 0; k < m; ++k) tk2[dst + k] = outv[k];
            __syncthreads();
            len = s_len;
            for (u32 i = tid; i < len; i += 256) tk[i] = tk2[i];
            __syncthreads();
        }
        __syncthreads();
        for (u32 i = tid; i < len0; i += 256) out[lo + i] = (i < len) ? tk[i] : ENC_HOLE;
        __syncthreads();
    }
}

// Squeeze ENC_HOLE words out of every segment, in place, and record the segment's edge (count +
// boundary tokens) so that the stream machinery (pack, read-back) can take over.  One warp per
// segment; a lane owns 16 consecutive words (SEG_TOKENS = 32 x 16).
__global__ void __launch_bounds__(256) k_compact_holes(u32 *__restrict__ w, u64 n, Edge *e0) {
    static_assert(SEG_TOKENS == 512, "k_compact_holes: one lane owns 16 words");
    const u32 lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    const u32 nseg = (u32)((n + SEG_TOKENS - 1) / SEG_TOKENS);
    for (u32 t = blockIdx.x * wpb + (threadIdx.x >> 5); t < nseg; t += gridDim.x * wpb) {
        const u64 base = (u64)t * SEG_TOKENS;
        const u32 cnt = (u32)((n - base < SEG_TOKENS) ? (n - base) : SEG_TOKENS);
        u32 v[16], kept = 0;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const u32 i = lane * 16 + k;
            v[k] = (i < cnt) ? w[base + i] : ENC_HOLE;
            kept += (v[k] != ENC_HOLE);
        }
        u32 incl = kept;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const u32 x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += x; }
        const u32 total = __shfl_sync(0xffffffffu, incl, 31);
        u32 dst = incl - kept;
        __syncwarp();   // every lane holds its words before anyone overwrites them
#pragma unroll
        for (int k = 0; k < 16; ++k) if (v[k] != ENC_HOLE) w[base + dst++] = v[k];
        __syncwarp();
        if (lane == 0) {
            Edge ed;
            edge_from_tokens(ed, w + base, total);
            e0[t] = ed;
        }
        __syncwarp();
    }
}

// total number of tokens of a segmented stream -> ctl->n (one block)
__global__ void __launch_bounds__(1024) k_total_count(Ctl *ctl, const Edge *e, u32 nseg) {
    __shared__ u64 s[1024];
    u64 sum = 0;
    for (u32 t = threadIdx.x; t < nseg; t += 1024) sum += e[t].count;
    s[threadIdx.x] = sum;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) { if (threadIdx.x < (u32)o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) { ctl->n = s[0]; ctl->nseg = nseg; ctl->cur = 0; ctl->edge_cur = 0; ctl->contig = 0; }
}
