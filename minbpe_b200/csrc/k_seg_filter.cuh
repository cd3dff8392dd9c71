// k_seg_filter.cuh — skip the segments a merge cannot touch (late iterations of train(): regex.py:49-66 replaces one pair
// per iteration, and after the first few hundred merges that pair lives in a small fraction of the text).
//
// Every 512-token segment keeps a SIGNATURE: 4,096 bits (512 B, a quarter of the segment's size; the filter reads ONE word
// of it), bit hash(x, y) set for every pair of
// adjacent tokens (x, y) INSIDE the segment (y unmarked: no pair spans chunks, regex.py:51-54).  Before a merge (a,b) -> z,
// k_seg_filter decides per segment from two 32-byte edge records and one word of its signature:
//     interior    bit(a, b) is set                               -> the pair may occur inside
//     right edge  last token == a and the next token == b        -> a merge starts at its last token
//     left edge   first token == b and the previous token == a   -> its first token is the tail of a merge
// Candidates go on a list that k_merge_seg<true> works through; for every other segment the filter itself carries the edge
// record over to the other parity buffer (what k_merge_seg does for an untouched segment), so a skipped segment costs ~70 B
// of traffic instead of 2 KB.  After the merge, k_sig_rebuild_cand recomputes the signatures of the listed segments from
// their tokens — the only segments whose token sequence can have changed — so every signature always describes its segment
// exactly (up to hash collisions, which only add candidates).  k_sig_build does the same for all segments whenever tokens
// move between segments (re-packing, the pack of the pairs (a,a)).  The merge pass, the statistics delta and all
// bookkeeping are k_merge_seg's, unchanged.
#pragma once
#include "common.cuh"
#include "k_seg.cuh"

#define SIG_LOG2 12                        // 4,096 bits per segment: a segment of 250 tokens sets ~6 % of them
#define SIG_WORDS ((1 << SIG_LOG2) / 32)
__device__ __forceinline__ u32 sig_bit(u32 x, u32 y) {   // 0 .. 2^SIG_LOG2 - 1; x = id of the left token, y = the right token word (unmarked)
    u32 h = x * 0x9e3779b1u ^ y * 0x85ebca77u;
    h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12;
    return h >> (32 - SIG_LOG2);
}

// signature of segment t from its tokens, by one warp; s_sig = SIG_WORDS words of shared memory private to the warp
__device__ __forceinline__ void sig_of_segment(const u32 *__restrict__ seg, u32 count, u32 *s_sig, u32 *__restrict__ out, u32 lane) {
    for (u32 k = lane; k < SIG_WORDS; k += 32) s_sig[k] = 0;
    __syncwarp();
    for (u32 i = lane; i + 1 < count; i += 32) {
        const u32 y = seg[i + 1];
        if (!(y & TOK_FLAG)) {
            const u32 b = sig_bit(seg[i] & TOK_MASK, y);
            atomicOr(&s_sig[b >> 5], 1u << (b & 31u));
        }
    }
    __syncwarp();
    for (u32 k = lane; k < SIG_WORDS; k += 32) out[k] = s_sig[k];
    __syncwarp();
}

// (Re)build all signatures: one warp per segment.  gate_same: only when the pair of the iteration in flight is (a,a) —
// that path packs the stream, which moves tokens between segments.
__global__ void __launch_bounds__(256) k_sig_build(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1, const Ctl *__restrict__ ctl,
                                                   const Edge *e0, const Edge *e1, u32 *__restrict__ sig, int gate_same) {
    if (gate_same && (ctl->done || ctl->a != ctl->b)) return;
    __shared__ u32 s_sig[8][SIG_WORDS];
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);
    const u32 nseg = ctl->nseg, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    for (u32 t = blockIdx.x * wpb + warp; t < nseg; t += gridDim.x * wpb)
        sig_of_segment(w + (u64)t * SEG_TOKENS, e[t].count, s_sig[warp], sig + (u64)t * SIG_WORDS, lane);
}

// the candidate segments of the merge selected in ctl (a != b); edge records of the others carried over
__global__ void __launch_bounds__(256) k_seg_filter(Ctl *ctl, const Edge *e0, const Edge *e1, Edge *e0w, Edge *e1w,
                                                    const u32 *__restrict__ sig, u32 *__restrict__ cand) {
    if (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter) return;
    if (ctl->a == ctl->b) return;                      // pairs (a,a) take the pack + k_merge<true> path
    const Edge *e_cur = ctl->edge_cur ? e1 : e0;
    Edge *e_next = ctl->edge_cur ? e0w : e1w;
    const u32 a = (u32)ctl->a, b = (u32)ctl->b;
    const u32 bab = sig_bit(a, b);
    const u32 nseg = ctl->nseg, lane = threadIdx.x & 31;
    // whole warps iterate together (the list append is warp-aggregated)
    const u32 nround = (nseg + 31u) & ~31u;
    for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < nround; t += gridDim.x * blockDim.x) {
        bool is_cand = false;
        if (t < nseg) {
            const uint4 *p = reinterpret_cast<const uint4 *>(&e_cur[t]);
            const uint4 q0 = p[0], q1 = p[1];          // f0 f1 f2 l0 | l1 count pad pad
            const u32 count = q1.y;
            if (count == 0) {
                u32 *o = reinterpret_cast<u32 *>(&e_next[t]);
#pragma unroll
                for (int k = 0; k < 8; ++k) o[k] = (k < 5) ? TOK_SENTINEL : 0u;
            } else {
                is_cand = (sig[(u64)t * SIG_WORDS + (bab >> 5)] >> (bab & 31u)) & 1u;
                if (!is_cand && (q1.x & TOK_MASK) == a) {                    // last token is a: does b follow it?
                    // an empty or missing neighbour is rare: walk to the next token then
                    const u32 nx = (t + 1 < nseg && e_cur[t + 1].count) ? e_cur[t + 1].f[0] : seg_next_first(e_cur, t, nseg);
                    is_cand = nx == b;                                       // unmarked b: same chunk
                }
                if (!is_cand && q0.x == b) {                                 // first token is an unmarked b: does a precede it?
                    u32 pv = TOK_SENTINEL;
                    for (long long s = (long long)t - 1; s >= 0; --s) if (e_cur[s].count) { pv = e_cur[s].l[1]; break; }
                    is_cand = pv != TOK_SENTINEL && (pv & TOK_MASK) == a;
                }
                if (!is_cand) {
                    uint4 *o = reinterpret_cast<uint4 *>(&e_next[t]);
                    o[0] = q0; o[1] = q1;
                }
            }
        }
        const u32 m = __ballot_sync(0xffffffffu, is_cand);
        if (m) {
            u32 base = 0;
            if (lane == 0) base = atomicAdd(&ctl->n_cand, (u32)__popc(m));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (is_cand) cand[base + __popc(m & ((1u << lane) - 1u))] = t;
        }
    }
}

// after the merge: the listed segments are the only ones whose tokens can have changed — their signatures from their
// tokens again (one warp per list entry).  The list is empty when the filter did not run this iteration (done, a table
// overflow of an earlier iteration, a pair (a,a)), so a non-empty list is the whole gate of the statistics as well: a
// merge whose own table update overflowed was performed and counts.
__global__ void __launch_bounds__(256) k_sig_rebuild_cand(Ctl *ctl, const u32 *__restrict__ buf0, const u32 *__restrict__ buf1,
                                                          const Edge *e0, const Edge *e1, u32 *__restrict__ sig, const u32 *__restrict__ cand) {
    const u32 n = ctl->n_cand;
    if (blockIdx.x == 0 && threadIdx.x == 0 && n) {
        ctl->cand_sum += n; ctl->seg_sum += ctl->nseg;      // statistics: how much of the stream the filtered merges looked at
    }
    if (!n) return;
    __shared__ u32 s_sig[8][SIG_WORDS];
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);            // the merge kernel has flipped the edge arrays: these are the new counts
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    for (u32 i = blockIdx.x * wpb + warp; i < n; i += gridDim.x * wpb) {
        const u32 t = cand[i];
        sig_of_segment(w + (u64)t * SEG_TOKENS, e[t].count, s_sig[warp], sig + (u64)t * SIG_WORDS, lane);
    }
}

// the list is consumed: the next k_seg_filter starts from an empty one (one thread)
__global__ void k_cand_reset(Ctl *ctl) { ctl->n_cand = 0; }
