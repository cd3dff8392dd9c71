// k_split.cuh — the GPT-4 split pattern (regex.py:19, applied by regex.py:41 / :114) on the device.
//
//   '(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]++[\r\n]*|\s*[\r\n]|\s+(?!\S)|\s+
//
// A regex matcher is sequential, but for THIS pattern "does a match start at character i?" is a
// function of the run structure (runs of letters / digits / whitespace / other).  split_logic.h
// states it on six SEGMENTED scan results (segments = runs) at a byte and at its predecessor, plus a
// few neighbouring bytes; the same header is pinned against the `regex` module on the CPU
// (oracle/split_harness.cpp, tests/test_split_rules.py).  Here:
//   k_split_classify    byte -> {class, char-start}                 (code-point class table from `regex`)
//                       <true>: the documents of a piece spread into the split buffer with one boundary byte between
//                       consecutive ones (bpe_dedup_add_docs, DESIGN.md §15)
//   k_split_reduce      tile aggregates of the forward and of the backward scan
//   k_split_scan_parts  exclusive scans of the aggregates (one block)
//   k_split_apply       per tile: both scans in shared memory seeded with the carries, the rule per
//                       character, and either the flag byte (offsets for encode / host callers) or the
//                       token word with the chunk mark (training: no offsets array, no flag array)
// Nothing per byte is materialised in HBM except the 1-byte class array.
#pragma once
#include "common.cuh"
#include "split_logic.h"

#define SP_THREADS 512
#define SP_ITEMS 8
#define SP_TILE (SP_THREADS * SP_ITEMS)   // 4096 bytes
#define SP_HALO 16                          // bytes of context either side of a tile (the rule reads -12 .. +8)

struct SmemBytes {   // accessor over a shared-memory window: element(pos) for global byte position pos
    const unsigned char *p;   // p[0] = global position `base`
    u64 base;
    __device__ __forceinline__ u32 operator()(u64 pos) const { return p[(int)((long long)pos - (long long)base)]; }
};
struct GmemBytes {
    const unsigned char *p;
    __device__ __forceinline__ u32 operator()(u64 pos) const { return p[pos]; }
};

// ---- documents (bpe_dedup_add_docs): nd documents of a piece, back to back in `src` (m bytes, doff[j] = start of
// document j, doff[0] = 0, none empty), are split in one call with one boundary byte between consecutive ones.  In the
// split buffer byte i of src sits at i + (its document's index); the boundary in front of document j at doff[j] + j - 1
// holds DOC_GAP with class SC_B, so the WITH_B rule (split_logic.h) ends every run there and treats either side as end /
// start of a text, as for a special-token occurrence of length 1 (k_special_meta).  The class is set by position: the
// byte's value does not matter.
#define DOC_GAP 0x00u
#define DOC_SPAN 16   // consecutive bytes per thread of k_split_classify<true>: one binary search over doff, then a walk

// the document of byte i of src: the last j with doff[j] <= i
__device__ __forceinline__ u32 doc_of(const u64 *__restrict__ doff, u32 nd, u64 i) {
    u32 lo = 0, hi = nd;
    while (hi - lo > 1) {
        const u32 mid = (lo + hi) >> 1;
        if (doff[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}
// boundary bytes in front of position p of the split buffer: the number of j >= 1 with doff[j] + j - 1 < p
__device__ __forceinline__ u32 gaps_before(const u64 *__restrict__ doff, u32 nd, u64 p) {
    u32 lo = 0, hi = nd;          // invariant: the gaps of documents 1..lo lie before p, those of hi.. do not
    while (hi - lo > 1) {
        const u32 mid = (lo + hi) >> 1;
        if (doff[mid] + mid - 1 < p) lo = mid; else hi = mid;
    }
    return lo;
}
// SPEC: the buffer also holds special-token occurrences (bpe_encode_docs), class SC_B with SM_SPEC (k_special_meta<true>);
// they are not gaps
template <bool SPEC = false>
__device__ __forceinline__ bool is_gap(const unsigned char *__restrict__ meta, u64 p) {
    return SPEC ? (meta[p] & (SM_CLS | SM_SPEC)) == SC_B : (meta[p] & SM_CLS) == SC_B;
}
// chunk start at position p of the split buffer of documents: not a boundary byte, and a flag of the rule or the first
// byte of a document (the boundary's own one-byte chunk is dropped)
template <bool SPEC = false>
__device__ __forceinline__ u32 doc_chunk_start(const unsigned char *__restrict__ flag, const unsigned char *__restrict__ meta, u64 p) {
    return !is_gap<SPEC>(meta, p) && (flag[p] || (p > 0 && is_gap<SPEC>(meta, p - 1))) ? 1u : 0u;
}

// meta[i] = class of the character byte i belongs to | SM_START on its first byte.
// DOCS: the split buffer `out` (n bytes) is filled from the documents in `src` first, and `b` is not read.  Every
// document is classified on its own bytes, so a character never reaches into the next document.
template <bool DOCS>
__global__ void __launch_bounds__(256) k_split_classify(const unsigned char *__restrict__ b, u64 n,
                                                        const unsigned char *__restrict__ cls_table,
                                                        unsigned char *__restrict__ meta, const unsigned char *__restrict__ src,
                                                        const u64 *__restrict__ doff, u32 nd, unsigned char *__restrict__ out) {
    if constexpr (!DOCS) {
        const GmemBytes B{b};
        for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
            meta[i] = (unsigned char)spl_meta_of(B, i, n, cls_table);
    } else {
        const u64 m = n - (nd - 1), stride = (u64)gridDim.x * blockDim.x;
        for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t * DOC_SPAN < m; t += stride) {
            const u64 lo = t * DOC_SPAN, hi = min(m, lo + DOC_SPAN);
            u32 d = doc_of(doff, nd, lo);
            u64 start = doff[d], next = d + 1 < nd ? doff[d + 1] : m;
            for (u64 i = lo; i < hi; ++i) {
                while (i >= next) { ++d; start = next; next = d + 1 < nd ? doff[d + 1] : m; }
                out[i + d] = src[i];
                meta[i + d] = (unsigned char)spl_meta_of(GmemBytes{src + start}, i - start, next - start, cls_table);
            }
        }
        for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x + 1; j < nd; j += stride) {
            out[doff[j] + j - 1] = DOC_GAP;
            meta[doff[j] + j - 1] = (unsigned char)(SM_START | SC_B);
        }
    }
}

// ---- ordered block primitives for the (non-commutative) segmented operators ----
struct FwdOp { __device__ __forceinline__ SplFwd operator()(SplFwd a, SplFwd b) const { return spl_fwd_combine(a, b); } };
struct BwdOp { __device__ __forceinline__ SplBwd operator()(SplBwd a, SplBwd b) const { return spl_bwd_combine(a, b); } };

// thread `tid` contributes v (thread order = text order); returns the ordered product of all threads' values
template <typename T, typename OP>
__device__ __forceinline__ T block_reduce_ordered(T v, OP op, T *sm, u32 nthreads) {
    const u32 tid = threadIdx.x;
    sm[tid] = v;
    __syncthreads();
    for (u32 o = 1; o < nthreads; o <<= 1) {     // adjacent pairs: operand order is preserved
        if ((tid & (2 * o - 1)) == 0 && tid + o < nthreads) sm[tid] = op(sm[tid], sm[tid + o]);
        __syncthreads();
    }
    const T r = sm[0];
    __syncthreads();
    return r;
}

// tile aggregates of both scans (WITH_B: the class array may hold special-token boundaries, k_special.cuh)
template <bool WITH_B>
__global__ void __launch_bounds__(SP_THREADS) k_split_reduce(const unsigned char *__restrict__ meta, u64 n,
                                                             SplFwd *__restrict__ fpart, SplBwd *__restrict__ bpart) {
    __shared__ SplFwd sf[SP_THREADS];
    __shared__ SplBwd sb[SP_THREADS];
    const u64 base = (u64)blockIdx.x * SP_TILE + (u64)threadIdx.x * SP_ITEMS;
    SplFwd f = spl_fwd_identity();
    SplBwd g = spl_bwd_identity();
    u32 m[SP_ITEMS + 2];   // meta of bytes base-1 .. base+SP_ITEMS
#pragma unroll
    for (int k = 0; k < SP_ITEMS + 2; ++k) {
        const u64 i = base + k;   // position of m[k] is i - 1
        m[k] = (i >= 1 && i - 1 < n) ? meta[i - 1] : 0u;
    }
#pragma unroll
    for (int k = 0; k < SP_ITEMS; ++k)
        if (base + k < n) f = spl_fwd_combine(f, spl_fwd_elem(base + k, m[k + 1], m[k]));
#pragma unroll
    for (int k = SP_ITEMS - 1; k >= 0; --k)
        if (base + k < n) g = spl_bwd_combine(spl_bwd_elem<WITH_B>(base + k, n, m[k + 1], m[k + 2]), g);
    f = block_reduce_ordered(f, FwdOp(), sf, SP_THREADS);
    g = block_reduce_ordered(g, BwdOp(), sb, SP_THREADS);
    if (threadIdx.x == 0) { fpart[blockIdx.x] = f; bpart[blockIdx.x] = g; }
}

// exclusive scans of the tile aggregates (one block): forward left-to-right, backward right-to-left
__global__ void __launch_bounds__(1024) k_split_scan_parts(SplFwd *__restrict__ fpart, SplBwd *__restrict__ bpart, u32 ntiles) {
    __shared__ SplFwd sf[1024];
    __shared__ SplBwd sb[1024];
    const u32 tid = threadIdx.x;
    const u32 per = (ntiles + 1023) / 1024;
    const u32 lo = min(ntiles, tid * per), hi = min(ntiles, lo + per);
    SplFwd f = spl_fwd_identity();
    for (u32 t = lo; t < hi; ++t) f = spl_fwd_combine(f, fpart[t]);
    SplBwd g = spl_bwd_identity();
    for (u32 t = hi; t > lo; --t) g = spl_bwd_combine(bpart[t - 1], g);
    sf[tid] = f; sb[tid] = g;
    __syncthreads();
    for (u32 o = 1; o < 1024; o <<= 1) {   // inclusive: forward over lower tids, backward over higher tids
        SplFwd fv = spl_fwd_identity(); SplBwd gv = spl_bwd_identity();
        if (tid >= o) fv = sf[tid - o];
        if (tid + o < 1024) gv = sb[tid + o];
        __syncthreads();
        sf[tid] = spl_fwd_combine(fv, sf[tid]); sb[tid] = spl_bwd_combine(sb[tid], gv);
        __syncthreads();
    }
    SplFwd frun = spl_fwd_identity();
    if (tid > 0) frun = sf[tid - 1];
    for (u32 t = lo; t < hi; ++t) { const SplFwd x = fpart[t]; fpart[t] = frun; frun = spl_fwd_combine(frun, x); }
    SplBwd grun = spl_bwd_identity();
    if (tid + 1 < 1024) grun = sb[tid + 1];
    for (u32 t = hi; t > lo; --t) { const SplBwd x = bpart[t - 1]; bpart[t - 1] = grun; grun = spl_bwd_combine(x, grun); }
}

// per tile: scans + rule.  TOKENS = false: flag[i] = 1 at chunk starts.  TOKENS = true: dst[i] = byte | chunk mark.
// PATTERN: 0 = the GPT-4 split pattern, 1 = the GPT-2 one (split_logic.h: same scans, another rule).
template <bool TOKENS, bool WITH_B, int PATTERN>
__global__ void __launch_bounds__(SP_THREADS) k_split_apply(const unsigned char *__restrict__ b, const unsigned char *__restrict__ meta, u64 n,
                                                            const unsigned char *__restrict__ contr,
                                                            const SplFwd *__restrict__ fpart, const SplBwd *__restrict__ bpart,
                                                            unsigned char *__restrict__ flag, u32 *__restrict__ dst) {
    __shared__ __align__(16) unsigned char s_b[SP_TILE + 2 * SP_HALO];
    __shared__ __align__(16) unsigned char s_m[SP_TILE + 2 * SP_HALO];
    __shared__ SplFwd sf[SP_THREADS];
    __shared__ SplBwd sb[SP_THREADS];
    const u32 tid = threadIdx.x;
    const u64 lo = (u64)blockIdx.x * SP_TILE;
    // window [lo - HALO, lo + TILE + HALO), zero outside the text
    for (u32 j = tid; j < SP_TILE + 2 * SP_HALO; j += SP_THREADS) {
        const u64 pos = lo + j;   // = real position + HALO
        const bool in = pos >= SP_HALO && pos - SP_HALO < n;
        s_b[j] = in ? b[pos - SP_HALO] : 0;
        s_m[j] = in ? meta[pos - SP_HALO] : 0;
    }
    __syncthreads();
    const SmemBytes B{s_b + SP_HALO, lo}, M{s_m + SP_HALO, lo};   // B(pos), M(pos) for pos in [lo - HALO, lo + TILE + HALO)
    const u64 base = lo + (u64)tid * SP_ITEMS;
    const unsigned char *mm = s_m + SP_HALO + tid * SP_ITEMS;     // mm[k] = meta of byte base + k (mm[-1], mm[SP_ITEMS] valid)
    SplFwd fe[SP_ITEMS]; SplBwd ge[SP_ITEMS];
    SplFwd f = spl_fwd_identity();
    SplBwd g = spl_bwd_identity();
#pragma unroll
    for (int k = 0; k < SP_ITEMS; ++k) {
        if (base + k < n) { fe[k] = spl_fwd_elem(base + k, mm[k], mm[k - 1]); ge[k] = spl_bwd_elem<WITH_B>(base + k, n, mm[k], mm[k + 1]); }
        else { fe[k] = spl_fwd_identity(); ge[k] = spl_bwd_identity(); }
        f = spl_fwd_combine(f, fe[k]);
    }
#pragma unroll
    for (int k = SP_ITEMS - 1; k >= 0; --k) g = spl_bwd_combine(ge[k], g);
    sf[tid] = f; sb[tid] = g;
    __syncthreads();
    for (u32 o = 1; o < SP_THREADS; o <<= 1) {
        SplFwd fv = spl_fwd_identity(); SplBwd gv = spl_bwd_identity();
        if (tid >= o) fv = sf[tid - o];
        if (tid + o < SP_THREADS) gv = sb[tid + o];
        __syncthreads();
        sf[tid] = spl_fwd_combine(fv, sf[tid]); sb[tid] = spl_bwd_combine(sb[tid], gv);
        __syncthreads();
    }
    SplFwd frun = fpart[blockIdx.x];                      // everything in front of the tile
    if (tid > 0) frun = spl_fwd_combine(frun, sf[tid - 1]);
    SplBwd grun = bpart[blockIdx.x];                      // everything behind the tile
    if (tid + 1 < SP_THREADS) grun = spl_bwd_combine(sb[tid + 1], grun);
    SplBwd gi[SP_ITEMS];
#pragma unroll
    for (int k = SP_ITEMS - 1; k >= 0; --k) { grun = spl_bwd_combine(ge[k], grun); gi[k] = grun; }
    u32 out[SP_ITEMS];
#pragma unroll
    for (int k = 0; k < SP_ITEMS; ++k) {
        const u64 i = base + k;
        const SplFwd fprev = frun;
        frun = spl_fwd_combine(frun, fe[k]);
        bool st = false;
        if (i < n && (mm[k] & SM_START))
            st = PATTERN == 1 ? spl_chunk_start_gpt2<WITH_B>(i, n, frun, gi[k], B, M) : spl_chunk_start<WITH_B>(i, n, frun, fprev, gi[k], B, M, contr);
        out[k] = TOKENS ? ((u32)s_b[SP_HALO + tid * SP_ITEMS + k] | (st ? TOK_FLAG : 0u)) : (st ? 1u : 0u);
    }
    if (TOKENS) {
        if (base + SP_ITEMS <= n) {
            uint4 *d = reinterpret_cast<uint4 *>(dst + base);   // base is a multiple of 8 words
            d[0] = make_uint4(out[0], out[1], out[2], out[3]);
            d[1] = make_uint4(out[4], out[5], out[6], out[7]);
        } else {
#pragma unroll
            for (int k = 0; k < SP_ITEMS; ++k) if (base + k < n) dst[base + k] = out[k];
        }
    } else {
        if (base + SP_ITEMS <= n) {
            *reinterpret_cast<uint2 *>(flag + base) = make_uint2(out[0] | (out[1] << 8) | (out[2] << 16) | (out[3] << 24),
                                                                 out[4] | (out[5] << 8) | (out[6] << 16) | (out[7] << 24));
        } else {
#pragma unroll
            for (int k = 0; k < SP_ITEMS; ++k) if (base + k < n) flag[base + k] = (unsigned char)out[k];
        }
    }
}

// text bytes -> token words with the chunk marks taken straight from the split flags
__global__ void __launch_bounds__(256) k_widen_marked(const unsigned char *__restrict__ src, const unsigned char *__restrict__ flag,
                                                      u32 *__restrict__ dst, u64 n) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
        dst[i] = (u32)src[i] | (flag[i] ? TOK_FLAG : 0u);
}

// ---- flag compaction: chunk offsets (3-kernel sum scan over the same tiles) ----
// DOCS: flags of a split buffer of documents (k_split_classify<true>): the chunk starts are doc_chunk_start's, and
// k_flag_scatter<true> writes them at their positions in the documents' own bytes (the boundary bytes taken out).  SPEC
// (with DOCS): the documents hold special-token occurrences, which stay (is_gap<true>)
template <bool DOCS, bool SPEC = false>
__global__ void __launch_bounds__(SP_THREADS) k_flag_reduce(const unsigned char *__restrict__ flag, u64 n, u32 *__restrict__ part,
                                                            const unsigned char *__restrict__ meta) {
    __shared__ u32 sm[SP_THREADS];
    const u64 base = (u64)blockIdx.x * SP_TILE + (u64)threadIdx.x * SP_ITEMS;
    u32 c = 0;
#pragma unroll
    for (int k = 0; k < SP_ITEMS; ++k) if (base + k < n) c += DOCS ? doc_chunk_start<SPEC>(flag, meta, base + k) : flag[base + k];
    sm[threadIdx.x] = c;
    __syncthreads();
    for (int o = SP_THREADS / 2; o > 0; o >>= 1) { if (threadIdx.x < (u32)o) sm[threadIdx.x] += sm[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) part[blockIdx.x] = sm[0];
}

__global__ void __launch_bounds__(1024) k_flag_scan_parts(const u32 *__restrict__ part, u64 *__restrict__ excl, u32 ntiles, u64 *total) {
    __shared__ u64 sm[1024];
    const u32 tid = threadIdx.x;
    const u32 per = (ntiles + 1023) / 1024;
    const u32 lo = min(ntiles, tid * per), hi = min(ntiles, lo + per);
    u64 sum = 0;
    for (u32 t = lo; t < hi; ++t) sum += part[t];
    sm[tid] = sum;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) { const u64 v = tid >= (u32)o ? sm[tid - o] : 0; __syncthreads(); sm[tid] += v; __syncthreads(); }
    u64 run = sm[tid] - sum;
    for (u32 t = lo; t < hi; ++t) { excl[t] = run; run += part[t]; }
    if (tid == 1023) *total = sm[1023];
}

// offs[] = text_base + position of every set flag (text_base: where this piece starts in the caller's text)
template <bool DOCS, bool SPEC = false>
__global__ void __launch_bounds__(SP_THREADS) k_flag_scatter(const unsigned char *__restrict__ flag, u64 n, const u64 *__restrict__ excl,
                                                             u64 *__restrict__ offs, u64 text_base, const unsigned char *__restrict__ meta,
                                                             const u64 *__restrict__ doff, u32 nd) {
    __shared__ u32 sm[SP_THREADS];
    const u32 tid = threadIdx.x;
    const u64 base = (u64)blockIdx.x * SP_TILE + (u64)tid * SP_ITEMS;
    u32 c = 0;
#pragma unroll
    for (int k = 0; k < SP_ITEMS; ++k) if (base + k < n) c += DOCS ? doc_chunk_start<SPEC>(flag, meta, base + k) : flag[base + k];
    sm[tid] = c;
    __syncthreads();
    for (int o = 1; o < SP_THREADS; o <<= 1) { const u32 v = tid >= (u32)o ? sm[tid - o] : 0; __syncthreads(); sm[tid] += v; __syncthreads(); }
    u64 dst = excl[blockIdx.x] + (sm[tid] - c);
    if constexpr (!DOCS) {
#pragma unroll
        for (int k = 0; k < SP_ITEMS; ++k) if (base + k < n && flag[base + k]) offs[dst++] = text_base + base + k;
    } else if (c) {
        u64 gaps = gaps_before(doff, nd, base);
        for (int k = 0; k < SP_ITEMS && base + k < n; ++k) {
            if (is_gap<SPEC>(meta, base + k)) ++gaps;
            else if (doc_chunk_start<SPEC>(flag, meta, base + k)) offs[dst++] = text_base + base + k - gaps;
        }
    }
}
