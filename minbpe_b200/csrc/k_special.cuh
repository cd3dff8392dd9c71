// k_special.cuh — the special-token front end of RegexTokenizer.encode (regex.py:123-164) on the device.
//
// The reference splits the text with re.split("(" + "|".join(re.escape(k) for k in special) + ")", text): leftmost
// match, the first alternative (dict order) that matches at a position wins, matches do not overlap; every special
// becomes one id, every part in between is encoded on its own (regex.py:152-163).  Here:
//   k_special_find    every text position where some special starts -> (position, lowest matching index), appended to a
//                     list (specials are rare; the host sorts the list and drops overlapped candidates left to right).
//                     A walk down a byte trie of the set (below): at most SPEC_MAX_LEN levels per position, whatever the
//                     number of specials
//   k_special_meta    bytes of the accepted occurrences get the boundary class SC_B in the splitter's class array, so
//                     the GPT-4 split treats the text on either side as separate texts (split_logic.h, WITH_B);
//                     <true> also marks them SM_SPEC (a split buffer of documents, DESIGN.md §16)
//   k_special_flags   chunk-start flags: one chunk per occurrence, and a chunk start right behind it
// The memoised encode (k_encode2.cuh) then needs nothing new: the specials are seeded into the memo table as chunks
// whose "encoding" is their single id (k_enc_seed_specials).
//
// The trie (DESIGN.md §19), built on the host by spec_set.  A node is reached through an edge word (u64):
//   bits  0..7   the byte that labels the edge
//   bits  8..16  the node's number of children (0..256)
//   bits 17..38  the index in `edge` of the node's first child edge; its children's edges are contiguous, sorted by byte
//   bits 39..55  the LOWEST index of a special that ends at the node (SPEC_NONE: none)
// The root's children are root[256], one edge word per first byte (a byte no special starts with: SPEC_ABSENT); they live
// in shared memory and are the first-byte filter.  Every deeper edge is in `edge`, read-only.  The winner at position i is
// the minimum of the lowest indices on the path that text[i:] spells: the first special in dict order that matches there.
#pragma once
#include "common.cuh"
#include "split_logic.h"

#define SPEC_MAX 65536       // specials per call: an index fits the 16 low bits of a candidate
#define SPEC_MAX_LEN 48      // bytes per special = E2_LMAX (k_encode2.cuh): a special must fit one memo slot
#define SPEC_NONE 0x1ffffu   // no special ends at this node (greater than every index)
#define SPEC_ABSENT ((u64)SPEC_NONE << 39)   // no child: no children, no special
#define SPEC_MAX_EDGES (1u << 22)            // edge indices are 22 bits; a set has at most SPEC_MAX * SPEC_MAX_LEN edges
static_assert((u64)SPEC_MAX * SPEC_MAX_LEN < SPEC_MAX_EDGES, "trie edge index field");

__host__ __device__ __forceinline__ u32 spec_e_byte(u64 e) { return (u32)(e & 0xffu); }
__host__ __device__ __forceinline__ u32 spec_e_kids(u64 e) { return (u32)(e >> 8) & 0x1ffu; }
__host__ __device__ __forceinline__ u32 spec_e_first(u64 e) { return (u32)(e >> 17) & (SPEC_MAX_EDGES - 1); }
__host__ __device__ __forceinline__ u32 spec_e_best(u64 e) { return (u32)(e >> 39) & SPEC_NONE; }
__host__ __device__ __forceinline__ u64 spec_e_make(u32 byte, u32 kids, u32 first, u32 best) {
    return (u64)byte | ((u64)kids << 8) | ((u64)first << 17) | ((u64)best << 39);
}

struct SpecDev {
    const u64 *root;   // [256] edge words of the root's children
    const u64 *edge;   // every deeper edge word
};

// the child of the node with edge word e along byte c: its edge word, or SPEC_ABSENT
__host__ __device__ __forceinline__ u64 spec_child(const u64 *__restrict__ edge, u64 e, u32 c) {
    u32 lo = spec_e_first(e), hi = lo + spec_e_kids(e);
    const u32 end = hi;
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
#ifdef __CUDA_ARCH__
        const u32 b = spec_e_byte(__ldg(&edge[mid]));
#else
        const u32 b = spec_e_byte(edge[mid]);
#endif
        if (b < c) lo = mid + 1; else hi = mid;
    }
    if (lo == end) return SPEC_ABSENT;
#ifdef __CUDA_ARCH__
    const u64 f = __ldg(&edge[lo]);
#else
    const u64 f = edge[lo];
#endif
    return spec_e_byte(f) == c ? f : SPEC_ABSENT;
}

// candidates: position << 16 | index (positions are below 2^32: spec_find checks)
__global__ void __launch_bounds__(256) k_special_find(const unsigned char *__restrict__ text, u64 n, SpecDev S,
                                                      u64 *__restrict__ list, u64 cap, ull *__restrict__ count) {
    __shared__ u64 s_root[256];
    s_root[threadIdx.x] = S.root[threadIdx.x];
    __syncthreads();
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 e = s_root[text[i]];
        u32 best = spec_e_best(e);
        for (u64 j = i + 1; j < n && spec_e_kids(e); ++j) {   // at most SPEC_MAX_LEN - 1 levels: the trie's depth
            e = spec_child(S.edge, e, text[j]);
            best = min(best, spec_e_best(e));
        }
        if (best != SPEC_NONE) {
            const ull q = atomicAdd(count, 1ull);
            if (q < cap) list[q] = (i << 16) | (u64)best;
        }
    }
}

// accepted occurrences: hit[j] = position << 8 | length.  DOCS: a split buffer of documents (bpe_encode_docs), whose gaps
// have class SC_B as well: the occurrence's bytes also get SM_SPEC, so that the compaction (k_flag_reduce / k_flag_scatter
// <true, true>) tells them apart from the gaps
template <bool DOCS>
__global__ void k_special_meta(unsigned char *__restrict__ meta, const u64 *__restrict__ hit, u64 m) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (u64)gridDim.x * blockDim.x) {
        const u64 pos = hit[j] >> 8;
        const u32 len = (u32)(hit[j] & 0xffu);
        for (u32 t = 0; t < len; ++t) meta[pos + t] = (unsigned char)((meta[pos + t] & SM_START) | SC_B | (DOCS ? SM_SPEC : 0u));
    }
}

__global__ void k_special_flags(unsigned char *__restrict__ flag, const u64 *__restrict__ hit, u64 m, u64 n) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (u64)gridDim.x * blockDim.x) {
        const u64 pos = hit[j] >> 8;
        const u32 len = (u32)(hit[j] & 0xffu);
        flag[pos] = 1;
        for (u32 t = 1; t < len; ++t) flag[pos + t] = 0;
        if (pos + len < n) flag[pos + len] = 1;     // the next part (or the next special) starts a chunk
    }
}
