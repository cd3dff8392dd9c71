// k_special.cuh — the special-token front end of RegexTokenizer.encode (regex.py:123-164) on the device.
//
// The reference splits the text with re.split("(" + "|".join(re.escape(k) for k in special) + ")", text): leftmost
// match, the first alternative (dict order) that matches at a position wins, matches do not overlap; every special
// becomes one id, every part in between is encoded on its own (regex.py:152-163).  Here:
//   k_special_find    every text position where some special starts -> (position, lowest matching index), appended to a
//                     list (specials are rare; the host sorts the list and drops overlapped candidates left to right)
//   k_special_meta    bytes of the accepted occurrences get the boundary class SC_B in the splitter's class array, so
//                     the GPT-4 split treats the text on either side as separate texts (split_logic.h, WITH_B);
//                     <true> also marks them SM_SPEC (a split buffer of documents, DESIGN.md §16)
//   k_special_flags   chunk-start flags: one chunk per occurrence, and a chunk start right behind it
// The memoised encode (k_encode2.cuh) then needs nothing new: the specials are seeded into the memo table as chunks
// whose "encoding" is their single id (k_enc_seed_specials).
#pragma once
#include "common.cuh"
#include "split_logic.h"

#define SPEC_MAX 64          // specials per call (bit mask per first byte)
#define SPEC_MAX_LEN 48      // bytes per special = E2_LMAX (k_encode2.cuh): a special must fit one memo slot

struct SpecDev {
    const unsigned char *blob;   // the specials' bytes back to back
    const u32 *off;              // [k + 1] offsets into blob
    const u64 *first;            // [256] bit s set: special s starts with this byte
    int k;
};

__global__ void __launch_bounds__(256) k_special_find(const unsigned char *__restrict__ text, u64 n, SpecDev S,
                                                      u64 *__restrict__ list, u64 cap, ull *__restrict__ count) {
    __shared__ u64 s_first[256];
    s_first[threadIdx.x] = S.first[threadIdx.x];
    __syncthreads();
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u64 m = s_first[text[i]];
        while (m) {
            const int s = __ffsll((long long)m) - 1;
            m &= m - 1;
            const u32 lo = S.off[s], len = S.off[s + 1] - lo;
            if (i + len > n) continue;
            bool same = true;
            for (u32 j = 1; j < len && same; ++j) same = text[i + j] == S.blob[lo + j];
            if (same) {   // lowest index first = the alternative the regex tries first
                const ull q = atomicAdd(count, 1ull);
                if (q < cap) list[q] = (i << 8) | (u64)s;
                break;
            }
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
