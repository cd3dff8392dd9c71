// k_merge.cuh — the fused merge pass: merge(ids, pair, idx) of base.py:25-41 over the whole
// stream in ONE read and ONE write, plus the statistics delta that turns get_stats() of
// iteration i into get_stats() of iteration i+1 (DESIGN.md "Incremental statistics").
//
//   read  4*n bytes   (16-byte loads, each 128-token warp row is one coalesced 512 B request)
//   write 4*(n-c) bytes (compacted in shared memory, stored as full 128 B lines)
//
// Structure: persistent CTAs take 4096-token tiles from a ticket counter; per tile
//   1. mark   — m(p) = "a merge starts at p": w[p]==a, w[p+1]==b in the same chunk, and for
//               a==b the greedy left-to-right rule = even distance from the start of the run
//   2. scan   — kept tokens per 128-token warp row, tile total, exclusive tile offset by a
//               single-pass decoupled look-back over 64-bit tile descriptors (epoch-tagged,
//               never cleared)
//   3. compact— kept tokens are scattered to a padded shared-memory staging tile and streamed
//               out with coalesced stores
//   4. delta  — every merge start adds 1 to L[left neighbour], R[right neighbour] or ZZ
#pragma once
#include "common.cuh"

#define MG_THREADS 256
#define MG_ROWS 4
#define MG_ROW_TOKENS (MG_THREADS * 4)           // 1024 tokens per row (one uint4 per thread)
#define MG_TILE (MG_ROW_TOKENS * MG_ROWS)        // 4096 tokens
#define MG_WARPS (MG_THREADS / 32)
#define MG_WROWS (MG_WARPS * MG_ROWS)            // 32 warp rows of 128 tokens
#define MG_HALO 8                                // mark bits kept for 8 positions either side

// tile descriptor: epoch(26) | status(2) | value(36)
#define DESC_AGG 1ull
#define DESC_INC 2ull
__device__ __forceinline__ u64 desc_pack(u32 epoch, u64 status, u64 value) {
    return ((u64)(epoch & 0x3ffffffu) << 38) | (status << 36) | (value & 0xfffffffffull);
}
__device__ __forceinline__ u32 desc_epoch(u64 d) { return (u32)(d >> 38); }
__device__ __forceinline__ u32 desc_status(u64 d) { return (u32)(d >> 36) & 3u; }
__device__ __forceinline__ u64 desc_value(u64 d) { return d & 0xfffffffffull; }

// Decoupled look-back, executed by one full warp.  Returns the exclusive prefix of `agg`.
// NOTE: with hundreds of tiles in flight the chain of inclusive prefixes is the critical path
// of a contiguous compaction (the known-prefix frontier moves one 32-tile window per L2 round
// trip); the segmented stream of k_merge_seg.cuh exists to avoid it.  This contiguous kernel remains for pairs (a,a) and packing.
__device__ __forceinline__ u64 tile_lookback(u64 *desc, u32 tile, u32 epoch, u64 agg) {
    const u32 lane = lane_id();
    if (tile == 0) {
        if (lane == 0) st_volatile_u64(&desc[0], desc_pack(epoch, DESC_INC, agg));
        return 0;
    }
    if (lane == 0) st_volatile_u64(&desc[tile], desc_pack(epoch, DESC_AGG, agg));
    u64 excl = 0;
    long long top = (long long)tile - 1;
    for (;;) {
        const long long idx = top - (long long)lane;
        u64 d;
        bool ok;
        do {
            d = (idx >= 0) ? ld_volatile_u64(&desc[idx]) : desc_pack(epoch, DESC_INC, 0);
            ok = (desc_epoch(d) == (epoch & 0x3ffffffu)) && (desc_status(d) != 0);
        } while (!__all_sync(0xffffffffu, ok));
        const u32 inc = __ballot_sync(0xffffffffu, desc_status(d) == DESC_INC);
        u64 v = desc_value(d);
        if (inc) {
            const u32 first = __ffs(inc) - 1;  // nearest tile that already knows its inclusive prefix
            if (lane > first) v = 0;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        excl += v;
        if (inc) break;
        top -= 32;
    }
    if (lane == 0) st_volatile_u64(&desc[tile], desc_pack(epoch, DESC_INC, excl + agg));
    return excl;
}

// padded staging index: +1 word every 32 so that the stride-4 scatter is bank-conflict free
__device__ __forceinline__ u32 stage_idx(u32 i) { return i + (i >> 5); }
#define MG_STAGE_WORDS (MG_TILE + MG_TILE / 32 + 8)

// mark bit of stream position q, for q in [ts - MG_HALO, ts + MG_TILE + MG_HALO)
__device__ __forceinline__ u32 mark_bit(const unsigned char *s_mnib, long long q, u64 ts) {
    const u32 i = (u32)(q - (long long)ts + MG_HALO);
    return (s_mnib[i >> 2] >> (i & 3)) & 1u;
}

struct MergeArgs {
    Ctl *ctl;
    u32 *buf0, *buf1;
    u64 *desc;       // tile descriptors
    ull *delta;      // [0,V) L, [V,2V) R, [2V] ZZ; NULL = plain merge (no statistics)
    u32 V;
    int force;       // 1: run even if ctl->done / iter >= max_iter (single-step API)
    const unsigned char *xbase;   // sharded loop: exchange block (k_xchg.cuh) whose current-parity delta vector replaces `delta`
    u64 xstride;
};

// SAME = the kernel instance for pairs (a,a); both instances are launched back to back and the
// one that does not match the selected pair returns at once (keeps the run-parity code and its
// registers out of the common a != b instance).
template <bool SAME>
__global__ void __launch_bounds__(MG_THREADS, SAME ? 2 : 3) k_merge(MergeArgs A) {
    Ctl *ctl = A.ctl;
    if (!A.force && (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter)) return;
    if ((ctl->a == ctl->b) != SAME) return;

    __shared__ u32 s_stage[MG_STAGE_WORDS];
    __shared__ unsigned char s_mnib[MG_TILE / 4 + 2 * (MG_HALO / 4)];
    __shared__ u32 s_cnt[MG_WROWS];
    __shared__ u32 s_off[MG_WROWS];
    __shared__ unsigned char s_rowfull[MG_WROWS], s_rowout[MG_WROWS];
    __shared__ u64 s_tileoff;
    __shared__ u32 s_tile, s_agg, s_tilecin, s_lastout;

    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u64 n = ctl->n;
    const u32 *__restrict__ w = ctl->cur ? A.buf1 : A.buf0;
    u32 *__restrict__ out = ctl->cur ? A.buf0 : A.buf1;
    const u32 a = (u32)ctl->a, b = (u32)ctl->b, z = (u32)ctl->z;
    const u32 epoch = ctl->epoch;
    const u32 ntiles = (u32)((n + MG_TILE - 1) / MG_TILE);
    ull *const delta = A.xbase ? x_local_delta(A.xbase, A.xstride) : A.delta;

    for (;;) {
        __syncthreads();
        if (tid == 0) s_tile = atomicAdd(&ctl->merge_ticket, 1u);
        __syncthreads();
        const u32 tile = s_tile;
        if (tile >= ntiles) break;
        const u64 ts = (u64)tile * MG_TILE;
        const bool full_tile = (ts + MG_TILE + 8 <= n);

        // ---- load: 4 rows of one uint4 per thread, plus the token after the lane's four ----
        u32 t[MG_ROWS][4], nxt[MG_ROWS];
#pragma unroll
        for (int r = 0; r < MG_ROWS; ++r) {
            const u64 base = ts + (u64)r * MG_ROW_TOKENS + tid * 4;
            if (full_tile) {
                const uint4 q = *reinterpret_cast<const uint4 *>(w + base);
                t[r][0] = q.x; t[r][1] = q.y; t[r][2] = q.z; t[r][3] = q.w;
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) t[r][k] = (base + k < n) ? w[base + k] : TOK_SENTINEL;
            }
        }
#pragma unroll
        for (int r = 0; r < MG_ROWS; ++r) {
            const u64 base = ts + (u64)r * MG_ROW_TOKENS + tid * 4;
            u32 v = __shfl_down_sync(0xffffffffu, t[r][0], 1);
            if (lane == 31) v = (base + 4 < n) ? w[base + 4] : TOK_SENTINEL;
            nxt[r] = v;
        }

        // ---- mark ------------------------------------------------------------------------
        u32 mn[MG_ROWS];  // mark nibble: bit k = a merge starts at the lane's k-th token
        if constexpr (!SAME) {
#pragma unroll
            for (int r = 0; r < MG_ROWS; ++r) {
                u32 m = 0;
                m |= (((t[r][0] ^ a) & TOK_MASK) == 0 && t[r][1] == b) ? 1u : 0u;
                m |= (((t[r][1] ^ a) & TOK_MASK) == 0 && t[r][2] == b) ? 2u : 0u;
                m |= (((t[r][2] ^ a) & TOK_MASK) == 0 && t[r][3] == b) ? 4u : 0u;
                m |= (((t[r][3] ^ a) & TOK_MASK) == 0 && nxt[r] == b) ? 8u : 0u;
                mn[r] = m;
            }
            // halo marks: positions ts-2, ts-1 (left) and te, te+1 (right); other halo bits 0
            if (tid < 2 * (MG_HALO / 4)) s_mnib[tid < MG_HALO / 4 ? tid : MG_TILE / 4 + tid] = 0;
            __syncthreads();
            if (tid == 0) {
                u32 m = 0;
                for (int j = 1; j <= 2; ++j) {
                    const long long q = (long long)ts - j;
                    if (q >= 0 && (((w[q] ^ a) & TOK_MASK) == 0) && (u64)q + 1 < n && w[q + 1] == b) m |= 1u << (4 - j);
                }
                s_mnib[MG_HALO / 4 - 1] = (unsigned char)m;   // bits 2,3 = positions ts-2, ts-1
            } else if (tid == 32) {
                u32 m = 0;
                for (int j = 0; j < 2; ++j) {
                    const u64 q = ts + MG_TILE + j;
                    if (q + 1 < n && (((w[q] ^ a) & TOK_MASK) == 0) && w[q + 1] == b) m |= 1u << j;
                }
                s_mnib[MG_HALO / 4 + MG_TILE / 4] = (unsigned char)m;
            }
        } else {
            // a == b: e(q) = "q continues a run of a" = w[q]==a (same chunk) and id(w[q-1])==a.
            // A merge starts at p iff e(p+1) and the number of consecutive e's ending at p is
            // even (p is at even distance from the run start).  Parity is carried lane -> warp
            // row -> tile; a block of all-ones e bits has even length and passes parity through.
            u32 en[MG_ROWS], e4[MG_ROWS], lanecin[MG_ROWS], haslow[MG_ROWS];
#pragma unroll
            for (int r = 0; r < MG_ROWS; ++r) {
                const u64 base = ts + (u64)r * MG_ROW_TOKENS + tid * 4;
                u32 prv = __shfl_up_sync(0xffffffffu, t[r][3], 1);
                if (lane == 0) prv = (base > 0 && base - 1 < n) ? w[base - 1] : TOK_SENTINEL;
                u32 e = 0;
                e |= (t[r][0] == a && (prv & TOK_MASK) == a) ? 1u : 0u;
                e |= (t[r][1] == a && (t[r][0] & TOK_MASK) == a) ? 2u : 0u;
                e |= (t[r][2] == a && (t[r][1] & TOK_MASK) == a) ? 4u : 0u;
                e |= (t[r][3] == a && (t[r][2] & TOK_MASK) == a) ? 8u : 0u;
                en[r] = e;
                e4[r] = (nxt[r] == a && (t[r][3] & TOK_MASK) == a) ? 1u : 0u;
                u32 p = 0;  // parity chain assuming incoming parity 0
#pragma unroll
                for (int k = 0; k < 4; ++k) p = ((e >> k) & 1u) ? (p ^ 1u) : 0u;
                const u32 nf = __ballot_sync(0xffffffffu, e != 0xfu);  // lanes that reset the chain
                const u32 lower = nf & ((1u << lane) - 1u);
                haslow[r] = lower != 0;
                const u32 src = lower ? (31 - __clz(lower)) : 0;
                lanecin[r] = __shfl_sync(0xffffffffu, p, src);
                const u32 topsrc = nf ? (31 - __clz(nf)) : 0;
                const u32 rowout = __shfl_sync(0xffffffffu, p, topsrc);
                if (lane == 0) { s_rowfull[r * MG_WARPS + warp] = (nf == 0); s_rowout[r * MG_WARPS + warp] = (unsigned char)rowout; }
            }
            if (warp == 0) {  // parity of the run of e's that ends just before the tile
                u32 cnt = 0;
                long long q = (long long)ts - 1;
                for (;;) {
                    const long long pos = q - (long long)lane;
                    const bool e = pos >= 1 && (u64)pos < n && w[pos] == a && (w[pos - 1] & TOK_MASK) == a;
                    const u32 bal = __ballot_sync(0xffffffffu, e);
                    if (bal == 0xffffffffu) { cnt += 32; q -= 32; continue; }
                    cnt += __ffs(~bal) - 1;
                    break;
                }
                if (lane == 0) s_tilecin = cnt & 1u;
            }
            if (tid < 2 * (MG_HALO / 4)) s_mnib[tid < MG_HALO / 4 ? tid : MG_TILE / 4 + tid] = 0;
            __syncthreads();
            u32 lastout = 0;
#pragma unroll
            for (int r = 0; r < MG_ROWS; ++r) {
                const int wr = r * MG_WARPS + warp;
                u32 rowcin = s_tilecin;
                for (int j = wr - 1; j >= 0; --j) if (!s_rowfull[j]) { rowcin = s_rowout[j]; break; }
                u32 p = haslow[r] ? lanecin[r] : rowcin;
                u32 m = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    p = ((en[r] >> k) & 1u) ? (p ^ 1u) : 0u;          // parity of the e-run ending at token k
                    const u32 enext = (k < 3) ? ((en[r] >> (k + 1)) & 1u) : e4[r];
                    m |= (enext && !p) ? (1u << k) : 0u;
                }
                mn[r] = m;
                if (r == MG_ROWS - 1) lastout = p;  // parity at the lane's last token of the last row
            }
            if (tid == MG_THREADS - 1) s_lastout = lastout;  // parity at position te-1
            if (tid == 0) {
                // left halo: P(ts-1) = s_tilecin.  m(ts-1) = e(ts) && !P(ts-1);
                // m(ts-2) = e(ts-1) && P(ts-1)   (P(ts-2) = P(ts-1)^1 when e(ts-1))
                const u32 pc = s_tilecin;
                const bool e_ts = ts >= 1 && ts < n && w[ts] == a && (w[ts - 1] & TOK_MASK) == a;
                const bool e_tsm1 = ts >= 2 && w[ts - 1] == a && (w[ts - 2] & TOK_MASK) == a;
                u32 m = 0;
                if (e_ts && !pc) m |= 8u;      // position ts-1
                if (e_tsm1 && pc) m |= 4u;     // position ts-2
                s_mnib[MG_HALO / 4 - 1] = (unsigned char)m;
            }
            __syncthreads();
            if (tid == 0) {
                // right halo: continue the chain past te-1
                const u64 te = ts + MG_TILE;
                u32 p = s_lastout, m = 0;
                // e(q) for q = te, te+1, te+2
                bool e[3];
                for (int j = 0; j < 3; ++j) {
                    const u64 q = te + j;
                    e[j] = q < n && w[q] == a && (w[q - 1] & TOK_MASK) == a;
                }
                p = e[0] ? (p ^ 1u) : 0u;            // P(te)
                if (e[1] && !p) m |= 1u;             // m(te)
                p = e[1] ? (p ^ 1u) : 0u;            // P(te+1)
                if (e[2] && !p) m |= 2u;             // m(te+1)
                s_mnib[MG_HALO / 4 + MG_TILE / 4] = (unsigned char)m;
            }
        }
        // publish mark nibbles
#pragma unroll
        for (int r = 0; r < MG_ROWS; ++r) s_mnib[MG_HALO / 4 + r * (MG_ROW_TOKENS / 4) + tid] = (unsigned char)mn[r];
        __syncthreads();

        // ---- scan: kept tokens per lane / warp row ------------------------------------------
        u32 keep[MG_ROWS], lpre[MG_ROWS];
#pragma unroll
        for (int r = 0; r < MG_ROWS; ++r) {
            const u64 base = ts + (u64)r * MG_ROW_TOKENS + tid * 4;
            const u32 prevn = s_mnib[MG_HALO / 4 + r * (MG_ROW_TOKENS / 4) + tid - 1];
            const u32 dropped = ((mn[r] << 1) | (prevn >> 3)) & 0xfu;  // token k is the 2nd half of a merge
            u32 valid = 0xfu;
            if (!full_tile) { const long long rem = (long long)n - (long long)base; valid = rem >= 4 ? 0xfu : (rem <= 0 ? 0u : ((1u << rem) - 1u)); }
            keep[r] = ~dropped & valid;
            const u32 c = __popc(keep[r]);
            // exclusive prefix of c over the lanes of the warp row
            u32 incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const u32 y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += y; }
            lpre[r] = incl - c;
            if (lane == 31) s_cnt[r * MG_WARPS + warp] = incl;
        }
        __syncthreads();

        // ---- tile offset: warp 0 scans the 32 warp-row counts, publishes, looks back --------
        if (warp == 0) {
            const u32 c = s_cnt[lane];
            u32 incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const u32 y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += y; }
            s_off[lane] = incl - c;
            const u32 agg = __shfl_sync(0xffffffffu, incl, 31);
            const u64 excl = tile_lookback(A.desc, tile, epoch, (u64)agg);
            if (lane == 0) {
                s_tileoff = excl; s_agg = agg;
                if (tile == ntiles - 1) ctl->n_next = excl + agg;
            }
        }
        __syncthreads();
        const u64 tileoff = s_tileoff;
        const u32 agg = s_agg;

        // ---- compact: scatter kept tokens into the padded staging tile ----------------------
#pragma unroll
        for (int r = 0; r < MG_ROWS; ++r) {
            u32 dst = s_off[r * MG_WARPS + warp] + lpre[r];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if ((keep[r] >> k) & 1u) {
                    const u32 v = ((mn[r] >> k) & 1u) ? (z | (t[r][k] & TOK_FLAG)) : t[r][k];
                    s_stage[stage_idx(dst)] = v;
                    ++dst;
                }
            }
        }

        // ---- delta: statistics change caused by each merge start ------------------------------
        if (delta) {
#pragma unroll
            for (int r = 0; r < MG_ROWS; ++r) {
                if (mn[r]) {
                    const u64 base = ts + (u64)r * MG_ROW_TOKENS + tid * 4;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if ((mn[r] >> k) & 1u) {
                            const u64 p = base + k;
                            // left neighbour: pair (x,a) at p-1 disappears, (x,z) appears — unless the
                            // left neighbour is itself the tail of a merge (then it is that merge's
                            // right-hand case) or p starts a chunk
                            if (p >= 1 && !(t[r][k] & TOK_FLAG) && !mark_bit(s_mnib, (long long)p - 2, ts)) {
                                const u32 x = w[p - 1] & TOK_MASK;
                                atomicAdd(&delta[x], 1ull);
                            }
                            // right neighbour y = token after the pair
                            if (p + 2 < n) {
                                const u32 y = w[p + 2];
                                if (!(y & TOK_FLAG)) {
                                    if (mark_bit(s_mnib, (long long)p + 2, ts)) atomicAdd(&delta[2 * (u64)A.V], 1ull);
                                    else atomicAdd(&delta[(u64)A.V + y], 1ull);
                                }
                            }
                        }
                    }
                }
            }
        }
        __syncthreads();

        // ---- stream the compacted tile out -----------------------------------------------------
#pragma unroll
        for (int j = 0; j < MG_TILE / MG_THREADS; ++j) {
            const u32 i = j * MG_THREADS + tid;
            if (i < agg) out[tileoff + i] = s_stage[stage_idx(i)];
        }
    }

    // ---- exit: the last CTA out flips the ping-pong buffers and resets the tickets ------------
    if (tid == 0) {
        __threadfence();
        const u32 e = atomicAdd(&ctl->merge_exit, 1u);
        if (e == gridDim.x - 1) {
            __threadfence();
            const u64 n_new = ntiles ? *(volatile u64 *)&ctl->n_next : 0;
            ctl->sum_in += n; ctl->sum_out += n_new;
            ctl->n = n_new;
            ctl->cur ^= 1u;
            ctl->iter += 1;
            ctl->epoch += 1;
            ctl->merge_ticket = 0; ctl->merge_exit = 0;
        }
    }
}
