// k_merge_seg.cuh — the fused merge pass (base.py:25-41 + the statistics delta) for a != b on the
// SEGMENTED stream.  One WARP owns one 512-token segment at a time: 16 tokens per lane in
// registers, compacted in place, independently of every other segment.  There is no prefix sum
// across segments and no block-level synchronisation in the loop: every warp is its own pipeline.
//
//   read   4 * count bytes per segment        (one 1-D bulk async copy, TMA / UBLKCP, into the
//                                              warp's private mbarrier ring, MS_STAGES deep)
//   write  only from the first 128-token row that changed to the new end of the segment
//          (16-byte stores, same address range); nothing for an untouched segment
//   + 32-byte edge records per segment (first 3 / last 2 tokens, count), double-buffered, so a
//     warp can see across its segment boundaries without reading a body that another warp rewrites
//
// Work distribution: a ticket (one atomic) hands a warp MS_BATCH consecutive segments; the warp
// loads their edge records once, then keeps MS_STAGES-1 bulk copies in flight ahead of the segment
// it is working on.  The marking and delta rules are the ones documented in k_merge.cuh.
//
// Batched pass (bpe_train's loop, SegArgs.batched, ctl->nk > 1): up to BATCH_MAX token-disjoint pairs that
// k_select_batch proved to be the next merges are marked and compacted in the same single pass, with one delta
// vector per member (DESIGN.md "Batched merges").  The segment loop is instantiated per member count NK (the kernel
// switches once on the block-uniform ctl->nk): the members' ids live in registers and every member test is unrolled.
//
// Statistics delta per warp: the segment's merge starts go to a per-warp list (warp prefix of the lanes' counts), the
// warp takes them 32 at a time, one per lane, and equal delta indices are folded across the warp with
// __match_any_sync, so the CTA's delta cache sees one shared atomic per distinct index and round.
#pragma once
#include "common.cuh"
#include "k_merge.cuh"
#include "k_seg.cuh"

#ifndef MS_WARPS
#define MS_WARPS 8
#endif
#define MS_THREADS (MS_WARPS * 32)
#ifndef MS_STAGES
#define MS_STAGES 2
#endif
#ifndef MS_MINBLOCKS
#define MS_MINBLOCKS 4
#endif
#ifndef MS_DCACHE_LOG2
#define MS_DCACHE_LOG2 9
#endif
#ifndef MS_BATCH
#define MS_BATCH 8                          // consecutive segments per ticket
#endif
#define MS_PAD 4                            // body starts at word 4 of a stage (16-byte aligned); s[-1], s[-2] = previous tokens
#define MS_SW (SEG_TOKENS + 8)              // words per stage: pad, body, three following tokens
#define MS_META 16                          // per stage: P0 P1 N0 N1 N2 seg count - | the segment's own edge record
#define MS_BE (MS_BATCH + 2)                // edge records of a batch and of the segment on either side
#define MS_DCACHE (1 << MS_DCACHE_LOG2)     // slots of the per-CTA delta cache (shared memory)
#define MS_LIST (SEG_TOKENS / 2)            // merge starts of a segment: never two adjacent tokens, so at most half of them
#define MS_WARP_WORDS (MS_STAGES * MS_SW + MS_STAGES * MS_META + MS_BE * 8 + MS_LIST)
#define MS_SMEM_BYTES (MS_WARPS * MS_WARP_WORDS * 4 + MS_WARPS * MS_STAGES * 8 + MS_DCACHE * 8 + 16)
#define MS_INVALID 0xffffffffu
static_assert(SEG_TOKENS == 512, "k_merge_seg: a lane owns 4 rows x 4 tokens of a 512-token segment");
static_assert((MS_SW * 4) % 16 == 0 && (MS_WARP_WORDS * 4) % 16 == 0, "bulk-copy destinations must stay 16-byte aligned");

// delta[idx] += cnt through a CTA-private shared-memory cache: the same few neighbour ids are hit by
// almost every merge of a dense iteration (global same-address atomics serialise in L2); the
// persistent CTA folds them here and flushes once at exit.
__device__ __noinline__ void delta_cache_add(u32 *s_dkey, u32 *s_dcnt, ull *delta, u32 idx, u32 cnt) {
    u32 slot = (idx * 2654435761u) >> (32 - MS_DCACHE_LOG2);
#pragma unroll 1
    for (int probe = 0; probe < 4; ++probe) {
        u32 k = reinterpret_cast<volatile u32 *>(s_dkey)[slot];
        if (k == 0xffffffffu) {
            const u32 old = atomicCAS(&s_dkey[slot], 0xffffffffu, idx);
            k = (old == 0xffffffffu) ? idx : old;
        }
        if (k == idx) { atomicAdd(&s_dcnt[slot], cnt); return; }
        slot = (slot + 1) & (MS_DCACHE - 1);
    }
    atomicAdd(&delta[idx], (ull)cnt);   // cache neighbourhood full
}

// The members of a pass: member j is the pair (a[j], b[j]) -> z + j.  NK = 1: the one pair (a, b) -> z.  The 2·NK ids
// are all distinct (k_select_batch), so a token is the left token of at most one member.
template <int NK>
struct Members {
    u32 a[NK], b[NK];
};

// the member whose left id is id(x) (NK: none); bj = its right id
template <int NK>
__device__ __forceinline__ u32 member_of(const Members<NK> &M, u32 x, u32 &bj) {
    u32 j = NK;
    bj = 0;
#pragma unroll
    for (int k = 0; k < NK; ++k)
        if ((x & TOK_MASK) == M.a[k]) { j = k; bj = M.b[k]; }
    return j;
}
// a merge starts at the token pair (x, y).  NK > 1: the right id of the member whose left id is id(x) is selected, then
// compared once (0x7fffffff: no member; no token word holds it, the sentinel carries the flag)
template <int NK>
__device__ __forceinline__ bool starts(const Members<NK> &M, u32 x, u32 y) {
    if constexpr (NK == 1) {
        return ((x ^ M.a[0]) & TOK_MASK) == 0 && y == M.b[0];
    } else {
        x &= TOK_MASK;
        u32 r = TOK_MASK;
#pragma unroll
        for (int k = 0; k < NK; ++k) r = x == M.a[k] ? M.b[k] : r;
        return y == r;
    }
}
// the member that starts at the token pair (x, y) (NK: none)
template <int NK>
__device__ __forceinline__ u32 start_of(const Members<NK> &M, u32 x, u32 y) {
    u32 bj;
    const u32 j = member_of(M, x, bj);
    return (j < NK && y == bj) ? j : NK;
}

// statistics delta of the merge that starts at the token at shared address `at` (rules: k_merge.cuh), as the two delta
// indices it adds 1 to (MS_INVALID: none).  The words at s[-2..-1] and s[count..count+2] hold the neighbouring segments'
// tokens (or the sentinel).  Member j is applied to the stream as the members before it have left it: a neighbour that
// starts a merge of an earlier member m is z+m by then, one that starts a merge of a later member is still itself.
// Delta vector of member j: [j(2V+1), (j+1)(2V+1)), laid out as for one merge.
template <int NK>
__device__ __forceinline__ void start_delta(u32 at, const Members<NK> &M, u32 z, u32 V, u32 &li, u32 &ri) {
    const u32 t0 = lds32(at), tm1 = lds32o<-4>(at), tm2 = lds32o<-8>(at), tp2 = lds32o<8>(at), tp3 = lds32o<12>(at);
    u32 bj;
    const u32 j = NK == 1 ? 0u : member_of(M, t0, bj);
    const u32 ml = start_of(M, tm2, tm1);   // member starting two tokens earlier
    const u32 mr = start_of(M, tp2, tp3);   // member starting two tokens later
    const u32 base = j * (2u * V + 1u);
    li = (tm1 != TOK_SENTINEL && !(t0 & TOK_FLAG) && ml != j) ? base + (ml < j ? z + ml : tm1 & TOK_MASK) : MS_INVALID;
    ri = !(tp2 & TOK_FLAG)   // also false for the sentinel (end of stream)
             ? base + (mr == j ? 2u * V : V + (mr < j ? z + mr : tp2)) : MS_INVALID;
}

// one delta index per lane (MS_INVALID: none), added to the cache once per distinct index: the lowest lane of each
// group of equal indices adds the group's size
__device__ __forceinline__ void delta_fold_add(u32 idx, u32 lane, u32 *s_dkey, u32 *s_dcnt, ull *delta) {
    const u32 grp = __match_any_sync(0xffffffffu, idx);
    if (idx != MS_INVALID && lane == (u32)(__ffs(grp) - 1)) delta_cache_add(s_dkey, s_dcnt, delta, idx, (u32)__popc(grp));
}

// statistics delta of a segment's merge starts, per warp.  mall: this lane's starts, bit 4r+i = token 4·lane+i of row r.
// The list holds the starts' byte offsets from the segment's token 0, in lane order.
template <int NK>
__device__ __forceinline__ void segment_delta(u32 s_a, u32 list_a, u32 lane, u32 mall, const Members<NK> &M, u32 z, u32 V,
                                              u32 *s_dkey, u32 *s_dcnt, ull *delta) {
    const u32 own = __popc(mall);
    u32 incl = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const u32 v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (u32)o) incl += v;
    }
    const u32 total = __shfl_sync(0xffffffffu, incl, 31);
    u32 p = list_a + (incl - own) * 4u;
#pragma unroll 1
    while (mall) {
        const u32 bit = __ffs(mall) - 1;
        mall &= mall - 1;
        sts32(p, (bit >> 2) * 512u + lane * 16u + (bit & 3u) * 4u);
        p += 4u;
    }
    __syncwarp();
#pragma unroll 1
    for (u32 base = 0; base < total; base += 32u) {   // warp-uniform
        u32 li = MS_INVALID, ri = MS_INVALID;
        if (base + lane < total) start_delta(s_a + lds32(list_a + (base + lane) * 4u), M, z, V, li, ri);
        delta_fold_add(li, lane, s_dkey, s_dcnt, delta);
        delta_fold_add(ri, lane, s_dkey, s_dcnt, delta);
    }
    __syncwarp();   // the list is rewritten by the next segment
}

struct SegArgs {
    Ctl *ctl;
    u32 *buf0, *buf1;
    Edge *e0, *e1;
    ull *delta;   // [0,V) L, [V,2V) R, [2V] ZZ; NULL = plain merge.  Batched: one such vector per member
    u32 V;
    int force;
    int batched;  // apply the ctl->nk members k_select_batch chose (bpe_train's loop); 0: the one pair (a, b)
    const unsigned char *xbase;   // sharded loop: the rank's exchange block (k_xchg.cuh); the delta vector is then
    u64 xstride;                  // the one of the current round's parity inside it, and `delta` is ignored
};

// one row (128 tokens, 4 per lane): merge starts m, kept tokens, replaced tokens written back to t[].
// Member j of M becomes z + j.  up: in, lane 31's starts of the row before (bit 3: at its last token); out, this row's.
template <int R, int NK>
__device__ __forceinline__ void mark_row(u32 la, u32 lane, u32 count, const Members<NK> &M, u32 z, u32 (&t)[4],
                                         u32 &mn, u32 &keep, u32 &dirty, u32 &up) {
    const uint4 q = lds128o<R * 512>(la);
    const u32 nx = lds32o<R * 512 + 16>(la);
    t[0] = q.x; t[1] = q.y; t[2] = q.z; t[3] = q.w;
    const u32 m = (starts(M, t[0], t[1]) ? 1u : 0u) | (starts(M, t[1], t[2]) ? 2u : 0u) | (starts(M, t[2], t[3]) ? 4u : 0u) |
                  (starts(M, t[3], nx) ? 8u : 0u);
    // a start at the token in front of this lane's first one: the lane before tested that pair (lane 0: lane 31, row before)
    const u32 pm = __shfl_sync(0xffffffffu, lane == 31 ? up : m, (lane + 31) & 31) >> 3;
    up = m;
    const u32 d = ((m << 1) | pm) & 0xfu;   // dropped: the token after a merge start
    u32 valid = 0xfu;
    if (R * 128u + 128u > count) {          // warp-uniform: the row that holds the end of the segment
        const int rem = (int)count - (int)(R * 128 + lane * 4);
        valid = rem >= 4 ? 0xfu : (rem <= 0 ? 0u : ((1u << rem) - 1u));
    }
    mn = m & valid;                         // a merge only starts at a token this segment owns
    keep = ~d & valid;
    dirty |= (mn | (keep ^ valid)) ? (1u << R) : 0u;
    if (mn) {                               // few lanes: the merged token takes its place in the registers
        auto zof = [&](u32 x) {
            u32 id = z;
#pragma unroll
            for (int j = 1; j < NK; ++j) if ((x & TOK_MASK) == M.a[j]) id = z + j;
            return id | (x & TOK_FLAG);
        };
        if (mn & 1u) t[0] = zof(t[0]);
        if (mn & 2u) t[1] = zof(t[1]);
        if (mn & 4u) t[2] = zof(t[2]);
        if (mn & 8u) t[3] = zof(t[3]);
    }
}

// write the kept tokens of one row to their compacted place (word offset `off` of the stage)
__device__ __forceinline__ void scatter_row(u32 s_a, u32 lane, u32 off, u32 row_kept, u32 lane_excl, u32 kp, const u32 (&t)[4]) {
    if (row_kept == 128u) {                 // warp-uniform: nothing dropped in this row, it only moves
        const u32 p = s_a + ((off + 4u * lane) << 2);
        if ((off & 3u) == 0) sts128(p, t[0], t[1], t[2], t[3]);
        else { sts32(p, t[0]); sts32o<4>(p, t[1]); sts32o<8>(p, t[2]); sts32o<12>(p, t[3]); }
    } else {
        u32 p = s_a + ((off + lane_excl) << 2);
        if (kp & 1u) sts32(p, t[0]);
        p += (kp << 2) & 4u;
        if (kp & 2u) sts32(p, t[1]);
        p += (kp << 1) & 4u;
        if (kp & 4u) sts32(p, t[2]);
        p += kp & 4u;
        if (kp & 8u) sts32(p, t[3]);
    }
}

// The pass over the segments with NK members (k_merge_seg below picks NK).
template <bool LIST, int NK>
__device__ __forceinline__ void merge_seg_pass(const SegArgs &A) {
    Ctl *ctl = A.ctl;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    u32 *s_warp = reinterpret_cast<u32 *>(smem_raw);                              // [MS_WARPS][MS_WARP_WORDS]
    u64 *s_bar = reinterpret_cast<u64 *>(s_warp + MS_WARPS * MS_WARP_WORDS);      // [MS_WARPS][MS_STAGES]
    u32 *s_dkey = reinterpret_cast<u32 *>(s_bar + MS_WARPS * MS_STAGES);          // [MS_DCACHE] delta index or 0xffffffff
    u32 *s_dcnt = s_dkey + MS_DCACHE;                                             // [MS_DCACHE]
    ull *s_drops = reinterpret_cast<ull *>(s_dcnt + MS_DCACHE);

    const u32 FULL = 0xffffffffu;
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u64 n = ctl->n;
    u32 *__restrict__ w = ctl->cur ? A.buf1 : A.buf0;                 // compacted in place
    const Edge *__restrict__ e_cur = ctl->edge_cur ? A.e1 : A.e0;
    Edge *__restrict__ e_next = ctl->edge_cur ? A.e0 : A.e1;
    const u32 z = (u32)ctl->z;
    const u32 nseg = ctl->nseg;
    Members<NK> M;
#pragma unroll
    for (int j = 0; j < NK; ++j) {
        M.a[j] = j ? (u32)ctl->bat_a[j] : (u32)ctl->a;
        M.b[j] = j ? (u32)ctl->bat_b[j] : (u32)ctl->b;
    }
    ull *const delta = A.xbase ? x_local_delta(A.xbase, A.xstride) : A.delta;
    const u32 *__restrict__ cand = LIST ? reinterpret_cast<const u32 *>(ctl->cand_ptr) : nullptr;
    const u32 n_cand = LIST ? ctl->n_cand : 0u;

    // this warp's private shared memory, as 32-bit shared-window byte addresses
    const u32 ws_a = smem_addr(s_warp + warp * MS_WARP_WORDS);   // [MS_STAGES][MS_SW] staging ring
    const u32 wmeta_a = ws_a + MS_STAGES * MS_SW * 4;            // [MS_STAGES][MS_META]
    const u32 wbe_a = wmeta_a + MS_STAGES * MS_META * 4;         // [MS_BE][8] edge records batch_seg-1 .. batch_seg+MS_BATCH
    const u32 wlist_a = wbe_a + MS_BE * 32;                      // [MS_LIST] merge starts of the segment (segment_delta)
    const u32 wbar_a = smem_addr(s_bar + warp * MS_STAGES);

    if (lane == 0) {
        for (int s = 0; s < MS_STAGES; ++s) mbar_init(s_bar + warp * MS_STAGES + s, 1);
        fence_mbar_init();
    }
    for (u32 i = tid; i < MS_DCACHE; i += MS_THREADS) { s_dkey[i] = 0xffffffffu; s_dcnt[i] = 0; }
    if (tid == 0) *s_drops = 0;
    __syncthreads();

    // ---- issue side: next non-empty segment of this warp -> bulk copy into `stage` ----
    u32 batch_seg = 0, batch_pos = MS_BATCH;   // warp-uniform
    u32 list_next = blockIdx.x * MS_WARPS + warp;   // LIST: this warp's next entry of the candidate list
    // byte offset inside the batch's edge-record window (relative to record k) of the word lane l copies
    // into meta[l]: meta[0..4] = P0 P1 N0 N1 N2 = previous record's l[1], l[0], next record's f[0..2];
    // meta[8..15] = the segment's own record (for the untouched case); meta[5] = seg, meta[6] = count
    const u32 meta_src = 4u * (lane == 0 ? 4u : lane == 1 ? 3u : lane < 5 ? 14u + lane : lane < 8 ? 0u : lane < 16 ? lane : 0u);
    bool exhausted = false;
    auto issue = [&](u32 stage) {
        const u32 meta_a = wmeta_a + stage * (MS_META * 4);
        for (;;) {
            if (exhausted) {
                if (lane == 0) sts32o<20>(meta_a, MS_INVALID);
                __syncwarp();
                return;
            }
            if (batch_pos == MS_BATCH) {
                u32 tk = 0;
                if (LIST) {
                    // one candidate at a time, list entries dealt out round-robin over all warps of the grid (a ticket per
                    // entry would be one atomic on one address per segment); its record and its neighbours' go to the last
                    // three slots of the window, where the code below finds those of the last segment of a batch
                    tk = list_next; list_next += gridDim.x * MS_WARPS;
                    if (tk >= n_cand) { exhausted = true; continue; }
                    batch_seg = cand[tk] - (MS_BATCH - 1); batch_pos = MS_BATCH - 1;
                } else {
                    if (lane == 0) tk = atomicAdd(&ctl->merge_ticket, 1u);
                    tk = __shfl_sync(FULL, tk, 0);
                    if ((u64)tk * MS_BATCH >= nseg) { exhausted = true; continue; }
                    batch_seg = tk * MS_BATCH; batch_pos = 0;
                }
                if (LIST ? (lane >= MS_BATCH - 1 && lane < MS_BE) : (lane < MS_BE)) {
                    const long long idx = (LIST ? (long long)(int)batch_seg : (long long)batch_seg) - 1 + lane;   // LIST: batch_seg may have wrapped below 0
                    uint4 q0, q1;   // f0 f1 f2 l0 | l1 count pad pad
                    if (idx >= 0 && idx < (long long)nseg) {
                        const uint4 *p = reinterpret_cast<const uint4 *>(&e_cur[idx]);
                        q0 = p[0]; q1 = p[1];
                    } else {        // past either end of the stream: a "long" neighbour made of sentinels
                        q0 = make_uint4(TOK_SENTINEL, TOK_SENTINEL, TOK_SENTINEL, TOK_SENTINEL);
                        q1 = make_uint4(TOK_SENTINEL, 3u, 0u, 0u);
                    }
                    sts128(wbe_a + lane * 32, q0.x, q0.y, q0.z, q0.w);
                    sts128(wbe_a + lane * 32 + 16, q1.x, q1.y, q1.z, q1.w);
                }
                __syncwarp();
            }
            const u32 k = batch_pos++;
            const u32 seg = batch_seg + k;
            if (seg >= nseg) { exhausted = true; continue; }
            const u32 rec_a = wbe_a + k * 32;          // record k = the segment in front of this one
            const u32 cnt = lds32o<32 + 20>(rec_a);
            if (cnt == 0) {   // empty segment: only its (empty) edge record is carried over
                if (lane < 8) reinterpret_cast<u32 *>(&e_next[seg])[lane] = (lane < 5) ? TOK_SENTINEL : 0u;
                continue;
            }
            const u32 cm1 = lds32o<20>(rec_a), cp1 = lds32o<64 + 20>(rec_a);
            const u32 st_a = ws_a + stage * (MS_SW * 4);
            u32 mv = lds32(rec_a + meta_src);
            if (lane == 5) mv = seg;
            if (lane == 6) mv = cnt;
            if (lane < 16) sts32(meta_a + lane * 4, mv);
            if (lane < 2) sts32(st_a + (MS_PAD - 1 - lane) * 4, mv);   // s[-1] = P0, s[-2] = P1
            if (!(cm1 >= 2 && cp1 >= 3)) {   // short / empty neighbours: walk the edge records
                __syncwarp();
                if (lane == 0) {
                    u32 N[3], P[2];
                    seg_neighbours(e_cur, seg, nseg, N, P);
                    sts32o<0>(meta_a, P[0]); sts32o<4>(meta_a, P[1]); sts32o<8>(meta_a, N[0]); sts32o<12>(meta_a, N[1]); sts32o<16>(meta_a, N[2]);
                    sts32o<(MS_PAD - 1) * 4>(st_a, P[0]); sts32o<(MS_PAD - 2) * 4>(st_a, P[1]);
                }
            }
            __syncwarp();
            if (lane == 0) {
                const u32 bytes = ((cnt + 3u) & ~3u) * 4u;
                fence_proxy_async_smem();   // the stage was last written with ordinary stores (in-place compaction)
                mbar_arrive_expect_tx_a(wbar_a + stage * 8, bytes);
                bulk_g2s_a(st_a + MS_PAD * 4, w + (u64)seg * SEG_TOKENS, bytes, wbar_a + stage * 8);
            }
            __syncwarp();
            return;
        }
    };

    for (u32 s = 0; s + 1 < MS_STAGES; ++s) issue(s);
    u32 drops = 0;
    for (u32 j = 0;; ++j) {
        const u32 stage = j % MS_STAGES;
        issue((j + MS_STAGES - 1) % MS_STAGES);   // the stage consumed in the previous round
        const u32 meta_a = wmeta_a + stage * (MS_META * 4);
        const u32 seg = lds32o<20>(meta_a);
        if (seg == MS_INVALID) break;
        const u32 count = lds32o<24>(meta_a);
        const u32 s_a = ws_a + stage * (MS_SW * 4) + MS_PAD * 4;   // address of token 0 of the segment
        mbar_wait_a(wbar_a + stage * 8, (j / MS_STAGES) & 1u);
        if (lane < 3) sts32(s_a + (count + lane) * 4, lds32(meta_a + 8 + lane * 4));   // the three tokens that follow
        __syncwarp();

        // ---- mark: row r = tokens [128r, 128r+128), four consecutive tokens per lane ----
        u32 t[4][4], mn[4] = {0, 0, 0, 0}, keep[4] = {0, 0, 0, 0};
        u32 dirty = 0;
        const u32 la = s_a + lane * 16;
        u32 up = starts(M, lds32o<-4>(s_a), lds32(s_a)) ? 8u : 0u;   // the pair (s[-1], s[0]), as lane 31 of row -1
        mark_row<0>(la, lane, count, M, z, t[0], mn[0], keep[0], dirty, up);
        if (count > 128u) mark_row<1>(la, lane, count, M, z, t[1], mn[1], keep[1], dirty, up);
        if (count > 256u) mark_row<2>(la, lane, count, M, z, t[2], mn[2], keep[2], dirty, up);
        if (count > 384u) mark_row<3>(la, lane, count, M, z, t[3], mn[3], keep[3], dirty, up);
        dirty = __reduce_or_sync(FULL, dirty);   // rows in which some token is replaced or dropped
        if (!dirty) {
            // untouched segment: nothing to write, the edge record carries over
            if (lane < 8) reinterpret_cast<u32 *>(&e_next[seg])[lane] = lds32(meta_a + 32 + lane * 4);
            __syncwarp();
            continue;
        }

        // ---- statistics delta of this segment's merge starts (reads the stage before it is rewritten) ----
        if (delta)
            segment_delta(s_a, wlist_a, lane, mn[0] | (mn[1] << 4) | (mn[2] << 8) | (mn[3] << 12), M, z, A.V, s_dkey, s_dcnt, delta);

        // ---- kept tokens per lane and row, packed one byte per row: one warp scan for all four rows ----
        const u32 own = __popc(keep[0]) | (__popc(keep[1]) << 8) | (__popc(keep[2]) << 16) | (__popc(keep[3]) << 24);
        u32 incl = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const u32 v = __shfl_up_sync(FULL, incl, o);
            if (lane >= (u32)o) incl += v;          // a row keeps at most 128 tokens: no carry between bytes
        }
        const u32 tot = __shfl_sync(FULL, incl, 31);
        const u32 excl = incl - own;
        const u32 k0 = tot & 0xffu, k1 = (tot >> 8) & 0xffu, k2 = (tot >> 16) & 0xffu, k3 = tot >> 24;
        const u32 off1 = k0, off2 = k0 + k1, off3 = off2 + k2;
        const u32 new_count = off3 + k3;
        const int first_dirty = __ffs(dirty) - 1;   // rows in front of it stay where they are
        __syncwarp();                               // all lanes hold their tokens; delta reads are done

        // ---- compact in place inside the stage, from the first dirty row on ----
        if (first_dirty <= 0) scatter_row(s_a, lane, 0u, k0, excl & 0xffu, keep[0], t[0]);
        if (first_dirty <= 1 && count > 128u) scatter_row(s_a, lane, off1, k1, (excl >> 8) & 0xffu, keep[1], t[1]);
        if (first_dirty <= 2 && count > 256u) scatter_row(s_a, lane, off2, k2, (excl >> 16) & 0xffu, keep[2], t[2]);
        if (count > 384u) scatter_row(s_a, lane, off3, k3, excl >> 24, keep[3], t[3]);
        __syncwarp();
        // ---- copy-out: 16-byte vectors from the first dirty row to the new end (the up to three
        //      words past new_count land in the dead part of the segment) ----
        {
            uint4 *__restrict__ gp = reinterpret_cast<uint4 *>(w + (u64)seg * SEG_TOKENS) + lane;
            const u32 vend = (new_count + 3u) >> 2;
            if (first_dirty <= 0 && lane < vend) gp[0] = lds128o<0>(la);
            if (first_dirty <= 1 && lane + 32u < vend) gp[32] = lds128o<512>(la);
            if (first_dirty <= 2 && lane + 64u < vend) gp[64] = lds128o<1024>(la);
            if (lane + 96u < vend) gp[96] = lds128o<1536>(la);
        }
        // ---- the segment's new edge record ----
        {
            // lane:  0 1 2 -> f[0..2]   3 4 -> l[0], l[1] = tokens new_count-2, new_count-1   5 -> count   6 7 -> 0
            const u32 idx = lane < 3 ? lane : new_count + lane - 5u;
            const bool have = lane < 3 ? (lane < new_count) : (new_count + lane >= 5u);
            u32 word = TOK_SENTINEL;
            if (have && lane < 5) word = lds32(s_a + (idx & (SEG_TOKENS - 1)) * 4);
            if (lane == 5) word = new_count;
            if (lane > 5) word = 0;
            if (lane < 8) reinterpret_cast<u32 *>(&e_next[seg])[lane] = word;   // Edge = f[3], l[2], count, pad[2]
        }
        drops += count - new_count;
        __syncwarp();   // the stage may be refilled from here on
    }

    if (lane == 0 && drops) atomicAdd(s_drops, (ull)drops);
    __syncthreads();
    if (delta)
        for (u32 i = tid; i < MS_DCACHE; i += MS_THREADS)
            if (s_dkey[i] != 0xffffffffu && s_dcnt[i]) atomicAdd(&delta[s_dkey[i]], (ull)s_dcnt[i]);
    // ---- exit: the last CTA out publishes the new stream length and flips the edge arrays ----
    if (tid == 0) {
        const ull cta_drops = *s_drops;
        if (cta_drops) atomicAdd(&ctl->drops, cta_drops);
        __threadfence();
        const u32 e = atomicAdd(&ctl->merge_exit, 1u);
        if (e == gridDim.x - 1) {
            __threadfence();
            const ull dropped = *(volatile ull *)&ctl->drops;
            ctl->sum_in += n; ctl->sum_out += n - dropped;
            ctl->n = n - dropped;
            ctl->drops = 0;
            ctl->edge_cur ^= 1u;
            ctl->iter += NK;
            ctl->epoch += 1;
            ctl->merge_ticket = 0; ctl->merge_exit = 0;
        }
    }
}

// LIST = false: every segment of the stream, MS_BATCH consecutive ones per ticket.  LIST = true: only the candidate segments
// k_seg_filter put on the list at ctl->cand_ptr, one per ticket (the filter carried the other segments' edge records over).
// The segment filter and the sharded loop only ever run one member, so LIST takes the NK = 1 pass alone.
template <bool LIST>
__global__ void __launch_bounds__(MS_THREADS, MS_MINBLOCKS) k_merge_seg(SegArgs A) {
    const Ctl *ctl = A.ctl;
    if (!A.force && (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter)) return;
    if (ctl->a == ctl->b) return;  // pairs (a,a) take the pack + k_merge<true> path
    static_assert(BATCH_MAX == 4, "k_merge_seg: one pass per member count 1..BATCH_MAX");
    if constexpr (LIST) {
        merge_seg_pass<true, 1>(A);
    } else {
        switch (A.batched ? ctl->nk : 1u) {   // block-uniform
        case 2: merge_seg_pass<false, 2>(A); break;
        case 3: merge_seg_pass<false, 3>(A); break;
        case 4: merge_seg_pass<false, 4>(A); break;
        default: merge_seg_pass<false, 1>(A); break;
        }
    }
}
