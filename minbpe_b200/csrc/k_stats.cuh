// k_stats.cuh — pair statistics: full histograms (get_stats, base.py:13-22), the device-wide
// arg-max with the reference's first-occurrence tie-break (basic.py:35 / regex.py:56), and the
// incremental table update that follows a merge.
#pragma once
#include "common.cuh"
#include "k_seg.cuh"

// =============================================================================================
// Full histograms.  Both walk the segmented stream: one warp per segment (grid-stride), four
// tokens per thread per step (16-byte loads; segment bases are 2 KB aligned), equal keys inside
// a warp are folded by __match_any_sync before the global reduction.  Stream position of token i
// of segment t is t*SEG_TOKENS + i (monotone in stream order, used for first-occurrence order).
// The pair (last token of t, first token of the next non-empty segment) belongs to segment t.
// =============================================================================================
struct SegTokens {
    u32 t[5];       // four tokens starting at i0 and the token after them
    u32 nvalid;     // how many of t[0..3] are real tokens of the segment
};

__device__ __forceinline__ SegTokens seg_load4(const u32 *__restrict__ seg, u32 count, u32 i0, const Edge *e, u32 t,
                                               u32 nseg) {
    SegTokens r;
    if (i0 + 4 <= count) {
        const uint4 q = *reinterpret_cast<const uint4 *>(seg + i0);
        r.t[0] = q.x; r.t[1] = q.y; r.t[2] = q.z; r.t[3] = q.w;
        r.nvalid = 4;
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) r.t[k] = (i0 + k < count) ? seg[i0 + k] : TOK_SENTINEL;
        r.nvalid = count - i0;
    }
    r.t[4] = (i0 + 4 < count) ? seg[i0 + 4] : TOK_SENTINEL;
    if (i0 + 4 >= count) {  // this thread owns the segment's last token: its right neighbour is in a later segment
        const u32 nf = seg_next_first(e, t, nseg);
        const u32 slot = count - i0;   // slot right after the last real token (1..4)
#pragma unroll
        for (u32 k = 1; k <= 4; ++k) if (slot == k) r.t[k] = nf;
    }
    return r;
}

// BYTE stream (all ids < 256) -> dense 256x256 vector, dense[p0*256+p1] += count.  Used once per
// train() for iteration 0; afterwards the table is maintained incrementally by the merge pass.
// Per-block open-addressing histogram in shared memory (text uses a few thousand of the 65,536
// byte pairs), equal keys of a warp folded first with __match_any_sync, one flush per block.
#define HD_SLOTS 4096
__global__ void __launch_bounds__(256) k_hist_dense(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1,
                                                    const Ctl *__restrict__ ctl, const Edge *e0, const Edge *e1,
                                                    ull *__restrict__ dense, u32 *__restrict__ err) {
    __shared__ u32 s_key[HD_SLOTS];   // 16-bit pair or 0xffffffff
    __shared__ u32 s_cnt[HD_SLOTS];
    for (u32 i = threadIdx.x; i < HD_SLOTS; i += blockDim.x) { s_key[i] = 0xffffffffu; s_cnt[i] = 0; }
    __syncthreads();
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);
    const u32 nseg = ctl->nseg;
    const u32 wpb = blockDim.x >> 5;
    for (u32 t = blockIdx.x * wpb + (threadIdx.x >> 5); t < nseg; t += gridDim.x * wpb) {
        const u32 count = e[t].count;
        const u32 *__restrict__ seg = w + (u64)t * SEG_TOKENS;
        for (u32 i0 = lane_id() * 4; i0 < count; i0 += 128) {
            const SegTokens r = seg_load4(seg, count, i0, e, t, nseg);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const u32 left = r.t[k] & TOK_MASK, right = r.t[k + 1];
                const bool valid = ((u32)k < r.nvalid) && !(right & TOK_FLAG);
                if (valid && (left > 255u || right > 255u)) *err = 1;
                const u32 key = valid ? ((left & 255u) << 8 | (right & 255u)) : 0xffffffffu;
                const u32 peers = __match_any_sync(__activemask(), key);
                if (valid && (__ffs(peers) - 1) == (int)lane_id()) {   // group leader adds the whole group
                    const u32 add = __popc(peers);
                    u32 slot = (key * 2654435761u) >> (32 - 12);
                    bool placed = false;
#pragma unroll 1
                    for (int probe = 0; probe < 8 && !placed; ++probe) {
                        u32 kk = reinterpret_cast<volatile u32 *>(s_key)[slot];
                        if (kk == 0xffffffffu) {
                            const u32 old = atomicCAS(&s_key[slot], 0xffffffffu, key);
                            kk = (old == 0xffffffffu) ? key : old;
                        }
                        if (kk == key) { atomicAdd(&s_cnt[slot], add); placed = true; }
                        slot = (slot + 1) & (HD_SLOTS - 1);
                    }
                    if (!placed) atomicAdd(&dense[key], (ull)add);
                }
            }
        }
    }
    __syncthreads();
    for (u32 i = threadIdx.x; i < HD_SLOTS; i += blockDim.x)
        if (s_key[i] != 0xffffffffu && s_cnt[i]) atomicAdd(&dense[s_key[i]], (ull)s_cnt[i]);
}

// The same histogram with a DENSE per-CTA table: all 65,536 byte pairs as 16-bit counters packed two per word
// (128 KB of dynamic shared memory, one CTA of 1024 threads per SM), one shared-memory atomicAdd per pair, no hashing and
// no warp-level matching.  A counter cannot overflow: the CTA flushes its table into the global vector (and clears it)
// after every round of at most HP_ROUND_TOKENS (< 65,536) tokens.  Rounds have the same trip count for every warp of the
// CTA, so the flush barriers are uniform.
#define HP_THREADS 1024
#define HP_SEGS_PER_WARP 3                                  // segments of 512 tokens per warp per round
#define HP_ROUND_TOKENS ((HP_THREADS / 32) * HP_SEGS_PER_WARP * SEG_TOKENS)
#define HP_SMEM_BYTES (65536 * 2)
static_assert(HP_ROUND_TOKENS < 65536, "a 16-bit counter must survive one round");
__global__ void __launch_bounds__(HP_THREADS) k_hist_dense_packed(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1,
                                                                  const Ctl *__restrict__ ctl, const Edge *e0, const Edge *e1,
                                                                  ull *__restrict__ dense, u32 *__restrict__ err) {
    extern __shared__ u32 s_hist[];   // [32768]: bin i = bits 16*(i&1).. of word i>>1
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wpb = HP_THREADS / 32;
    for (u32 i = tid; i < 32768u; i += HP_THREADS) s_hist[i] = 0;
    __syncthreads();
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);
    const u32 nseg = ctl->nseg;
    // segment t belongs to CTA (t / wpb) % gridDim.x, warp t % wpb; this CTA's k-th segment group = blockIdx.x + k * gridDim.x
    const u32 groups = (nseg + wpb - 1) / wpb;                                  // groups of wpb consecutive segments
    const u32 my_groups = groups > blockIdx.x ? (groups - blockIdx.x + gridDim.x - 1) / gridDim.x : 0u;
    const u32 rounds = (my_groups + HP_SEGS_PER_WARP - 1) / HP_SEGS_PER_WARP;   // block-uniform
    for (u32 r = 0; r < rounds; ++r) {
        for (u32 j = 0; j < HP_SEGS_PER_WARP; ++j) {
            const u32 k = r * HP_SEGS_PER_WARP + j;
            if (k >= my_groups) break;
            const u32 t = (blockIdx.x + k * gridDim.x) * wpb + warp;
            if (t >= nseg) continue;
            const u32 count = e[t].count;
            const u32 *__restrict__ seg = w + (u64)t * SEG_TOKENS;
            for (u32 i0 = lane * 4; i0 < count; i0 += 128) {
                const SegTokens q = seg_load4(seg, count, i0, e, t, nseg);
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const u32 left = q.t[c] & TOK_MASK, right = q.t[c + 1];
                    if ((u32)c < q.nvalid && !(right & TOK_FLAG)) {
                        if (left > 255u || right > 255u) *err = 1;
                        const u32 bin = (left & 255u) << 8 | (right & 255u);
                        atomicAdd(&s_hist[bin >> 1], 1u << (16u * (bin & 1u)));
                    }
                }
            }
        }
        __syncthreads();
        for (u32 i = tid; i < 32768u; i += HP_THREADS) {
            const u32 v = s_hist[i];
            if (v) {
                if (v & 0xffffu) atomicAdd(&dense[2 * i], (ull)(v & 0xffffu));
                if (v >> 16) atomicAdd(&dense[2 * i + 1], (ull)(v >> 16));
                s_hist[i] = 0;
            }
        }
        __syncthreads();
    }
}

// first-use cross-check of the packed histogram against k_hist_dense (b200bpe.cu hist_dense): flag |= 1 on any difference
__global__ void k_dense_compare(const ull *__restrict__ a, const ull *__restrict__ b, u32 *__restrict__ flag) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 65536u && a[i] != b[i]) *flag = 1;
}

// dense 256x256 vector -> table entries (one thread per bin)
__global__ void k_dense_to_table(const ull *__restrict__ dense, Table t, Ctl *ctl) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 65536u) return;
    const ull c = dense[i];
    if (!c) return;
    const u64 slot = table_upsert(t, pack_pair(i >> 8, i & 255u), &ctl->table_used);
    t.counts[slot] = c;
}

// Arbitrary stream -> hash table with first-occurrence positions (count += 1, first = min).  This
// is get_stats() (base.py:13-22) for the C ABI and the "rescan" verification mode: the scan the
// north star describes — 16-byte loads, equal keys of a warp folded with __match_any_sync, a
// per-block open-addressing histogram {pair, count, first position} in shared memory, one flush of
// every block's table into the global one (device-wide combine); keys that do not find a slot
// within a few probes go to the global table directly.
#define HH_SLOTS 2048
__device__ __forceinline__ void hist_global_add(Table &tab, Ctl *ctl, u64 key, ull add, u64 pos) {
    // a full histogram inserts without reservations: refuse (and flag) rather than fill the table up
    if (*(volatile ull *)&ctl->table_used >= (3 * (tab.mask + 1)) / 4) { ctl->overflow = 1; return; }
    const u64 slot = table_upsert(tab, key, &ctl->table_used);
    atomicAdd((ull *)&tab.counts[slot], add);
    if (tab.first) atomicMin((ull *)&tab.first[slot], (ull)pos);
}

__global__ void __launch_bounds__(256) k_hist_hash(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1,
                                                   Ctl *ctl, const Edge *e0, const Edge *e1, Table tab, int gated) {
    if (gated && (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter)) return;
    __shared__ ull s_key[HH_SLOTS];
    __shared__ ull s_first[HH_SLOTS];
    __shared__ u32 s_cnt[HH_SLOTS];
    for (u32 i = threadIdx.x; i < HH_SLOTS; i += blockDim.x) { s_key[i] = KEY_EMPTY; s_first[i] = POS_NONE; s_cnt[i] = 0; }
    __syncthreads();
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);
    const u32 nseg = ctl->nseg;
    const u32 wpb = blockDim.x >> 5;
    for (u32 t = blockIdx.x * wpb + (threadIdx.x >> 5); t < nseg; t += gridDim.x * wpb) {
        const u32 count = e[t].count;
        const u32 *__restrict__ seg = w + (u64)t * SEG_TOKENS;
        // warp-uniform trip count: every lane reaches every __match_any_sync below, so the full mask names exactly the
        // lanes that execute it (__activemask() would not guarantee that: lanes past the segment's end leave early)
        for (u32 base = 0; base < count; base += 128) {
            const u32 i0 = base + lane_id() * 4;
            SegTokens r;
            r.nvalid = 0;
            if (i0 < count) r = seg_load4(seg, count, i0, e, t, nseg);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const bool valid = ((u32)k < r.nvalid) && !(r.t[k + 1] & TOK_FLAG);
                const u64 key = valid ? pack_pair(r.t[k] & TOK_MASK, r.t[k + 1]) : KEY_EMPTY;
                __syncwarp();
                const u32 peers = __match_any_sync(0xffffffffu, key);
                // the lowest lane of a group also holds the group's smallest position
                if (valid && (__ffs(peers) - 1) == (int)lane_id()) {
                    const u32 add = __popc(peers);
                    const u64 pos = (u64)t * SEG_TOKENS + i0 + k;
                    u32 slot = (u32)(hash64(key) & (HH_SLOTS - 1));
                    bool placed = false;
#pragma unroll 1
                    for (int probe = 0; probe < 6 && !placed; ++probe) {
                        ull kk = reinterpret_cast<volatile ull *>(s_key)[slot];
                        if (kk == KEY_EMPTY) {
                            const ull old = atomicCAS(&s_key[slot], (ull)KEY_EMPTY, (ull)key);
                            kk = (old == KEY_EMPTY) ? key : old;
                        }
                        if (kk == key) {
                            atomicAdd(&s_cnt[slot], add);
                            atomicMin(&s_first[slot], (ull)pos);
                            placed = true;
                        }
                        slot = (slot + 1) & (HH_SLOTS - 1);
                    }
                    if (!placed) hist_global_add(tab, ctl, key, add, pos);
                }
            }
        }
    }
    __syncthreads();
    for (u32 i = threadIdx.x; i < HH_SLOTS; i += blockDim.x)
        if (s_key[i] != KEY_EMPTY && s_cnt[i]) hist_global_add(tab, ctl, s_key[i], s_cnt[i], s_first[i]);
}

// =============================================================================================
// Arg-max over the table: max count, how many pairs share it, one slot holding it.
// Two-level: per-thread -> warp shuffle -> block -> last block (ticket) reduces the partials.
// When the max is unique the winning pair is final; otherwise k_find_first resolves the tie by
// stream position, which is what the reference's dict insertion order amounts to.
// =============================================================================================
struct Best { u64 count; u64 slot; u32 tied; };

__device__ __forceinline__ Best best_combine(Best x, Best y) {
    if (y.count > x.count) return y;
    if (y.count == x.count) { x.tied += y.tied; if (y.slot < x.slot) x.slot = y.slot; }
    return x;
}

__device__ __forceinline__ Best best_warp_reduce(Best v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Best y;
        y.count = __shfl_xor_sync(0xffffffffu, v.count, o);
        y.slot = __shfl_xor_sync(0xffffffffu, v.slot, o);
        y.tied = __shfl_xor_sync(0xffffffffu, v.tied, o);
        v = best_combine(v, y);
    }
    return v;
}

// log layout: pairs int32[2*i], counts int64[i]
__device__ __forceinline__ void record_selection(Ctl *ctl, int a, int b, u64 count, int *log_pairs, long long *log_counts) {
    ctl->a = a; ctl->b = b; ctl->z = (int)(ctl->first_idx + ctl->iter);
    if (log_pairs) { log_pairs[2 * ctl->iter] = a; log_pairs[2 * ctl->iter + 1] = b; log_counts[ctl->iter] = (long long)count; }
}

__global__ void __launch_bounds__(256) k_argmax(Table t, Ctl *ctl, Best *partials, int *log_pairs, long long *log_counts) {
    if (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter) return;
    const u64 cap = t.mask + 1;
    Best v; v.count = 0; v.slot = POS_NONE; v.tied = 0;
    // two 64-bit counts per 16-byte load
    const ulonglong2 *c2 = reinterpret_cast<const ulonglong2 *>(t.counts);
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < cap / 2; i += (u64)gridDim.x * blockDim.x) {
        ulonglong2 c = c2[i];
        if (c.x) { Best y; y.count = c.x; y.slot = 2 * i; y.tied = 1; v = best_combine(v, y); }
        if (c.y) { Best y; y.count = c.y; y.slot = 2 * i + 1; y.tied = 1; v = best_combine(v, y); }
    }
    v = best_warp_reduce(v);
    __shared__ Best s[8];
    __shared__ bool last;
    if (lane_id() == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < (int)(blockDim.x >> 5); ++k) v = best_combine(v, s[k]);
        partials[blockIdx.x] = v;
        __threadfence();
        last = (atomicAdd(&ctl->argmax_exit, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // last block: reduce the per-block partials
    Best r; r.count = 0; r.slot = POS_NONE; r.tied = 0;
    for (u32 k = threadIdx.x; k < gridDim.x; k += blockDim.x) {
        Best y;
        y.count = ld_volatile_u64(&partials[k].count);
        y.slot = ld_volatile_u64(&partials[k].slot);
        y.tied = ld_volatile_u32(&partials[k].tied);
        r = best_combine(r, y);
    }
    r = best_warp_reduce(r);
    if (lane_id() == 0) s[threadIdx.x >> 5] = r;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < (int)(blockDim.x >> 5); ++k) r = best_combine(r, s[k]);
        ctl->argmax_exit = 0;
        ctl->best_count = r.count; ctl->best_slot = r.slot; ctl->n_tied = r.tied;
        ctl->found_pos = POS_NONE;
        ctl->tie_local = 0;
        ctl->nk = 1;                                        // k_select_batch may add members
        if (r.count == 0) ctl->done = 1;                   // max({}) -> ValueError in the reference
        else if (r.tied == 1) {
            const u64 key = t.keys[r.slot];
            record_selection(ctl, (int)(key >> 32), (int)(key & 0xffffffffu), r.count, log_pairs, log_counts);
        }
    }
}

// =============================================================================================
// Batched merges (DESIGN.md "Batched merges").  With the pairs of the table sorted by count, p1 = the arg-max, the next
// k merges are exactly p1 .. pk, in that order, when c1 > c2 > ... > ck > c(k+1), every pj has two different ids and
// the 2k ids are all distinct.  A merge only lowers counts of pairs that share an id with it, and every pair it creates
// has at most the count of such a pair, which is not a member: at most c(k+1).  So each member stays the unique maximum
// until its turn, with the count it has now, and no tie-break is involved.  Being token-disjoint, the members never
// overlap in the stream: one pass of k_merge_seg applies all of them.
// k_select_batch runs after k_argmax when the arg-max is unique and a != b: the top BATCH_MAX+1 entries of the table
// (per-thread lists, warp merge, one list per block, the last block merges the blocks' lists), then the rule above.
// =============================================================================================
#define TOPN (BATCH_MAX + 1)
struct TopList { u64 c[TOPN]; u64 s[TOPN]; };   // count, slot; descending count, then ascending slot; count 0 = empty

__device__ __forceinline__ bool top_before(u64 c, u64 s, u64 c2, u64 s2) { return c > c2 || (c == c2 && s < s2); }

__device__ __forceinline__ void top_insert(TopList &l, u64 c, u64 s) {
    if (!c || !top_before(c, s, l.c[TOPN - 1], l.s[TOPN - 1])) return;
#pragma unroll
    for (int i = TOPN - 1; i >= 0; --i) {
        if (i > 0 && top_before(c, s, l.c[i - 1], l.s[i - 1])) { l.c[i] = l.c[i - 1]; l.s[i] = l.s[i - 1]; }
        else { l.c[i] = c; l.s[i] = s; break; }
    }
}

__device__ __forceinline__ void top_clear(TopList &l) {
#pragma unroll
    for (int i = 0; i < TOPN; ++i) { l.c[i] = 0; l.s[i] = POS_NONE; }
}

// the warp's TOPN best entries, on every lane: TOPN rounds of "best head of all lanes, its lane pops it"
__device__ __forceinline__ TopList top_warp_merge(TopList l) {
    TopList r;
#pragma unroll
    for (int k = 0; k < TOPN; ++k) {
        u64 c = l.c[0], s = l.s[0];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const u64 c2 = __shfl_xor_sync(0xffffffffu, c, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
            if (top_before(c2, s2, c, s)) { c = c2; s = s2; }
        }
        r.c[k] = c; r.s[k] = s;
        if (c && l.c[0] == c && l.s[0] == s) {   // slots are unique: exactly one lane holds the winner
#pragma unroll
            for (int i = 0; i + 1 < TOPN; ++i) { l.c[i] = l.c[i + 1]; l.s[i] = l.s[i + 1]; }
            l.c[TOPN - 1] = 0; l.s[TOPN - 1] = POS_NONE;
        }
    }
    return r;
}

// block-wide: every thread's list -> thread 0's list (s_l: [8] lists of shared memory)
__device__ __forceinline__ TopList top_block_merge(TopList l, TopList *s_l) {
    l = top_warp_merge(l);
    if (lane_id() == 0) s_l[threadIdx.x >> 5] = l;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
            for (int i = 0; i < TOPN; ++i) top_insert(l, s_l[w].c[i], s_l[w].s[i]);
    return l;
}

__global__ void __launch_bounds__(256) k_select_batch(Table t, Ctl *ctl, TopList *partials, int *log_pairs, long long *log_counts) {
    if (ctl->done || ctl->overflow || ctl->iter + 1 >= ctl->max_iter || ctl->n_tied != 1 || ctl->a == ctl->b) return;
    const u64 cap = t.mask + 1;
    TopList l;
    top_clear(l);
    const ulonglong2 *c2 = reinterpret_cast<const ulonglong2 *>(t.counts);
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < cap / 2; i += (u64)gridDim.x * blockDim.x) {
        const ulonglong2 c = c2[i];
        top_insert(l, c.x, 2 * i);
        top_insert(l, c.y, 2 * i + 1);
    }
    __shared__ TopList s_l[8];
    __shared__ bool last;
    l = top_block_merge(l, s_l);
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = l;
        __threadfence();
        last = (atomicAdd(&ctl->argmax_exit, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    top_clear(l);
    for (u32 k = threadIdx.x; k < gridDim.x * TOPN; k += blockDim.x) {
        const TopList *p = &partials[k / TOPN];
        top_insert(l, ld_volatile_u64(&p->c[k % TOPN]), ld_volatile_u64(&p->s[k % TOPN]));
    }
    __syncthreads();   // s_l is reused
    l = top_block_merge(l, s_l);
    if (threadIdx.x != 0) return;
    ctl->argmax_exit = 0;
    s_l[0] = l;   // indexed with a run-time member number below: from shared memory, so that `l` stays in registers
    const TopList &L = s_l[0];
    if (L.s[0] != ctl->best_slot) return;   // cannot happen: the table did not change since k_argmax
    const u32 limit = min((u32)BATCH_MAX, ctl->max_iter - ctl->iter);
    u32 ids[2 * BATCH_MAX];
    ids[0] = (u32)ctl->a; ids[1] = (u32)ctl->b;
    u32 k = 1;   // c1 > c2 holds: the arg-max is unique
    for (; k < limit; ++k) {
        if (!(L.c[k] > L.c[k + 1])) break;   // c(k+1) must stay below the new member's count
        const u64 key = t.keys[L.s[k]];
        const u32 x = (u32)(key >> 32), y = (u32)(key & 0xffffffffu);
        bool ok = x != y;
        for (u32 i = 0; i < 2 * k; ++i) ok = ok && ids[i] != x && ids[i] != y;
        if (!ok) break;
        ids[2 * k] = x; ids[2 * k + 1] = y;
        ctl->bat_a[k] = (int)x; ctl->bat_b[k] = (int)y;
        if (log_pairs) {
            const u32 it = ctl->iter + k;
            log_pairs[2 * it] = (int)x; log_pairs[2 * it + 1] = (int)y; log_counts[it] = (long long)L.c[k];
        }
    }
    ctl->nk = k;
}

// =============================================================================================
// Tie-break: among the pairs whose count equals the max, the reference picks the one inserted
// first into the dict = the one whose first occurrence in the current stream is earliest.
// Scan the stream from the front in tiles, look each pair up, stop at the first tile that holds a
// hit (later tiles exit as soon as they see found_pos in front of them).  Expected cost is
// n / (tied * count) tokens — a tiny prefix unless counts are ~1.
// =============================================================================================
#define FF_GROUP 8
__global__ void __launch_bounds__(256) k_find_first(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1,
                                                    const Edge *e0, const Edge *e1, Table t, Ctl *ctl,
                                                    int *log_pairs, long long *log_counts, int sharded) {
    if (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter || ctl->n_tied <= 1) return;
    const u32 *w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);
    // sharded loop: none of the tied pairs has ever occurred in this shard -> nothing to scan, answer "not here"
    const u32 nseg = (sharded && !ctl->tie_local) ? 0u : ctl->nseg;
    const u64 best = ctl->best_count;
    __shared__ bool last;
    __shared__ u64 s_found;
    for (u32 g = blockIdx.x;; g += gridDim.x) {   // groups of FF_GROUP segments, in stream order
        const u32 sg0 = g * FF_GROUP;
        const u64 base = (u64)sg0 * SEG_TOKENS;
        if (threadIdx.x == 0) s_found = ld_volatile_u64(&ctl->found_pos);
        __syncthreads();
        if (sg0 >= nseg || s_found < base) break;  // block-uniform: a hit in front of this group ends the scan
        u64 hit = POS_NONE;
        for (u32 i = threadIdx.x; i < FF_GROUP * SEG_TOKENS; i += blockDim.x) {   // ascending stream position
            const u32 sg = sg0 + (i >> SEG_SHIFT), off = i & (SEG_TOKENS - 1);
            if (sg >= nseg) break;
            const u32 count = e[sg].count;
            if (off >= count) continue;
            const u32 right = (off + 1 < count) ? w[base + i + 1] : seg_next_first(e, sg, nseg);
            if (!(right & TOK_FLAG)) {
                const u64 slot = table_find(t, pack_pair(w[base + i] & TOK_MASK, right));
                if (slot != POS_NONE && t.counts[slot] == best) { hit = base + i; break; }  // this thread's first hit
            }
        }
        if (hit != POS_NONE) atomicMin((ull *)&ctl->found_pos, (ull)hit);
        __syncthreads();
    }
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); last = (atomicAdd(&ctl->ff_exit, 1u) == gridDim.x - 1); }
    __syncthreads();
    if (last && threadIdx.x == 0) {
        __threadfence();
        ctl->ff_exit = 0;
        const u64 p = ld_volatile_u64(&ctl->found_pos);
        if (p == POS_NONE) {
            if (sharded) ctl->a = -1;   // none of the tied pairs occurs in this rank's shard
            else ctl->done = 1;         // cannot happen when the table matches the stream
        } else {
            const u32 sg = (u32)(p >> SEG_SHIFT), i = (u32)(p & (SEG_TOKENS - 1));
            const u32 right = (i + 1 < e[sg].count) ? w[p + 1] : seg_next_first(e, sg, nseg);
            record_selection(ctl, (int)(w[p] & TOK_MASK), (int)right, best, log_pairs, log_counts);
        }
    }
}

// =============================================================================================
// Sharded loop: "may this pair occur in MY shard?"  A rank keeps a bitmap over pair hashes with a bit
// for every pair that has ever existed in its shard (the byte pairs of iteration 0, then the pairs
// each local merge creates: (x,z) for L[x] > 0, (z,y) for R[y] > 0, (z,z) for ZZ > 0 — the only
// ways a pair can appear).  Bits are never cleared, so the answer is conservative: a set bit costs
// at most the scan that was done unconditionally before; a clear bit proves absence.  On a tie whose
// pairs live only in other ranks' shards, this rank skips the scan of its whole shard.
// =============================================================================================
#define PRESENT_LOG2 24
__device__ __forceinline__ u32 present_hash(u64 key) { return (u32)(hash64(key) >> 24) & ((1u << PRESENT_LOG2) - 1u); }
__device__ __forceinline__ void present_set(u32 *bm, u64 key) { const u32 x = present_hash(key); atomicOr(&bm[x >> 5], 1u << (x & 31u)); }
__device__ __forceinline__ bool present_get(const u32 *bm, u64 key) { const u32 x = present_hash(key); return (bm[x >> 5] >> (x & 31u)) & 1u; }

__global__ void k_present_init(const ull *__restrict__ dense, u32 *__restrict__ bm) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 65536u && dense[i]) present_set(bm, pack_pair(i >> 8, i & 255u));
}

// after a merge, from the LOCAL delta vector (before it is summed across ranks)
__global__ void k_present_update(const ull *__restrict__ delta, u32 V, const Ctl *__restrict__ ctl, u32 *__restrict__ bm) {
    if (ctl->done || ctl->overflow || ctl->a < 0) return;
    const u32 z = (u32)ctl->z;
    const u32 x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x < V) {
        if (delta[x]) present_set(bm, pack_pair(x, z));
        if (delta[V + x]) present_set(bm, pack_pair(z, x));
    }
    if (x == 0 && delta[2ull * V]) present_set(bm, pack_pair(z, z));
}

// on a tie: does any pair at the max count possibly occur in this shard?
__global__ void __launch_bounds__(256) k_tie_present(Table t, Ctl *ctl, const u32 *__restrict__ bm) {
    if (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter || ctl->n_tied <= 1) return;
    const u64 best = ctl->best_count;
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s <= t.mask; s += (u64)gridDim.x * blockDim.x) {
        const u64 key = t.keys[s];
        if (key != KEY_EMPTY && t.counts[s] == best && present_get(bm, key)) ctl->tie_local = 1;
    }
}

// =============================================================================================
// Incremental update of the table after merging (a,b) -> z.  The merge kernel leaves, per token
// id x, L[x] = number of merges whose left neighbour is an unmerged x, R[x] = number of merges
// whose right neighbour is an unmerged x, and ZZ = number of merges directly followed by another
// merge.  Then (DESIGN.md "Incremental statistics"):
//     count(x,a) -= L[x]   count(x,z) = L[x]
//     count(b,x) -= R[x]   count(z,x) = R[x]
//     count(b,a) -= ZZ     count(z,z) = ZZ         count(a,b) = 0
// delta layout: [0,V) = L, [V,2V) = R, [2V] = ZZ, V = vocab capacity.  The vector is zeroed.
// =============================================================================================
__device__ __forceinline__ void table_sub(const Table &t, u64 key, u64 skip_key, ull d) {
    if (key == skip_key) return;  // (a,b) itself is zeroed wholesale
    const u64 slot = table_find(t, key);
    if (slot != POS_NONE) atomicAdd((ull *)&t.counts[slot], (ull)(0ull - d));
}

// Every non-zero delta entry creates exactly one new pair (it contains the new id z, so it cannot
// be in the table yet).  A slot is reserved first; when the table is at its load limit the entry
// is left untouched and ctl->overflow is raised: the host grows the table and re-runs this kernel
// (`retry`), which applies exactly the entries that are still non-zero.
__device__ __forceinline__ bool table_reserve(Ctl *ctl) {
    const ull r = atomicAdd(&ctl->table_used, 1ull);
    if (r < ctl->table_limit) return true;
    atomicAdd(&ctl->table_used, (ull)(0ull - 1ull));
    ctl->overflow = 1;
    return false;
}

// Member j > 0 of a batched pass (use_ctl only) is a launch of its own, after member j-1's: its left and right
// neighbours may be ids an earlier member created, whose pairs that member's launch inserts.
__global__ void __launch_bounds__(256) k_apply_delta(Table t, Ctl *ctl, ull *__restrict__ delta, u32 V,
                                                     int a_arg, int b_arg, int z_arg, int use_ctl, int retry, int member = 0) {
    if (use_ctl && (ctl->done || ctl->iter > ctl->max_iter)) return;
    if (use_ctl && ctl->overflow && !retry) return;   // an earlier iteration is waiting for the host
    if (member > 0 && (!use_ctl || (u32)member >= ctl->nk)) return;
    const u32 a = use_ctl ? (u32)(member ? ctl->bat_a[member] : ctl->a) : (u32)a_arg,
              b = use_ctl ? (u32)(member ? ctl->bat_b[member] : ctl->b) : (u32)b_arg,
              z = use_ctl ? (u32)ctl->z + (u32)member : (u32)z_arg;
    delta += (u64)member * (2ull * V + 1);
    const u64 kab = pack_pair(a, b);
    const u32 x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x < V) {
        const ull l = delta[x];
        if (l && table_reserve(ctl)) {
            delta[x] = 0;
            table_sub(t, pack_pair(x, a), kab, l);
            const u64 s = table_upsert(t, pack_pair(x, z), nullptr);
            atomicAdd((ull *)&t.counts[s], l);
        }
        const ull r = delta[V + x];
        if (r && table_reserve(ctl)) {
            delta[V + x] = 0;
            table_sub(t, pack_pair(b, x), kab, r);
            const u64 s = table_upsert(t, pack_pair(z, x), nullptr);
            atomicAdd((ull *)&t.counts[s], r);
        }
    }
    if (x == 0) {
        const ull zz = delta[2 * (u64)V];
        if (zz && table_reserve(ctl)) {
            delta[2 * (u64)V] = 0;
            table_sub(t, pack_pair(b, a), kab, zz);
            const u64 s = table_upsert(t, pack_pair(z, z), nullptr);
            atomicAdd((ull *)&t.counts[s], zz);
        }
        const u64 s = table_find(t, kab);
        if (s != POS_NONE) t.counts[s] = 0;
    }
}

// Copy live entries (count > 0) into a fresh table (growth / dropping dead pairs).
__global__ void k_rehash(Table src, Table dst, Ctl *ctl) {
    const u64 cap = src.mask + 1;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (u64)gridDim.x * blockDim.x) {
        const u64 k = src.keys[i];
        const u64 c = src.counts[i];
        if (k != KEY_EMPTY && c) {
            const u64 s = table_upsert(dst, k, &ctl->table_used);
            dst.counts[s] = c;
        }
    }
}

// =============================================================================================
// Sharded training (one process per GPU, DESIGN.md "Multi-GPU"): every rank holds the same global
// pair table, so the arg-max agrees everywhere; only a tie needs the ranks to talk, because the
// reference's first-occurrence rule is "lowest rank (= earliest text) that sees a tied pair".
// Each rank packs its local candidate into one int64, the host all-reduces it with MIN.
//   word = rank << 58 | p0 << 29 | p1        (INT64_MAX: nothing to offer)
// =============================================================================================
#define CAND_NONE 0x7fffffffffffffffll
__global__ void k_pack_candidate(const Ctl *ctl, long long *cand, int rank) {
    if (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter || ctl->a < 0) { cand[0] = CAND_NONE; return; }
    cand[0] = ((long long)rank << 58) | ((long long)ctl->a << 29) | (long long)ctl->b;
}

__global__ void k_commit_candidate(Ctl *ctl, const long long *cand, int *log_pairs, long long *log_counts) {
    if (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter) return;
    const long long w = cand[0];
    if (w == CAND_NONE) { ctl->done = 1; return; }   // no rank has a pair left
    record_selection(ctl, (int)((w >> 29) & 0x1fffffff), (int)(w & 0x1fffffff), ctl->best_count, log_pairs, log_counts);
}
