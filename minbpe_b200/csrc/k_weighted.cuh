// k_weighted.cuh — the training loop on a WEIGHTED stream (DESIGN.md "Training on distinct chunks").
//
// A weighted stream is a list of entries, each an occurrence of a chunk in text order, with a weight >= 1: the number
// of occurrences of the same bytes it stands for.  The stream keeps the ordinary layout (one token word per token, bit 31
// marks the first token of an entry); the weights live in a separate array, one u64 per entry, in stream order.
//
// Which entry holds a token: a merge never removes a chunk-start mark (the merged token keeps the mark of its first
// half) and compaction never moves a token to another segment, so the number of marks in a segment stays the same
// between two packs.  base[t] = marks in all segments before t (k_wt_marks + k_wt_scan, after every load and pack);
// the token at offset p of segment t then belongs to entry base[t] + (marks in [0, p]) - 1.
//
// The kernels below only add what weights change: the full histogram of iteration 0 and the statistics delta of a
// merge, both adding the entry's weight where the plain kernels add 1.  The delta is computed by a pass of its own in
// front of the plain merge (k_merge_seg / k_merge<true> launched without a delta vector), so the merge kernels are
// the ones of the unweighted loop.  Marks, tie-breaks (k_find_first), the batched-merge rule (k_select_batch) and the
// table update (k_apply_delta) are unchanged: counts are u64 sums either way.
#pragma once
#include "common.cuh"
#include "k_seg.cuh"
#include "k_stats.cuh"

// segments of the current stream, and the token count of segment t.  contig: the stream was just packed (ctl->contig)
// and its edge records are stale: every segment is full except the last.
__device__ __forceinline__ u32 wt_nseg(const Ctl *ctl, bool contig) {
    return contig ? (u32)((ctl->n + SEG_TOKENS - 1) / SEG_TOKENS) : ctl->nseg;
}
__device__ __forceinline__ u32 wt_count(const Ctl *ctl, const Edge *e, u32 t, bool contig) {
    if (!contig) return e[t].count;
    const u64 rest = ctl->n - (u64)t * SEG_TOKENS;
    return rest < SEG_TOKENS ? (u32)rest : (u32)SEG_TOKENS;
}

// chunk-start marks per segment -> cnt[t].  Runs when forced (after a load) or when the stream was just packed.
__global__ void __launch_bounds__(256) k_wt_marks(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1, const Ctl *ctl,
                                                  const Edge *e0, const Edge *e1, u32 *__restrict__ cnt, int force) {
    const bool contig = ctl->contig != 0;
    if (!force && !contig) return;
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);
    const u32 nseg = wt_nseg(ctl, contig);
    const u32 wpb = blockDim.x >> 5, lane = lane_id();
    for (u32 t = blockIdx.x * wpb + (threadIdx.x >> 5); t < nseg; t += gridDim.x * wpb) {
        const u32 count = wt_count(ctl, e, t, contig);
        const u32 *__restrict__ seg = w + (u64)t * SEG_TOKENS;
        u32 c = 0;
        for (u32 i = lane; i < count; i += 32) c += seg[i] >> 31;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) cnt[t] = c;
    }
}

// base[t] = exclusive prefix sum of cnt (one block of 1024 threads; the same slicing as k_scan_counts)
__global__ void __launch_bounds__(1024) k_wt_scan(const Ctl *ctl, const u32 *__restrict__ cnt, u64 *__restrict__ base, int force) {
    const bool contig = ctl->contig != 0;
    if (!force && !contig) return;
    const u32 nseg = wt_nseg(ctl, contig);
    const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 per = ((nseg + 31) / 32 + 31) & ~31u;
    const u32 lo = min(nseg, warp * per), hi = min(nseg, lo + per);
    u64 sum = 0;
    for (u32 t = lo + lane; t < hi; t += 32) sum += cnt[t];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __shared__ u64 s_w[32];
    if (lane == 0) s_w[warp] = sum;
    __syncthreads();
    u64 run = 0;
    for (u32 k = 0; k < warp; ++k) run += s_w[k];
    for (u32 t0 = lo; t0 < hi; t0 += 32) {
        const u32 t = t0 + lane;
        const u32 c = (t < hi) ? cnt[t] : 0u;
        u32 incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const u32 v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += v; }
        if (t < hi) base[t] = run + (incl - c);
        run += __shfl_sync(0xffffffffu, incl, 31);
    }
}

// One warp on segment t of the segmented stream: lane l owns offsets [16l, 16l+16).  tok(i) reads across the segment's
// ends (two tokens back, three ahead; TOK_SENTINEL past the ends of the stream); entry(i) is the entry holding offset i
// for offsets visited in ascending order from 16l.
struct WtSeg {
    const u32 *seg;
    u32 count, lo, hi;
    u32 N[3], P[2];
    u64 ent;        // entry of the last mark seen, + 1 (base[t] + marks in [0, i])
    __device__ __forceinline__ u32 tok(int i) const {
        if (i < 0) return P[-1 - i];
        if ((u32)i >= count) return N[i - (int)count];
        return seg[i];
    }
};

__device__ __forceinline__ WtSeg wt_seg_begin(const u32 *w, const Edge *e, u32 t, u32 nseg, const u64 *base) {
    WtSeg s;
    const u32 lane = lane_id();
    s.seg = w + (u64)t * SEG_TOKENS;
    s.count = e[t].count;
    s.lo = min(s.count, lane * 16u);
    s.hi = min(s.count, s.lo + 16u);
    seg_neighbours(e, t, nseg, s.N, s.P);
    u32 own = 0;
    for (u32 i = s.lo; i < s.hi; ++i) own += s.seg[i] >> 31;
    u32 incl = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const u32 v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += v; }
    s.ent = base[t] + (incl - own);
    return s;
}

// Iteration 0 on a weighted stream: every pair of the stream adds its entry's weight to the table (get_stats() of the
// whole text: regex.py:51-54 summed over the occurrences each entry stands for).
__global__ void __launch_bounds__(256) k_wt_hist(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1, Ctl *ctl,
                                                 const Edge *e0, const Edge *e1, const u64 *__restrict__ base,
                                                 const u64 *__restrict__ wts, Table tab) {
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);
    const u32 nseg = ctl->nseg;
    const u32 wpb = blockDim.x >> 5;
    for (u32 t = blockIdx.x * wpb + (threadIdx.x >> 5); t < nseg; t += gridDim.x * wpb) {
        WtSeg s = wt_seg_begin(w, e, t, nseg, base);
        for (u32 i = s.lo; i < s.hi; ++i) {
            const u32 t0 = s.seg[i], t1 = s.tok((int)i + 1);
            s.ent += t0 >> 31;
            if (t1 & TOK_FLAG) continue;   // next chunk, or the end of the stream
            hist_global_add(tab, ctl, pack_pair(t0 & TOK_MASK, t1), (ull)wts[s.ent - 1], 0);
        }
    }
}

// the member of the pass (ids at ma[j], mb[j]) whose merge starts at the token pair (x, y); nk: none
__device__ __forceinline__ u32 wt_member(u32 x, u32 y, u32 nk, const u32 *ma, const u32 *mb) {
    u32 j = 0;
    for (; j < nk; ++j) if ((x & TOK_MASK) == ma[j] && y == mb[j]) break;
    return j;
}

// Statistics delta of a merge pass with a != b on the segmented stream, weighted: the rules of delta_one / delta_batch
// (k_merge_seg.cuh) with the weight of the merge's entry in place of 1.  Runs before the merge pass, on the stream the
// pass reads.  batched: the ctl->nk members k_select_batch chose, one delta vector of 2V+1 counters each.
__global__ void __launch_bounds__(256) k_wt_delta_seg(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1, const Ctl *ctl,
                                                      const Edge *e0, const Edge *e1, const u64 *__restrict__ base,
                                                      const u64 *__restrict__ wts, ull *__restrict__ delta, u32 V,
                                                      int batched, int force) {
    if (!force && (ctl->done || ctl->overflow || ctl->iter >= ctl->max_iter)) return;
    if (ctl->a == ctl->b) return;
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const Edge *e = edges_cur(ctl, e0, e1);
    const u32 nseg = ctl->nseg;
    const u32 nk = batched ? ctl->nk : 1u, z = (u32)ctl->z;
    u32 ma[BATCH_MAX], mb[BATCH_MAX];
    ma[0] = (u32)ctl->a; mb[0] = (u32)ctl->b;
    for (u32 j = 1; j < nk; ++j) { ma[j] = (u32)ctl->bat_a[j]; mb[j] = (u32)ctl->bat_b[j]; }
    const u32 wpb = blockDim.x >> 5;
    for (u32 t = blockIdx.x * wpb + (threadIdx.x >> 5); t < nseg; t += gridDim.x * wpb) {
        WtSeg s = wt_seg_begin(w, e, t, nseg, base);
        for (u32 i = s.lo; i < s.hi; ++i) {
            const int p = (int)i;
            const u32 t0 = s.seg[i];
            s.ent += t0 >> 31;
            const u32 j = wt_member(t0, s.tok(p + 1), nk, ma, mb);
            if (j == nk) continue;
            const ull wt = wts[s.ent - 1];
            const u32 tm1 = s.tok(p - 1), tm2 = s.tok(p - 2), tp2 = s.tok(p + 2), tp3 = s.tok(p + 3);
            const u32 ml = wt_member(tm2, tm1, nk, ma, mb);   // member starting two tokens earlier
            const u32 mr = wt_member(tp2, tp3, nk, ma, mb);   // member starting two tokens later
            ull *d = delta + (u64)j * (2ull * V + 1);
            if (tm1 != TOK_SENTINEL && !(t0 & TOK_FLAG) && ml != j) atomicAdd(&d[ml < j ? z + ml : tm1 & TOK_MASK], wt);
            if (!(tp2 & TOK_FLAG)) atomicAdd(&d[mr == j ? 2ull * V : (u64)V + (mr < j ? z + mr : tp2)], wt);
        }
    }
}

// Statistics delta of a merge of a pair (a,a), weighted, on the stream enqueue_pack has just made contiguous (the same
// gate as the pack).  The greedy left-to-right rule of k_merge<true>: e(q) = "q continues a run of a", a merge starts at
// p iff e(p+1) and the run of e's ending at p has even length.  One thread per 512-token block walks it in order.
__global__ void __launch_bounds__(256) k_wt_delta_same(const u32 *__restrict__ buf0, const u32 *__restrict__ buf1, const Ctl *ctl,
                                                       const u64 *__restrict__ base, const u64 *__restrict__ wts,
                                                       ull *__restrict__ delta, u32 V, int force) {
    if (!pack_wanted(ctl, force)) return;
    const u32 *__restrict__ w = ctl->cur ? buf1 : buf0;
    const u64 n = ctl->n;
    const u32 a = (u32)ctl->a;
    const u64 nblk = (n + SEG_TOKENS - 1) / SEG_TOKENS;
    auto ev = [&](long long q) -> bool { return q >= 1 && (u64)q < n && w[q] == a && (w[q - 1] & TOK_MASK) == a; };
    for (u64 blk = (u64)blockIdx.x * blockDim.x + threadIdx.x; blk < nblk; blk += (u64)gridDim.x * blockDim.x) {
        const long long s = (long long)blk * SEG_TOKENS;
        const long long end = min((long long)n, s + SEG_TOKENS);
        u32 par = 0;                                        // parity of the run of e's ending at q (q = s - 5 here)
        for (long long q = s - 5; ev(q); --q) par ^= 1u;
        u32 m4 = 0, m3 = 0, m2 = 0, m1 = 0;                 // m(q-4) .. m(q-1)
        u64 ent = base[blk];                                // base + marks in [s, p]
        for (long long q = s - 4; q <= end + 1; ++q) {
            if (q >= 0) par = ev(q) ? (par ^ 1u) : 0u;
            const u32 m0 = (q >= 0 && ev(q + 1) && !par) ? 1u : 0u;
            const long long p = q - 2;                      // m(p-2) = m4, m(p) = m2, m(p+2) = m0
            if (p >= s) {
                const u32 tp = w[p];
                ent += tp >> 31;
                if (m2) {
                    const ull wt = wts[ent - 1];
                    if (p >= 1 && !(tp & TOK_FLAG) && !m4) atomicAdd(&delta[w[p - 1] & TOK_MASK], wt);
                    if ((u64)p + 2 < n) {
                        const u32 y = w[p + 2];
                        if (!(y & TOK_FLAG)) atomicAdd(&delta[m0 ? 2ull * V : (u64)V + y], wt);
                    }
                }
            }
            m4 = m3; m3 = m2; m2 = m1; m1 = m0;
        }
    }
}
