// common.cuh — shared definitions for the sm_90a BPE kernels.
#pragma once
#ifndef BPE_SIMT_EMU
#include <cuda_runtime.h>
#endif
#include <stdint.h>

typedef uint32_t u32;
typedef uint64_t u64;
typedef unsigned long long ull;

// ---- token words ---------------------------------------------------------------------------
// The stream is one 32-bit word per token: bits 0..30 = id, bit 31 = "first token of a chunk".
// A pair (w[p], w[p+1]) exists iff p+1 < n and w[p+1] has no chunk mark (regex.py:51-54: stats
// are accumulated chunk by chunk, so no pair spans two chunks).  Comparing w[p+1] against an
// unmarked id therefore tests "same id AND same chunk" in one instruction.
#define TOK_FLAG 0x80000000u
#define TOK_MASK 0x7fffffffu
#define TOK_SENTINEL 0xffffffffu  // out-of-range filler: marked, id 0x7fffffff never used

// ---- pair-count table ----------------------------------------------------------------------
#define KEY_EMPTY 0xffffffffffffffffull
#define POS_NONE 0xffffffffffffffffull

__host__ __device__ __forceinline__ u64 pack_pair(u32 a, u32 b) { return ((u64)a << 32) | (u64)b; }

__host__ __device__ __forceinline__ u64 hash64(u64 x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33; return x;
}

struct Table {
    u64 *keys;    // [cap]  packed pair or KEY_EMPTY
    u64 *counts;  // [cap]  occurrences in the current stream (global count when sharded)
    u64 *first;   // [cap]  first position (only maintained by the full-histogram kernel), may be NULL
    u64 mask;     // cap - 1
};

// Find the slot of `key`, inserting it (count 0) if absent.  *inserted counts new slots.
__device__ __forceinline__ u64 table_upsert(const Table &t, u64 key, ull *used_counter) {
    u64 slot = hash64(key) & t.mask;
    for (;;) {
        u64 k = t.keys[slot];
        if (k == key) return slot;
        if (k == KEY_EMPTY) {
            u64 old = atomicCAS((ull *)&t.keys[slot], (ull)KEY_EMPTY, (ull)key);
            if (old == KEY_EMPTY) { if (used_counter) atomicAdd(used_counter, 1ull); return slot; }
            if (old == key) return slot;
        }
        slot = (slot + 1) & t.mask;
    }
}

// Slot of `key` or POS_NONE.
__device__ __forceinline__ u64 table_find(const Table &t, u64 key) {
    u64 slot = hash64(key) & t.mask;
    for (;;) {
        u64 k = t.keys[slot];
        if (k == key) return slot;
        if (k == KEY_EMPTY) return POS_NONE;
        slot = (slot + 1) & t.mask;
    }
}

// ---- device-resident control block ---------------------------------------------------------
// Most merges one pass of bpe_train's loop may carry (k_select_batch): each member adds a delta vector of 2V+1 counters.
#ifndef BATCH_MAX
#define BATCH_MAX 4
#endif
// Everything the per-iteration kernels need to chain without the host: stream length, which
// ping-pong buffer is current, the pair selected for the next merge, tickets.
struct Ctl {
    u64 n;            // current stream length (tokens)
    u64 n_next;       // written by the tile that ends the stream during a merge
    u32 cur;          // index of the ping-pong buffer holding the current stream
    u32 iter;         // merges completed
    u32 done;         // 1: no pair left (the reference raises ValueError here)
    u32 epoch;        // look-back descriptor epoch: +1 per merge launch, never reset (starts at 1)
    int a, b, z;      // pair selected for merge `iter`, and its new id
    u32 n_tied;       // number of pairs at the max count
    u64 best_count;   // max count
    u64 best_slot;    // a slot holding the max count
    u64 found_pos;    // find-first result (POS_NONE = not found)
    ull table_used;   // occupied table slots
    u32 merge_ticket; // tile dispenser of the merge kernel
    u32 merge_exit;   // CTAs that left the merge kernel
    u32 argmax_exit;
    u32 ff_exit;
    u64 sum_in, sum_out;  // sum over iterations of n before / after (for GB/s accounting)
    u32 first_idx;
    u32 max_iter;     // stop after this many merges
    // segmented stream (DESIGN.md "Stream layout"): nseg segments of SEG_TOKENS capacity each
    u32 nseg;         // segments in use
    u32 edge_cur;     // which of the two edge arrays describes the current stream
    ull drops;        // tokens removed by the merge in flight (summed by CTAs at exit)
    u32 gather_exit;
    u32 contig;       // 1: the current buffer is a contiguous stream whose edge records are stale
    u64 table_limit;  // k_apply_delta stops inserting at this many occupied slots ...
    u32 overflow;     // ... and raises this; the host grows the table and re-runs the apply
    u32 tie_local;    // sharded loop: 1 = some pair tied at the max may occur in this rank's shard (k_tie_present)
    // segment filter (k_seg_filter.cuh) — appended, so that the offsets every other kernel uses do not move
    u32 n_cand;       // candidate segments of the merge in flight (entries of the list at cand_ptr)
    u64 cand_ptr;     // device address of u32 cand[]
    u64 cand_sum;     // sum of n_cand over the filtered merges of this bpe_train call (statistics)
    u64 seg_sum;      // sum of nseg over the same merges
    // batched merge pass (k_select_batch, DESIGN.md "Batched merges") — appended as well
    u32 nk;                   // merges of the pass in flight: member 0 = (a, b) -> z, member j = (bat_a[j], bat_b[j]) -> z + j
    int bat_a[BATCH_MAX], bat_b[BATCH_MAX];   // [0] unused
};

// ---- segmented stream ------------------------------------------------------------------------
// The stream lives in fixed segments of SEG_TOKENS words: segment t owns words
// [t*SEG_TOKENS, (t+1)*SEG_TOKENS) and holds `count` tokens at its start.  A merge compacts
// every segment in place, so no cross-segment prefix sum (and no serial dependency between warps)
// is needed; the stream order is (segment, offset).  One segment = the 512 tokens one warp keeps
// in registers (16 per lane), so the merge pass needs no block-level synchronisation at all.
// Edge records let a warp see the tokens next to its segment without touching the neighbour's
// body while that body is being rewritten; they are double-buffered by merge parity.
#define SEG_TOKENS 512
#define SEG_SHIFT 9
struct __align__(32) Edge {
    u32 f[3];    // first three tokens (TOK_SENTINEL where the segment is shorter)
    u32 l[2];    // last two tokens: l[1] = last, l[0] = the one before it
    u32 count;
    u32 pad[2];
};

// ---- exchange block of the sharded loop (k_xchg.cuh): header + two delta vectors, in every rank's HBM ----
#define XCHG_MAX_RANKS 16
#define XCHG_HDR_BYTES 1024

struct XHdr {
    u32 seq;                          // exchange rounds completed (local copy; identical on every rank)
    u32 exit_count;                   // blocks that left k_xchg_apply
    u32 applied;                      // ctl->iter up to which the table has been updated (an iteration whose merge was
                                      // gated off — done, max_iter — must not run an exchange round either)
    u32 pad;
    u64 dflag[XCHG_MAX_RANKS];        // dflag[r] = s+1: rank r's delta of round s is complete
    u64 cflag[XCHG_MAX_RANKS];        // cflag[r] = s+1: rank r's candidate of round s is in cand[r]
    long long cand[XCHG_MAX_RANKS];
    u64 pflag[XCHG_MAX_RANKS];        // bpe_xchg_probe: pflag[r] = probe round rank r has reached
    u64 magic;                        // written at creation; a peer that can read it can pull from this block
    u64 probe_round;
};
static_assert(sizeof(XHdr) <= XCHG_HDR_BYTES, "exchange header must fit its slot");

// the delta buffer the merge kernels of round XHdr.seq add into
__device__ __forceinline__ ull *x_local_delta(const unsigned char *xbase, u64 delta_stride) {
    const u32 s = reinterpret_cast<const XHdr *>(xbase)->seq;
    return reinterpret_cast<ull *>(const_cast<unsigned char *>(xbase) + XCHG_HDR_BYTES + (u64)(s & 1u) * delta_stride);
}

// ---- small helpers -------------------------------------------------------------------------
#ifndef BPE_SIMT_EMU
__device__ __forceinline__ u64 ld_volatile_u64(const u64 *p) {
    u64 v;
    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_volatile_u64(u64 *p, u64 v) {
    asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ u32 ld_volatile_u32(const u32 *p) {
    u32 v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
#endif
__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }

#ifndef BPE_SIMT_EMU
// ---- mbarrier + bulk async copy (TMA 1-D) — hand-written PTX for sm_90a ----------------------
__device__ __forceinline__ u32 smem_addr(const void *p) { return (u32)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(u64 *bar, u32 count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
// make mbarrier initialisation visible to the async proxy before the first bulk copy targets it
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// ordinary shared-memory stores before a bulk copy that overwrites the same bytes
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- shared memory through 32-bit shared-window addresses kept in registers.  Generic pointers into dynamic
//      shared memory make the compiler rebuild the window base (S2R SR_CgaCtaId + LEA) and the index
//      arithmetic in front of every access; the merge kernel's inner loop addresses shared memory
//      explicitly instead. ----
__device__ __forceinline__ u32 lds32(u32 addr) {
    u32 v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
template <int OFF>
__device__ __forceinline__ u32 lds32o(u32 addr) {
    u32 v;
    asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(addr), "n"(OFF) : "memory");
    return v;
}
template <int OFF>
__device__ __forceinline__ uint4 lds128o(u32 addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4+%5];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr), "n"(OFF) : "memory");
    return v;
}
__device__ __forceinline__ void sts32(u32 addr, u32 v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
template <int OFF>
__device__ __forceinline__ void sts32o(u32 addr, u32 v) { asm volatile("st.shared.u32 [%0+%1], %2;" ::"r"(addr), "n"(OFF), "r"(v) : "memory"); }
__device__ __forceinline__ void sts128(u32 addr, u32 x, u32 y, u32 z, u32 w) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_a(u32 bar_a, u32 tx_bytes) {
    u64 state;
    asm volatile("mbarrier.arrive.expect_tx.release.cta.shared::cta.b64 %0, [%1], %2;" : "=l"(state) : "r"(bar_a), "r"(tx_bytes) : "memory");
    (void)state;
}
// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes (or 20 us elapse)
// instead of burning issue slots in a polling loop; wake-up on completion is immediate
__device__ __forceinline__ void mbar_wait_a(u32 bar_a, u32 parity) {
    u32 ok;
    do {
        asm volatile("{\n\t.reg .pred P;\n\t"
                     "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\t"
                     "selp.b32 %0, 1, 0, P;\n\t}"
                     : "=r"(ok) : "r"(bar_a), "r"(parity), "r"(20000u) : "memory");
    } while (!ok);
}
// global -> shared bulk copy (SASS: UBLKCP); bytes, src and dst must be multiples of 16
__device__ __forceinline__ void bulk_g2s_a(u32 dst_a, const void *src_gmem, u32 bytes, u32 bar_a) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_a), "l"(src_gmem), "r"(bytes), "r"(bar_a) : "memory");
}

#else  // BPE_SIMT_EMU ================================================================================
// The same helpers for the CPU SIMT emulator (tests/emu/cuda_emu.h — test infrastructure, never part of
// libb200bpe.so): polling loads yield to the other emulated threads, "shared-window addresses" are byte
// offsets into the block's dynamic shared memory, a bulk copy completes at issue, and the mbarrier word keeps
// {outstanding bytes, pending arrivals, phase} with the PTX phase/parity semantics.
static inline u64 ld_volatile_u64(const u64 *p) { emu::spin(); return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
static inline void st_volatile_u64(u64 *p, u64 v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
static inline u32 ld_volatile_u32(const u32 *p) { emu::spin(); return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
static inline char *emu_smem() { return reinterpret_cast<char *>(emu::dyn_smem()); }
static inline u32 smem_addr(const void *p) { return (u32)(reinterpret_cast<const char *>(p) - emu_smem()); }
struct EmuMbar { int tx; unsigned char pending, init; unsigned short phase; };
static_assert(sizeof(EmuMbar) == 8, "one mbarrier word");
static inline void emu_mbar_check(EmuMbar *m) { if (m->pending == 0 && m->tx == 0) { m->phase ^= 1u; m->pending = m->init; } }
static inline void mbar_init(u64 *bar, u32 count) { EmuMbar *m = reinterpret_cast<EmuMbar *>(bar); m->tx = 0; m->pending = m->init = (unsigned char)count; m->phase = 0; }
static inline void fence_mbar_init() {}
static inline void fence_proxy_async_smem() {}
static inline u32 lds32(u32 addr) { return *reinterpret_cast<u32 *>(emu_smem() + addr); }
template <int OFF> static inline u32 lds32o(u32 addr) { return *reinterpret_cast<u32 *>(emu_smem() + addr + OFF); }
template <int OFF> static inline uint4 lds128o(u32 addr) { return *reinterpret_cast<uint4 *>(emu_smem() + addr + OFF); }
static inline void sts32(u32 addr, u32 v) { *reinterpret_cast<u32 *>(emu_smem() + addr) = v; }
template <int OFF> static inline void sts32o(u32 addr, u32 v) { *reinterpret_cast<u32 *>(emu_smem() + addr + OFF) = v; }
static inline void sts128(u32 addr, u32 x, u32 y, u32 z, u32 w) { *reinterpret_cast<uint4 *>(emu_smem() + addr) = make_uint4(x, y, z, w); }
static inline void mbar_arrive_expect_tx_a(u32 bar_a, u32 tx_bytes) {
    EmuMbar *m = reinterpret_cast<EmuMbar *>(emu_smem() + bar_a);
    m->tx += (int)tx_bytes; m->pending -= 1; emu_mbar_check(m);
}
static inline void mbar_wait_a(u32 bar_a, u32 parity) {
    const EmuMbar *m = reinterpret_cast<const EmuMbar *>(emu_smem() + bar_a);
    while ((u32)(m->phase & 1u) == parity) emu::spin();      // the phase with this parity has not completed yet
}
static inline void bulk_g2s_a(u32 dst_a, const void *src_gmem, u32 bytes, u32 bar_a) {
    memcpy(emu_smem() + dst_a, src_gmem, bytes);
    EmuMbar *m = reinterpret_cast<EmuMbar *>(emu_smem() + bar_a);
    m->tx -= (int)bytes; emu_mbar_check(m);
}
#endif
