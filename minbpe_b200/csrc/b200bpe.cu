// b200bpe.cu — host side of libb200bpe.so: the C ABI of include/b200bpe.h over the sm_90a
// kernels in k_load.cuh / k_stats.cuh / k_merge.cuh / k_encode.cuh.
//
// Build: see build.py (nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -shared).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "../../include/b200bpe.h"
#include "common.cuh"
#include "k_load.cuh"
#include "k_merge.cuh"
#include "k_merge_seg.cuh"
#include "k_seg.cuh"
#include "k_seg_filter.cuh"
#include "k_stats.cuh"
#include "k_encode.cuh"
#include "k_split.cuh"
#include "k_decode.cuh"
#include "k_xchg.cuh"
#include "k_encode2.cuh"
#include "k_special.cuh"
#include "k_weighted.cuh"
#include "k_dedup.cuh"

#define BPE_ABI_VERSION 6

namespace {   // the owner types stay private to the library: they add no exported symbol

// A device allocation of `cap` elements of T with one owner: the destructor frees it, a move hands it on, a copy does not
// compile.  It converts to T *, so kernel arguments and cudaMemcpyAsync / cudaMemsetAsync take it as they are.
template <class T>
struct DevBuf {
    T *p = nullptr;
    u64 cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) { reset(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
        return *this;
    }
    ~DevBuf() { reset(); }
    void reset() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    operator T *() const { return p; }
    T *operator->() const { return p; }   // device addresses of fields (&h->ctl->n)
};

// A CUDA event with one owner (timing on the handle's stream)
struct Event {
    cudaEvent_t e = nullptr;
    Event() = default;
    Event(const Event &) = delete;
    Event &operator=(const Event &) = delete;
    Event(Event &&o) noexcept : e(o.e) { o.e = nullptr; }
    ~Event() { if (e) cudaEventDestroy(e); }
    cudaError_t create() { return cudaEventCreate(&e); }
    operator cudaEvent_t() const { return e; }
};

// The pair-count table's device arrays; the kernels take the Table view by value
struct PairTable {
    DevBuf<u64> keys, counts, first;
    u64 mask = 0;   // slots - 1
    operator Table() const { return {keys, counts, first, mask}; }
};

}  // namespace

struct EncState;
struct SpecSet;
struct GenEnc;
struct DdSession;
struct bpe_handle {
    int device = 0;
    std::unique_ptr<EncState> enc;       // memoised chunk encode (encode2_host.inl): rank table, memo, id pool, scratch
    std::unique_ptr<bpe_handle, int (*)(bpe_handle *)> enc_scratch{nullptr, bpe_destroy};   // general encode path
                                         // (encode_host.inl) works on its own stream buffers
    std::unique_ptr<SpecSet> spec;       // special tokens of the current encode call (special_host.inl)
    std::unique_ptr<GenEnc> gen;         // general encode path: device scratch + the rank table of the last merges seen (encode_host.inl)
    std::unique_ptr<DdSession> dd;       // counting session of bpe_dedup_begin / _add_docs / _finish (dedup_host.inl)
    int sms = 0;
    cudaStream_t stream = nullptr;       // the stream every kernel of this handle runs on
    cudaStream_t own_stream = nullptr;   // created by bpe_create; `stream` may point at a caller's stream instead
    std::string err;

    // token stream: two ping-pong buffers
    DevBuf<u32> buf[2];
    bool loaded = false;
    bool bytes_only = false;  // every id < 256 (fresh byte stream)
    // weighted stream (bpe_load_chunks_weighted, k_weighted.cuh): one weight per entry, the entry base of every segment
    bool weighted = false;
    DevBuf<u64> wts; u64 n_entries = 0;
    DevBuf<u32> wt_cnt; DevBuf<u64> wt_base;
    bool wt_fresh = false;    // the weighted stream is as loaded: no bpe_train / bpe_replay since (bpe_read_chunk_entries)

    DevBuf<Ctl> ctl;       // device
    Ctl *h_ctl = nullptr;  // pinned host mirror

    PairTable table;
    bool table_valid = false;  // table == get_stats(current stream)
    DevBuf<u64> desc;
    DevBuf<Edge> edge[2]; DevBuf<u64> seg_offs;   // segmented stream metadata
    DevBuf<ull> delta; u32 V = 0;      // V = layout of the delta vector the kernels index (L[0,V) R[V,2V) ZZ[2V])
    u32 delta_cap = 0;                 // vocabulary capacity of the OWNED buffer `delta` (step mode uses the caller's)
    u32 delta_vecs = 0;                // delta vectors of 2*delta_cap+1 counters in it: one per member of a batched pass
    bool batching = false;             // bpe_train's loop may carry several merges per pass (k_select_batch)
    u32 max_id = 255;                  // largest id in the loaded stream (bpe_load_ids); byte streams: 255
    DevBuf<ull> dense;
    DevBuf<ull> dense2; DevBuf<u32> d_cmp;         // first-use cross-check of the packed histogram kernel (hist_dense)
    int hist_mode = 0;                             // 0 = not decided, 1 = k_hist_dense_packed, 2 = k_hist_dense
    // segment filter (k_seg_filter.cuh): signatures, candidate list
    DevBuf<u32> sig, cand;
    bool filt_active = false;                      // the iterations being enqueued use the filter
    bool sig_valid = false;                        // the signatures describe the current stream
    DevBuf<u32> d_err;
    DevBuf<int> log_pairs; DevBuf<long long> log_counts;
    DevBuf<Best> partials;
    DevBuf<TopList> top_partials;      // k_select_batch: one list per block
    DevBuf<unsigned char> d_cls, d_contr;   // code-point class / contraction tables of the GPT-4 splitter
    DevBuf<unsigned char> d_cls_o200k;      // class table of the o200k split: GPT-4 class | case class << 5 (bpe_o200k_table)
    // sharded loop over NVLink peer memory (k_xchg.cuh): the rank's exchange block and its peers' mappings
    unsigned char *xchg = nullptr; u64 xchg_bytes = 0, xchg_stride = 0; u32 xchg_V = 0;
    XArgs xargs = {};
    bool xchg_attached = false;
    DevBuf<u32> d_present;      // sharded loop: bitmap of pair hashes that have occurred in this shard (k_stats.cuh)
    DevBuf<unsigned char> split_slab;   // working set of the splitter, kept between calls (split_host.inl)
    int argmax_grid = 0, merge_grid_same = 0, merge_grid_seg = 0, ff_grid = 0;

    // options
    int step_poll_every = 16;
    int opt_kernel_timing = 0, opt_rescan = 0, opt_batch = 256, opt_table_log2 = 0;
    int opt_memo_log2 = 0;   // BPE_OPT_ENC_MEMO_LOG2 (test hook): log2 slots of the encode memo table, 0 = default
    u32 opt_vocab_cap = 0;   // BPE_OPT_VOCAB_CAP: lower bound of the delta-vector layout V used by bpe_train
    int opt_seg_filter = 0;      // BPE_OPT_SEG_FILTER: 0 = off, 1 = switch it on when merges have become sparse, 2 = always
    int opt_hist_kernel = 2;     // BPE_OPT_HIST_KERNEL: 2 = k_hist_dense (default), 1 = k_hist_dense_packed,
                                 // 0 = decide at the first large stream (cross-check + timing)
    int opt_dedup_log2 = 0;      // BPE_OPT_DEDUP_LOG2 (test hook): log2 slots of the chunk table of bpe_load_text_gpt4_dedup, 0 = default
    u64 dd_stats[8] = {};        // bpe_dedup_stats of the last bpe_load_text_gpt4_dedup / bpe_dedup_finish
    int opt_split_pattern = 0;   // BPE_OPT_SPLIT_PATTERN: 0 = GPT-4 split pattern, 1 = GPT-2, 3 = o200k (bpe_split_gpt4 / bpe_load_text_gpt4 / bpe_encode_text_gpt4*)

    bpe_timing tm = {};
    std::vector<Event> ev_pool;  // per-launch timing of the fused merge kernel (BPE_OPT_KERNEL_TIMING)
    int ev_used = 0;

    __attribute__((visibility("hidden"))) ~bpe_handle();   // after the .inl files, where the sub-states are complete types
};

static thread_local std::string g_create_err;
static void xchg_release(bpe_handle *h);
static u64 g_split_piece_override = 0;   // BPE_OPT_SPLIT_PIECE (test hook): bytes per piece of the device splitter

static int fail(bpe_handle *h, int code, const std::string &msg) {
    if (h) h->err = msg; else g_create_err = msg;
    return code;
}

#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return fail(h, BPE_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));      \
    } while (0)

static inline int grid_for(u64 work_items, int threads, int max_blocks) {
    u64 b = (work_items + threads - 1) / threads;
    if (b < 1) b = 1;
    if (b > (u64)max_blocks) b = max_blocks;
    return (int)b;
}

extern "C" int bpe_abi_version(void) { return BPE_ABI_VERSION; }

extern "C" const char *bpe_last_error(const bpe_handle *h) { return h ? h->err.c_str() : g_create_err.c_str(); }

// ------------------------------------------------------------------------------------------------
// Room for `need` elements; the contents are not kept.  A buffer that is too small is freed FIRST and then allocated
// again with `alloc` elements (default: `need`), so the old and the new block never coexist; if that fails, the buffer is
// left empty.
template <class T>
static int dev_reserve(bpe_handle *h, DevBuf<T> &b, u64 need, u64 alloc = 0) {
    if (need <= b.cap) return BPE_OK;
    b.reset();
    const u64 n = std::max(need, alloc);
    T *q = nullptr;
    const cudaError_t e = cudaMalloc(&q, n * sizeof(T));
    if (e != cudaSuccess)
        return fail(h, BPE_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
    b.p = q; b.cap = n;
    return BPE_OK;
}

// Room for `need` elements, keeping the first `used`: the buffer at least doubles when it grows.
template <class T>
static int dev_grow(bpe_handle *h, DevBuf<T> &b, u64 need, u64 used) {
    if (need <= b.cap) return BPE_OK;
    DevBuf<T> nb;
    int rc = dev_reserve(h, nb, std::max<u64>(need, 1), b.cap * 2);
    if (rc) return rc;
    if (used) CU(cudaMemcpyAsync(nb, b, used * sizeof(T), cudaMemcpyDeviceToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    b = std::move(nb);
    return BPE_OK;
}

// `cap` empty slots (with_first: first positions too); arrays of another size are freed before the new ones are allocated
static int table_reset(bpe_handle *h, PairTable &t, u64 cap, bool with_first) {
    if (!t.keys || t.mask + 1 != cap) {
        t = PairTable();
        int rc;
        if ((rc = dev_reserve(h, t.keys, cap)) || (rc = dev_reserve(h, t.counts, cap)) ||
            (with_first && (rc = dev_reserve(h, t.first, cap)))) { t = PairTable(); return rc; }
        t.mask = cap - 1;
    }
    CU(cudaMemsetAsync(t.keys, 0xff, cap * 8, h->stream));
    CU(cudaMemsetAsync(t.counts, 0, cap * 8, h->stream));
    if (with_first) CU(cudaMemsetAsync(t.first, 0xff, cap * 8, h->stream));
    return BPE_OK;
}

static u64 next_pow2(u64 x) { u64 p = 1; while (p < x) p <<= 1; return p; }

// stream, control block, histogram scratch, launch geometry of a new handle; errors go to h->err
static int handle_init(bpe_handle *h, int device, const cudaDeviceProp &prop) {
    h->device = device;
    h->sms = prop.multiProcessorCount;
    CU(cudaSetDevice(device));
    CU(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    h->stream = h->own_stream;
    int rc;
    if ((rc = dev_reserve(h, h->ctl, 1))) return rc;
    CU(cudaMallocHost(&h->h_ctl, sizeof(Ctl)));
    if ((rc = dev_reserve(h, h->dense, 65536)) || (rc = dev_reserve(h, h->d_err, 2)))   // d_err: [0] error flag, [1] max id seen by k_copy_ids
        return rc;
    int occ_same = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_same, k_merge<true>, MG_THREADS, 0);
    if (occ_same < 1) occ_same = 1;
    h->merge_grid_same = h->sms * occ_same;
    int occ_fast = 0;
    CU(cudaFuncSetAttribute(k_merge_seg<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, MS_SMEM_BYTES));
    CU(cudaFuncSetAttribute(k_merge_seg<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, MS_SMEM_BYTES));
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_fast, k_merge_seg<false>, MS_THREADS, MS_SMEM_BYTES);
    if (occ_fast < 1) return fail(h, BPE_ERR_CUDA, "k_merge_seg does not fit on an SM");
    h->merge_grid_seg = h->sms * occ_fast;
    h->argmax_grid = h->sms * 2;
    h->ff_grid = h->sms * 4;
    if ((rc = dev_reserve(h, h->partials, h->argmax_grid)) || (rc = dev_reserve(h, h->top_partials, h->argmax_grid))) return rc;
    memset(h->h_ctl, 0, sizeof(Ctl));
    h->h_ctl->epoch = 1;
    h->h_ctl->found_pos = POS_NONE;
    CU(cudaMemcpy(h->ctl, h->h_ctl, sizeof(Ctl), cudaMemcpyHostToDevice));
    return BPE_OK;
}

extern "C" int bpe_create(int device, bpe_handle **out) {
    if (!out) return fail(nullptr, BPE_ERR_ARG, "bpe_create: out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, BPE_ERR_CUDA, std::string("bpe_create: no CUDA device (") + cudaGetErrorString(e) +
                                               "); libb200bpe has no CPU fallback");
    if (device < 0 || device >= ndev) return fail(nullptr, BPE_ERR_ARG, "bpe_create: device index out of range");
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, device);
    if (e != cudaSuccess) return fail(nullptr, BPE_ERR_CUDA, cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return fail(nullptr, BPE_ERR_CUDA, std::string("bpe_create: device '") + prop.name + "' is sm_" +
                                               std::to_string(prop.major) + std::to_string(prop.minor) +
                                               "; this library contains sm_90a code only");
    std::unique_ptr<bpe_handle> owner(new (std::nothrow) bpe_handle());   // frees whatever was made if a step fails
    if (!owner) return fail(nullptr, BPE_ERR_INTERNAL, "out of host memory");
    if (int rc = handle_init(owner.get(), device, prop)) return fail(nullptr, rc, owner->err);
    *out = owner.release();
    return BPE_OK;
}

extern "C" int bpe_destroy(bpe_handle *h) {
    if (!h) return BPE_OK;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    xchg_release(h);
    delete h;   // every buffer, event and sub-state has its owner in the handle
    return BPE_OK;
}

extern "C" int bpe_set_option(bpe_handle *h, int opt, int64_t value) {
    if (!h) return BPE_ERR_ARG;
    switch (opt) {
        case BPE_OPT_KERNEL_TIMING: h->opt_kernel_timing = value != 0; break;
        case BPE_OPT_RESCAN: h->opt_rescan = value != 0; break;
        case BPE_OPT_BATCH: h->opt_batch = (int)std::max<int64_t>(1, std::min<int64_t>(value, 4096)); break;
        case BPE_OPT_TABLE_LOG2:
            if (value != 0 && (value < 10 || value > 30)) return fail(h, BPE_ERR_ARG, "table log2 must be 0 or in [10,30]");
            h->opt_table_log2 = (int)value; break;
        case BPE_OPT_VOCAB_CAP:
            if (value < 0 || value >= 0x3fffffff) return fail(h, BPE_ERR_ARG, "vocabulary capacity out of range");
            h->opt_vocab_cap = (u32)value; break;
        case BPE_OPT_ENC_MEMO_LOG2:
            if (value != 0 && (value < 6 || value > 28)) return fail(h, BPE_ERR_ARG, "memo log2 must be 0 or in [6,28]");
            h->opt_memo_log2 = (int)value;
            cudaSetDevice(h->device); cudaStreamSynchronize(h->stream);
            h->enc.reset();   // re-created with the new size by the next encode call
            break;
        case BPE_OPT_SEG_FILTER:
            if (value < 0 || value > 2) return fail(h, BPE_ERR_ARG, "segment filter must be 0 (off), 1 (when sparse) or 2 (always)");
            h->opt_seg_filter = (int)value; h->filt_active = false; h->sig_valid = false;
            break;
        case BPE_OPT_HIST_KERNEL:
            if (value < 0 || value > 2) return fail(h, BPE_ERR_ARG, "hist kernel must be 0 (auto), 1 (packed) or 2 (hashed)");
            h->opt_hist_kernel = (int)value;
            if (value == 0) h->hist_mode = 0;
            break;
        case BPE_OPT_SPLIT_PATTERN:
            if (value != 0 && value != 1 && value != 3) return fail(h, BPE_ERR_ARG, "split pattern must be 0 (GPT-4), 1 (GPT-2) or 3 (o200k)");
            h->opt_split_pattern = (int)value; break;
        case BPE_OPT_DEDUP_LOG2:
            if (value != 0 && (value < 4 || value > 30)) return fail(h, BPE_ERR_ARG, "dedup log2 must be 0 or in [4,30]");
            h->opt_dedup_log2 = (int)value; break;
        case BPE_OPT_SPLIT_PIECE:
            if (value != 0 && value < 4096) return fail(h, BPE_ERR_ARG, "split piece must be 0 (default) or >= 4096 bytes");
            g_split_piece_override = (u64)value; break;
        default: return fail(h, BPE_ERR_ARG, "unknown option");
    }
    return BPE_OK;
}

extern "C" int bpe_get_timing(bpe_handle *h, bpe_timing *out) {
    if (!h || !out) return BPE_ERR_ARG;
    *out = h->tm;
    return BPE_OK;
}

// ------------------------------------------------------------------------------------------------
// stream buffers
static int ensure_stream_capacity(bpe_handle *h, u64 n) {
    // round up to whole tiles (+ slack) so 16-byte loads at the tail stay inside the allocation
    const u64 need = ((n + MG_TILE - 1) / MG_TILE + 1) * MG_TILE;
    int rc;
    if (need > h->buf[0].cap || need > h->buf[1].cap) {
        // make room first: the splitter's slab and both old buffers go before the new ones are allocated
        h->split_slab.reset(); h->buf[0].reset(); h->buf[1].reset();
        if ((rc = dev_reserve(h, h->buf[0], need)) || (rc = dev_reserve(h, h->buf[1], need))) return rc;
    }
    const u64 tiles = need / MG_TILE + 1;
    if (tiles > h->desc.cap) {
        if ((rc = dev_reserve(h, h->desc, tiles))) return rc;
        CU(cudaMemsetAsync(h->desc, 0, tiles * 8, h->stream));
    }
    const u64 segs = need / SEG_TOKENS + 1;
    if (segs > h->edge[0].cap || segs > h->edge[1].cap || segs > h->seg_offs.cap) {
        h->edge[0].reset(); h->edge[1].reset(); h->seg_offs.reset();
        if ((rc = dev_reserve(h, h->edge[0], segs)) || (rc = dev_reserve(h, h->edge[1], segs)) || (rc = dev_reserve(h, h->seg_offs, segs)))
            return rc;
    }
    return BPE_OK;
}

// edge records for a stream that was just written contiguously into the current buffer
static int build_edges(bpe_handle *h, u64 n) {
    const u64 nseg = (n + SEG_TOKENS - 1) / SEG_TOKENS;
    k_build_edges<<<grid_for(nseg, 256, h->sms * 4), 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], 0);
    CU(cudaGetLastError());
    return BPE_OK;
}

// pack the segmented stream back into full segments (other ping-pong buffer becomes current)
static void enqueue_pack(bpe_handle *h, int force) {
    k_scan_counts<<<1, 1024, 0, h->stream>>>(h->ctl, h->edge[0], h->edge[1], h->seg_offs, force);
    k_gather<<<h->sms * 8, 256, 0, h->stream>>>(h->ctl, h->buf[0], h->buf[1], h->edge[0], h->edge[1], h->seg_offs, nullptr, force, 1);
    h->tm.kernel_launches += 2;
}
static void enqueue_edges_after_contig(bpe_handle *h) {
    k_build_edges<<<h->sms * 4, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], 1);
    h->tm.kernel_launches += 1;
}

// entry base of every segment of a weighted stream (k_weighted.cuh); force = 0: only if the stream was just packed
static void enqueue_wt_bases(bpe_handle *h, int force) {
    k_wt_marks<<<h->sms * 8, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->wt_cnt, force);
    k_wt_scan<<<1, 1024, 0, h->stream>>>(h->ctl, h->wt_cnt, h->wt_base, force);
    h->tm.kernel_launches += 2;
}

static int push_ctl(bpe_handle *h) {
    CU(cudaMemcpyAsync(h->ctl, h->h_ctl, sizeof(Ctl), cudaMemcpyHostToDevice, h->stream));
    return BPE_OK;
}
static int pull_ctl(bpe_handle *h) {
    CU(cudaMemcpyAsync(h->h_ctl, h->ctl, sizeof(Ctl), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return BPE_OK;
}

static int reset_ctl_for_stream(bpe_handle *h, u64 n) {
    int rc = pull_ctl(h);  // keep the epoch counter monotonic
    if (rc) return rc;
    const u32 epoch = h->h_ctl->epoch ? h->h_ctl->epoch : 1;
    memset(h->h_ctl, 0, sizeof(Ctl));
    h->h_ctl->epoch = epoch;
    h->h_ctl->n = n;
    h->h_ctl->found_pos = POS_NONE;
    h->h_ctl->first_idx = 256;
    return push_ctl(h);
}

static int check_offsets(bpe_handle *h, const uint64_t *offs, uint64_t k, uint64_t n) {
    if (!offs || k == 0) return BPE_OK;
    if (offs[0] != 0) return fail(h, BPE_ERR_ARG, "chunk_offsets[0] must be 0");
    for (u64 i = 1; i < k; ++i)
        if (offs[i] <= offs[i - 1] || offs[i] >= n) return fail(h, BPE_ERR_ARG, "chunk_offsets must be strictly increasing and < n");
    return BPE_OK;
}

// upload chunk offsets piecewise and mark the chunk starts in buf[0]
static int mark_chunks(bpe_handle *h, u32 *dst, const uint64_t *offs, uint64_t k, uint64_t n) {
    u64 zero = 0;
    if (!offs || k == 0) { offs = &zero; k = n ? 1 : 0; }
    if (k == 0) return BPE_OK;
    const u64 piece = 1ull << 24;  // 16M offsets = 128 MB per piece
    DevBuf<u64> d_offs;
    int rc = dev_reserve(h, d_offs, std::min(piece, k));
    if (rc) return rc;
    for (u64 s = 0; s < k; s += piece) {
        const u64 m = std::min(piece, k - s);
        CU(cudaMemcpyAsync(d_offs, offs + s, m * 8, cudaMemcpyHostToDevice, h->stream));
        k_set_flags<<<grid_for(m, 256, h->sms * 8), 256, 0, h->stream>>>(dst, d_offs, m, n);
        CU(cudaStreamSynchronize(h->stream));
        h->tm.h2d_bytes += m * 8;
    }
    return BPE_OK;
}

static int load_bytes_into(bpe_handle *h, u32 *dst, const uint8_t *bytes, uint64_t n, const unsigned char *d_perm) {
    const u64 piece = 1ull << 28;  // 256 MiB of text per staging copy
    if (n == 0) return BPE_OK;
    DevBuf<unsigned char> d_bytes;
    int rc = dev_reserve(h, d_bytes, std::min(piece, n));
    if (rc) return rc;
    for (u64 s = 0; s < n; s += piece) {
        const u64 m = std::min(piece, n - s);
        CU(cudaMemcpyAsync(d_bytes, bytes + s, m, cudaMemcpyHostToDevice, h->stream));
        k_widen_bytes<<<grid_for(m / 16 + 1, 256, h->sms * 8), 256, 0, h->stream>>>(d_bytes, dst + s, m, d_perm);
        CU(cudaStreamSynchronize(h->stream));
        h->tm.h2d_bytes += m;
    }
    return BPE_OK;
}

extern "C" int bpe_load_stream(bpe_handle *h, const uint8_t *bytes, uint64_t n, const uint64_t *chunk_offsets,
                               uint64_t n_chunks) {
    if (!h) return BPE_ERR_ARG;
    if (!bytes && n) return fail(h, BPE_ERR_ARG, "bytes is NULL");
    if (n >= (1ull << 36)) return fail(h, BPE_ERR_ARG, "stream too long (limit 2^36 tokens)");
    CU(cudaSetDevice(h->device));
    int rc = check_offsets(h, chunk_offsets, n_chunks, n);
    if (rc) return rc;
    h->tm.h2d_bytes = 0;
    h->loaded = false; h->table_valid = false; h->weighted = false;
    if ((rc = ensure_stream_capacity(h, n))) return rc;
    if ((rc = load_bytes_into(h, h->buf[0], bytes, n, nullptr))) return rc;
    if ((rc = mark_chunks(h, h->buf[0], chunk_offsets, n_chunks, n))) return rc;
    if ((rc = reset_ctl_for_stream(h, n))) return rc;
    if ((rc = build_edges(h, n))) return rc;
    h->loaded = true; h->bytes_only = true; h->max_id = 255;
    return BPE_OK;
}

extern "C" int bpe_load_ids(bpe_handle *h, const int32_t *ids, uint64_t n, const uint64_t *chunk_offsets,
                            uint64_t n_chunks) {
    if (!h) return BPE_ERR_ARG;
    if (!ids && n) return fail(h, BPE_ERR_ARG, "ids is NULL");
    if (n >= (1ull << 36)) return fail(h, BPE_ERR_ARG, "stream too long (limit 2^36 tokens)");
    CU(cudaSetDevice(h->device));
    int rc = check_offsets(h, chunk_offsets, n_chunks, n);
    if (rc) return rc;
    h->tm.h2d_bytes = 0;
    h->loaded = false; h->table_valid = false; h->weighted = false;
    if ((rc = ensure_stream_capacity(h, n))) return rc;
    h->max_id = 0;
    if (n) {
        // stage through buf[1] (same size), then convert into buf[0]
        CU(cudaMemcpyAsync(h->buf[1], ids, n * 4, cudaMemcpyHostToDevice, h->stream));
        CU(cudaMemsetAsync(h->d_err, 0, 8, h->stream));
        k_copy_ids<<<grid_for(n, 256, h->sms * 8), 256, 0, h->stream>>>((const int *)h->buf[1].p, h->buf[0], n, h->d_err);
        u32 bad[2] = {0, 0};
        CU(cudaMemcpyAsync(bad, h->d_err, 8, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        if (bad[0]) return fail(h, BPE_ERR_ARG, "ids must be in [0, 2^31-1)");
        h->max_id = bad[1];
        h->tm.h2d_bytes += n * 4;
    }
    if ((rc = mark_chunks(h, h->buf[0], chunk_offsets, n_chunks, n))) return rc;
    if ((rc = reset_ctl_for_stream(h, n))) return rc;
    if ((rc = build_edges(h, n))) return rc;
    h->loaded = true; h->bytes_only = false;
    return BPE_OK;
}

extern "C" int bpe_stream_len(bpe_handle *h, uint64_t *n) {
    if (!h || !n) return BPE_ERR_ARG;
    if (!h->loaded) return fail(h, BPE_ERR_STATE, "no stream loaded");
    CU(cudaSetDevice(h->device));
    int rc = pull_ctl(h);
    if (rc) return rc;
    *n = h->h_ctl->n;
    return BPE_OK;
}

extern "C" int bpe_read_stream(bpe_handle *h, int32_t *out, uint64_t cap, uint64_t *n) {
    if (!h || !n) return BPE_ERR_ARG;
    if (!h->loaded) return fail(h, BPE_ERR_STATE, "no stream loaded");
    CU(cudaSetDevice(h->device));
    int rc = pull_ctl(h);
    if (rc) return rc;
    const u64 len = h->h_ctl->n;
    *n = len;
    if (cap < len) return fail(h, BPE_ERR_CAPACITY, "output buffer too small");
    if (len == 0) return BPE_OK;
    if (!out) return fail(h, BPE_ERR_ARG, "out is NULL");
    const u32 cur = h->h_ctl->cur;
    // pack the segments into the idle ping-pong buffer (the stream itself stays as it is), strip
    // the chunk marks there, copy out
    k_scan_counts<<<1, 1024, 0, h->stream>>>(h->ctl, h->edge[0], h->edge[1], h->seg_offs, 1);
    k_gather<<<h->sms * 8, 256, 0, h->stream>>>(h->ctl, h->buf[0], h->buf[1], h->edge[0], h->edge[1], h->seg_offs,
                                                 h->buf[cur ^ 1], 1, 0);
    k_strip_flags<<<grid_for(len, 256, h->sms * 8), 256, 0, h->stream>>>(h->buf[cur ^ 1], (int *)h->buf[cur ^ 1].p, len);
    CU(cudaMemcpyAsync(out, h->buf[cur ^ 1], len * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->tm.d2h_bytes = len * 4;
    return BPE_OK;
}

// ------------------------------------------------------------------------------------------------
// weighted stream (k_weighted.cuh): entries = chunk occurrences in text order, each standing for `weight` occurrences
// storage of a weighted stream of n_entries entries over the stream just loaded (its segments: h->seg_offs.cap)
static int wt_alloc(bpe_handle *h, u64 n_entries) {
    int rc = dev_reserve(h, h->wts, n_entries);
    if (!rc) rc = dev_reserve(h, h->wt_cnt, h->seg_offs.cap);
    return rc ? rc : dev_reserve(h, h->wt_base, h->seg_offs.cap);
}
// the weights are in h->wts: entry bases, and the handle holds a weighted stream
static int wt_finish(bpe_handle *h, u64 n_entries) {
    enqueue_wt_bases(h, 1);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(h->stream));
    h->n_entries = n_entries;
    h->weighted = true; h->loaded = true; h->wt_fresh = true;
    return BPE_OK;
}

// the arguments of bpe_load_chunks_weighted / bpe_load_chunks_weighted_dedup: a non-empty text tiled by its chunks, a weight
// >= 1 per chunk, then the checks of bpe_load_stream; *wsum = the sum of the weights
static int check_weighted(bpe_handle *h, const char *who, const uint8_t *bytes, u64 n, const uint64_t *chunk_offsets,
                          u64 n_chunks, const uint64_t *weights, u64 *wsum) {
    if (n && (!chunk_offsets || !n_chunks)) return fail(h, BPE_ERR_ARG, std::string(who) + ": a non-empty text needs chunk offsets");
    if (!n && n_chunks) return fail(h, BPE_ERR_ARG, std::string(who) + ": chunks of an empty text");
    if (n_chunks && !weights) return fail(h, BPE_ERR_ARG, "weights is NULL");
    *wsum = 0;
    for (u64 i = 0; i < n_chunks; ++i) {
        if (weights[i] == 0) return fail(h, BPE_ERR_ARG, "weights must be >= 1");
        *wsum += weights[i];
    }
    if (!bytes && n) return fail(h, BPE_ERR_ARG, "bytes is NULL");
    if (n >= (1ull << 36)) return fail(h, BPE_ERR_ARG, "stream too long (limit 2^36 tokens)");
    return check_offsets(h, chunk_offsets, n_chunks, n);
}

extern "C" int bpe_load_chunks_weighted(bpe_handle *h, const uint8_t *bytes, uint64_t n, const uint64_t *chunk_offsets,
                                        uint64_t n_chunks, const uint64_t *weights) {
    if (!h) return BPE_ERR_ARG;
    u64 wsum = 0;
    int rc = check_weighted(h, "bpe_load_chunks_weighted", bytes, n, chunk_offsets, n_chunks, weights, &wsum);
    if (rc || (rc = bpe_load_stream(h, bytes, n, chunk_offsets, n_chunks))) return rc;   // leaves an unweighted stream
    h->loaded = false;
    if ((rc = wt_alloc(h, n_chunks))) return rc;
    if (n_chunks) CU(cudaMemcpyAsync(h->wts, weights, n_chunks * 8, cudaMemcpyHostToDevice, h->stream));
    h->tm.h2d_bytes += n_chunks * 8;
    return wt_finish(h, n_chunks);   // synchronises: `weights` is the caller's buffer
}

extern "C" int bpe_read_chunk_weights(bpe_handle *h, uint64_t *out, uint64_t cap, uint64_t *n) {
    if (!h || !n) return BPE_ERR_ARG;
    if (!h->loaded) return fail(h, BPE_ERR_STATE, "no stream loaded");
    if (!h->weighted) return fail(h, BPE_ERR_STATE, "bpe_read_chunk_weights: the loaded stream is not weighted");
    *n = h->n_entries;
    if (cap < h->n_entries) return fail(h, BPE_ERR_CAPACITY, "output buffer too small");
    if (!h->n_entries) return BPE_OK;
    if (!out) return fail(h, BPE_ERR_ARG, "out is NULL");
    CU(cudaSetDevice(h->device));
    CU(cudaMemcpyAsync(out, h->wts, h->n_entries * 8, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->tm.d2h_bytes = h->n_entries * 8;
    return BPE_OK;
}

// the sharded loop (step_host.inl) has no weighted form
static int refuse_weighted(bpe_handle *h, const char *what) {
    return h->weighted ? fail(h, BPE_ERR_STATE, std::string(what) + ": not available on a weighted stream (bpe_load_chunks_weighted)")
                       : BPE_OK;
}

// ------------------------------------------------------------------------------------------------
// get_stats (base.py:13-22)
extern "C" int bpe_get_stats(bpe_handle *h, int32_t *pairs, int64_t *counts, uint64_t cap, uint64_t *n_pairs) {
    if (!h || !n_pairs) return BPE_ERR_ARG;
    if (!h->loaded) return fail(h, BPE_ERR_STATE, "no stream loaded");
    if (h->weighted) return fail(h, BPE_ERR_STATE, "bpe_get_stats: not available on a weighted stream (bpe_load_chunks_weighted)");
    CU(cudaSetDevice(h->device));
    int rc = pull_ctl(h);
    if (rc) return rc;
    const u64 n = h->h_ctl->n;
    // distinct pairs <= n - 1; keep the load factor <= 0.5
    const u64 tcap = next_pow2(std::max<u64>(1024, 2 * n));
    PairTable t;
    if ((rc = table_reset(h, t, tcap, true))) return rc;
    const u64 used_before = h->h_ctl->table_used;
    {   // the scratch table counts its own occupancy (k_hist_hash refuses inserts near a full table)
        const ull zero = 0;
        CU(cudaMemcpyAsync(&h->ctl->table_used, &zero, 8, cudaMemcpyHostToDevice, h->stream));
    }
    k_hist_hash<<<h->sms * 8, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], t, 0);
    std::vector<u64> keys(tcap), cnt(tcap), first(tcap);
    CU(cudaMemcpyAsync(keys.data(), t.keys, tcap * 8, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(cnt.data(), t.counts, tcap * 8, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(first.data(), t.first, tcap * 8, cudaMemcpyDeviceToHost, h->stream));
    // k_hist_hash bumped ctl->table_used for the scratch table: restore it
    h->h_ctl->table_used = used_before;
    CU(cudaMemcpyAsync(&h->ctl->table_used, &h->h_ctl->table_used, 8, cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    std::vector<u64> order;
    for (u64 i = 0; i < tcap; ++i) if (keys[i] != KEY_EMPTY) order.push_back(i);
    std::sort(order.begin(), order.end(), [&](u64 x, u64 y) { return first[x] < first[y]; });
    *n_pairs = order.size();
    h->tm.d2h_bytes = tcap * 24;
    if (order.size() > cap) return fail(h, BPE_ERR_CAPACITY, "pairs/counts buffers too small");
    for (u64 i = 0; i < order.size(); ++i) {
        pairs[2 * i] = (int32_t)(keys[order[i]] >> 32);
        pairs[2 * i + 1] = (int32_t)(keys[order[i]] & 0xffffffffu);
        counts[i] = (int64_t)cnt[order[i]];
    }
    return BPE_OK;
}

// ------------------------------------------------------------------------------------------------
// merge (base.py:25-41), single step
// One merge over the stream.  Pairs a != b: the segmented in-place pass.  Pairs (a,a) need the
// run-parity carry along the stream, so they pack the stream and use the contiguous kernel
// (which also refills every segment).  Every kernel gates itself on the device-resident pair, so
// the whole sequence is enqueued unconditionally; `same` >= 0 lets the host skip the no-ops when
// it knows the pair (single-step API).
// `batched`: the pass applies the members k_select_batch chose (bpe_train's loop only; a pair (a,a) is never batched).
// Weighted stream (k_weighted.cuh): the weighted delta is computed by a pass of its own in front of the merge, which then
// runs without a delta vector.
static void launch_merge(bpe_handle *h, ull *delta, int force, int same = -1, bool use_xchg = false, bool batched = false) {
    const unsigned char *xbase = use_xchg ? h->xchg : nullptr;
    ull *const wdelta = h->weighted ? delta : nullptr;   // weighted: the delta passes add into it ...
    if (wdelta) delta = nullptr;                          // ... and the merge kernels below are plain merges
    if (same != 1) {
        if (wdelta) {
            k_wt_delta_seg<<<h->sms * 8, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->wt_base,
                                                              h->wts, wdelta, h->V, batched, force);
            h->tm.kernel_launches += 1;
        }
        SegArgs S;
        S.ctl = h->ctl; S.buf0 = h->buf[0]; S.buf1 = h->buf[1]; S.e0 = h->edge[0]; S.e1 = h->edge[1];
        S.delta = delta; S.V = h->V; S.force = force; S.batched = batched; S.xbase = xbase; S.xstride = h->xchg_stride;
        if (h->filt_active) k_merge_seg<true><<<h->merge_grid_seg, MS_THREADS, MS_SMEM_BYTES, h->stream>>>(S);
        else k_merge_seg<false><<<h->merge_grid_seg, MS_THREADS, MS_SMEM_BYTES, h->stream>>>(S);
        h->tm.kernel_launches += 1;
    }
    if (same != 0) {
        MergeArgs A;
        A.ctl = h->ctl; A.buf0 = h->buf[0]; A.buf1 = h->buf[1]; A.desc = h->desc; A.delta = delta; A.V = h->V; A.force = force;
        A.xbase = xbase; A.xstride = h->xchg_stride;
        enqueue_pack(h, force);
        if (h->weighted) {            // gated on the pack having run (ctl->contig), like the edges below
            enqueue_wt_bases(h, 0);
            if (wdelta) {
                const u64 nblk = (h->h_ctl->n + SEG_TOKENS - 1) / SEG_TOKENS;   // host copy: an upper bound of the device's
                k_wt_delta_same<<<grid_for(nblk, 256, h->sms * 8), 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->wt_base,
                                                                                       h->wts, wdelta, h->V, force);
                h->tm.kernel_launches += 1;
            }
        }
        k_merge<true><<<h->merge_grid_same, MG_THREADS, 0, h->stream>>>(A);
        h->tm.kernel_launches += 1;
        if (h->weighted) enqueue_wt_bases(h, 0);
        enqueue_edges_after_contig(h);
        if (h->filt_active) {      // the pack moved tokens between segments: signatures from the tokens again (gated on a == b)
            k_sig_build<<<h->sms * 8, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->sig, 1);
            h->tm.kernel_launches += 1;
        }
    }
}

extern "C" int bpe_merge(bpe_handle *h, int32_t a, int32_t b, int32_t idx, uint64_t *new_len) {
    if (!h) return BPE_ERR_ARG;
    if (!h->loaded) return fail(h, BPE_ERR_STATE, "no stream loaded");
    if (h->weighted) return fail(h, BPE_ERR_STATE, "bpe_merge: not available on a weighted stream (bpe_load_chunks_weighted)");
    if (a < 0 || b < 0 || idx < 0 || a == 0x7fffffff || b == 0x7fffffff || idx == 0x7fffffff)
        return fail(h, BPE_ERR_ARG, "ids must be in [0, 2^31-1)");
    CU(cudaSetDevice(h->device));
    int rc = pull_ctl(h);
    if (rc) return rc;
    h->h_ctl->a = a; h->h_ctl->b = b; h->h_ctl->z = idx;
    if ((rc = push_ctl(h))) return rc;
    launch_merge(h, nullptr, 1, a == b ? 1 : 0);
    CU(cudaGetLastError());
    if ((rc = pull_ctl(h))) return rc;
    h->table_valid = false;
    if (idx > 255) h->bytes_only = false;
    h->max_id = std::max(h->max_id, (u32)idx);
    if (new_len) *new_len = h->h_ctl->n;
    return BPE_OK;
}

// ------------------------------------------------------------------------------------------------
// training loop (basic.py:31-45 / regex.py:49-66)
// The table starts small (the arg-max scans every slot each iteration) and doubles on demand:
// k_apply_delta stops inserting at ctl->table_limit and raises ctl->overflow (handle_overflow).
static u64 auto_table_cap(bpe_handle *h, u64 n_unbounded_inserts) {
    if (h->opt_table_log2) return 1ull << h->opt_table_log2;
    u64 c = 1ull << 17;   // a byte stream has at most 65536 distinct pairs
    while (c < 2 * n_unbounded_inserts + 2) c <<= 1;
    return c;
}
#define TABLE_MAX_LOAD 0.6

// The owned delta vectors (`vecs` of them, one per member of a batched pass) must cover vocabulary capacity V; h->V
// (the layout every kernel indexes with) is set to exactly V.  The capacity of the owned buffer is tracked separately:
// the step API points the kernels at a caller's buffer and changes h->V without touching h->delta.
static int ensure_delta(bpe_handle *h, u32 V, u32 vecs = 1) {
    bool fresh = false;
    if (!h->delta || h->delta_cap < V || h->delta_vecs < vecs) {
        h->delta.reset(); h->delta_cap = 0; h->delta_vecs = 0;   // sized for (V, vecs) exactly, also when that is smaller
        int rc = dev_reserve(h, h->delta, (u64)vecs * (2ull * V + 1));
        if (rc) return rc;
        h->delta_cap = V; h->delta_vecs = vecs;
        fresh = true;
    }
    if (fresh || h->V != V)   // new buffer or the layout changes: all zero again
        CU(cudaMemsetAsync(h->delta, 0, (u64)h->delta_vecs * (2ull * h->delta_cap + 1) * 8, h->stream));
    h->V = V;
    return BPE_OK;
}
// the device log of the merges of one run (bpe_train, the step API): a pair and its count per merge
static int ensure_log(bpe_handle *h, int num_merges) {
    const int rc = dev_reserve(h, h->log_pairs, 2ull * num_merges);
    return rc ? rc : dev_reserve(h, h->log_counts, (u64)num_merges);
}
// Batched passes index BATCH_MAX delta vectors with one 32-bit flat index (the merge kernel's shared-memory cache keys,
// 0xffffffff = empty) and allocate them all: vocabularies up to 2^21 ids.
static bool batch_fits(u32 V) { return V <= (1u << 21); }

// Byte-pair histogram of the current (byte) stream into dense_out[65536] (zeroed by the caller).
// k_hist_dense_packed (dense 16-bit counters in 128 KB of shared memory) replaces k_hist_dense (hashed per-block table +
// __match_any_sync folding, 19 ms per GiB).  It was written when no GPU was reachable and has only run on the CPU SIMT
// emulator, so a handle's first histogram of a LARGE stream (>= 8 Mi tokens; smaller ones just take k_hist_dense) runs both
// kernels, timed with events, and compares all 65,536 counters on the device: equal and not slower -> the packed kernel
// from then on; otherwise (or 128 KB of shared memory refused) -> k_hist_dense stays.  bpe_timing.hist_kernel
// reports which one is in use.  (Drop the cross-check once `pytest -m gpu` has passed with hist_kernel == 1 on every GPU model in use.)
#define HIST_DECIDE_MIN_TOKENS (8ull << 20)   /* smaller streams say nothing about speed: they take k_hist_dense, undecided */
static int hist_dense(bpe_handle *h, ull *dense_out) {
    const int grid_old = h->sms * 3;
    if (h->opt_hist_kernel && h->hist_mode != h->opt_hist_kernel) {      // BPE_OPT_HIST_KERNEL: forced (tests)
        if (h->opt_hist_kernel == 1 &&
            cudaFuncSetAttribute(k_hist_dense_packed, cudaFuncAttributeMaxDynamicSharedMemorySize, HP_SMEM_BYTES) != cudaSuccess)
            return fail(h, BPE_ERR_CUDA, "k_hist_dense_packed: 128 KB of shared memory refused");
        h->hist_mode = h->opt_hist_kernel;
    }
    if (h->hist_mode == 0 && h->h_ctl->n >= HIST_DECIDE_MIN_TOKENS) {
        h->hist_mode = 2;
        if (cudaFuncSetAttribute(k_hist_dense_packed, cudaFuncAttributeMaxDynamicSharedMemorySize, HP_SMEM_BYTES) == cudaSuccess) {
            int rc;
            if ((rc = dev_reserve(h, h->dense2, 65536)) || (rc = dev_reserve(h, h->d_cmp, 1))) return rc;
            CU(cudaMemsetAsync(h->dense2, 0, 65536 * 8, h->stream));
            CU(cudaMemsetAsync(h->d_cmp, 0, 4, h->stream));
            Event ev[3];
            for (auto &e : ev) CU(e.create());
            cudaEventRecord(ev[0], h->stream);
            k_hist_dense<<<grid_old, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], dense_out, h->d_err);
            cudaEventRecord(ev[1], h->stream);
            if (cudaGetLastError() != cudaSuccess) return fail(h, BPE_ERR_CUDA, "k_hist_dense launch failed");
            k_hist_dense_packed<<<h->sms, HP_THREADS, HP_SMEM_BYTES, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->dense2, h->d_err);
            cudaEventRecord(ev[2], h->stream);
            if (cudaGetLastError() != cudaSuccess) {      // the launch itself was refused (a launch error is not sticky): keep k_hist_dense
                h->tm.kernel_launches += 1;
                h->tm.hist_kernel = 2;
                return BPE_OK;
            }
            k_dense_compare<<<65536 / 256, 256, 0, h->stream>>>(dense_out, h->dense2, h->d_cmp);
            h->tm.kernel_launches += 3;
            u32 differ = 1;
            cudaError_t e = cudaMemcpyAsync(&differ, h->d_cmp, 4, cudaMemcpyDeviceToHost, h->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
            float ms_old = 0, ms_new = 0;
            if (e == cudaSuccess) { cudaEventElapsedTime(&ms_old, ev[0], ev[1]); cudaEventElapsedTime(&ms_new, ev[1], ev[2]); }
            if (e != cudaSuccess) return fail(h, BPE_ERR_CUDA, std::string("hist_dense: ") + cudaGetErrorString(e));
            // adopted only when it gives the same 65,536 counters AND is not slower on this very stream
            if (!differ && ms_new <= ms_old) h->hist_mode = 1;
            h->tm.hist_kernel = (uint64_t)h->hist_mode;
            return BPE_OK;      // dense_out holds k_hist_dense's result either way
        }
    }
    if (h->hist_mode == 1)
        k_hist_dense_packed<<<h->sms, HP_THREADS, HP_SMEM_BYTES, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], dense_out, h->d_err);
    else
        k_hist_dense<<<grid_old, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], dense_out, h->d_err);
    h->tm.kernel_launches += 1;
    h->tm.hist_kernel = (uint64_t)h->hist_mode;
    return BPE_OK;
}

// (re)build the pair-count table from the current stream
static int build_table(bpe_handle *h, u64 cap) {
    int rc;
    if ((rc = table_reset(h, h->table, cap, false))) return rc;
    const ull zero = 0;
    CU(cudaMemcpyAsync(&h->ctl->table_used, &zero, 8, cudaMemcpyHostToDevice, h->stream));
    if (h->weighted) {      // weighted sums straight into the table; takes no part in the choice of hist_dense
        CU(cudaMemsetAsync(h->d_err, 0, 4, h->stream));
        k_wt_hist<<<h->sms * 8, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->wt_base, h->wts, h->table);
        h->tm.kernel_launches += 1;
    } else if (h->bytes_only) {
        CU(cudaMemsetAsync(h->dense, 0, 65536 * 8, h->stream));
        CU(cudaMemsetAsync(h->d_err, 0, 4, h->stream));
        if ((rc = hist_dense(h, h->dense))) return rc;
        k_dense_to_table<<<65536 / 256, 256, 0, h->stream>>>(h->dense, h->table, h->ctl);
        h->tm.kernel_launches += 1;
    } else {
        k_hist_hash<<<h->sms * 8, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->table, 0);
        h->tm.kernel_launches += 1;
    }
    CU(cudaGetLastError());
    return BPE_OK;
}

// grow / clean the table: live entries are re-inserted into a fresh table of `cap` slots
static int rehash_table(bpe_handle *h, u64 cap) {
    PairTable nt;
    int rc = table_reset(h, nt, cap, false);
    if (rc) return rc;
    const ull zero = 0;
    CU(cudaMemcpyAsync(&h->ctl->table_used, &zero, 8, cudaMemcpyHostToDevice, h->stream));
    k_rehash<<<grid_for(h->table.mask + 1, 256, h->sms * 8), 256, 0, h->stream>>>(h->table, nt, h->ctl);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(h->stream));
    h->table = std::move(nt);
    h->tm.kernel_launches++;
    return BPE_OK;
}

// fold the event pairs recorded since the last call into tm.merge_kernel_ms (stream must be idle)
static void drain_kernel_events(bpe_handle *h) {
    for (int i = 0; i + 1 < h->ev_used; i += 2) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, h->ev_pool[i], h->ev_pool[i + 1]) == cudaSuccess) h->tm.merge_kernel_ms += ms;
    }
    h->ev_used = 0;
}

static void timed_merge(bpe_handle *h, ull *delta, bool use_xchg = false, bool batched = false) {
    if (!h->opt_kernel_timing) { launch_merge(h, delta, 0, -1, use_xchg, batched); return; }
    while ((int)h->ev_pool.size() < h->ev_used + 2) { h->ev_pool.emplace_back(); h->ev_pool.back().create(); }
    cudaEventRecord(h->ev_pool[h->ev_used], h->stream);
    launch_merge(h, delta, 0, -1, use_xchg, batched);
    cudaEventRecord(h->ev_pool[h->ev_used + 1], h->stream);
    h->ev_used += 2;
}

// ctl->overflow was raised by k_apply_delta: some delta entries of the last performed pass are
// still pending.  Double the table (dead pairs are dropped on the way), re-run the apply.  A batched
// pass (nk members) re-runs every member's apply in member order: a member whose apply overflowed
// stopped the ones after it, and re-applying a finished member changes nothing (its delta is zero).
static int handle_overflow(bpe_handle *h, u32 nk = 1) {
    int rc;
    for (u32 j = 0; j < nk; ++j) {
        do {
            if (h->h_ctl->overflow) {
                const u64 new_cap = (h->table.mask + 1) * 2;
                if ((rc = rehash_table(h, new_cap))) return rc;
                if ((rc = pull_ctl(h))) return rc;
                h->h_ctl->overflow = 0;
                h->h_ctl->table_limit = (u64)(TABLE_MAX_LOAD * (double)new_cap);
                if ((rc = push_ctl(h))) return rc;
            }
            k_apply_delta<<<(h->V + 255) / 256, 256, 0, h->stream>>>(h->table, h->ctl, h->delta, h->V, 0, 0, 0, 1, 1, (int)j);
            h->tm.kernel_launches++;
            if ((rc = pull_ctl(h))) return rc;
        } while (h->h_ctl->overflow);
    }
    return BPE_OK;
}

// Between batches: when merges have emptied the segments below half full on average, pack the
// stream into full segments again (fewer, fuller segments = less per-segment overhead).
static void maybe_repack(bpe_handle *h) {
    const u64 nseg = h->h_ctl->nseg;
    if (nseg < 64 || h->h_ctl->contig) return;
    if (2 * h->h_ctl->n >= nseg * (u64)SEG_TOKENS) return;
    enqueue_pack(h, 1);
    if (h->weighted) enqueue_wt_bases(h, 0);
    enqueue_edges_after_contig(h);
    if (h->filt_active) {
        k_sig_build<<<h->sms * 8, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->sig, 0);
        h->tm.kernel_launches += 1;
    }
}

// ---- segment filter (k_seg_filter.cuh) ---------------------------------------------------------------------------
static void filt_rebuild(bpe_handle *h, int gate_same) {
    k_sig_build<<<h->sms * 8, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->sig, gate_same);
    h->tm.kernel_launches += 1;
}

// switch the filter on for the iterations enqueued from here on: storage, list address in the control block, signatures
// of the stream as it is now
static int filt_activate(bpe_handle *h) {
    const u64 want = (u64)h->h_ctl->nseg + 64;      // segments of the stream as it is now (the count only ever falls), not the buffers' capacity
    int rc;
    if ((rc = dev_reserve(h, h->sig, want * SIG_WORDS)) || (rc = dev_reserve(h, h->cand, want))) return rc;
    const u64 ptr = (u64)(uintptr_t)h->cand.p;
    const u32 zero = 0;
    CU(cudaMemcpyAsync(&h->ctl->cand_ptr, &ptr, 8, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(&h->ctl->n_cand, &zero, 4, cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));          // `ptr` / `zero` are stack variables
    h->h_ctl->cand_ptr = ptr; h->h_ctl->n_cand = 0;
    filt_rebuild(h, 0);
    h->filt_active = true;
    return BPE_OK;
}

static void enqueue_iteration(bpe_handle *h) {
    if (h->opt_rescan) {
        // verification mode: rebuild the histogram from the stream, no incremental update
        cudaMemsetAsync(h->table.keys, 0xff, (h->table.mask + 1) * 8, h->stream);
        cudaMemsetAsync(h->table.counts, 0, (h->table.mask + 1) * 8, h->stream);
        cudaMemsetAsync(&h->ctl->table_used, 0, 8, h->stream);
        k_hist_hash<<<h->sms * 4, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->ctl, h->edge[0], h->edge[1], h->table, 1);
        h->tm.kernel_launches++;
    }
    if (h->filt_active) { k_cand_reset<<<1, 1, 0, h->stream>>>(h->ctl); h->tm.kernel_launches++; }
    k_argmax<<<h->argmax_grid, 256, 0, h->stream>>>(h->table, h->ctl, h->partials, h->log_pairs, h->log_counts);
    k_find_first<<<h->ff_grid, 256, 0, h->stream>>>(h->buf[0], h->buf[1], h->edge[0], h->edge[1], h->table, h->ctl, h->log_pairs, h->log_counts, 0);
    h->tm.kernel_launches += 2;
    // several provably determined merges in one pass; not with the rescan mode (no delta) or the segment filter (its
    // candidate list is the one pair's)
    const bool batched = h->batching && !h->opt_rescan && !h->filt_active;
    if (batched) {
        k_select_batch<<<h->argmax_grid, 256, 0, h->stream>>>(h->table, h->ctl, h->top_partials, h->log_pairs, h->log_counts);
        h->tm.kernel_launches++;
    }
    if (h->filt_active) {    // candidate segments of the selected pair; k_merge_seg<true> works through that list only
        k_seg_filter<<<h->sms * 8, 256, 0, h->stream>>>(h->ctl, h->edge[0], h->edge[1], h->edge[0], h->edge[1], h->sig, h->cand);
        h->tm.kernel_launches++;
    }
    if (h->opt_rescan) timed_merge(h, nullptr);
    else {
        timed_merge(h, h->delta, false, batched);
        for (int j = 0; j < (batched ? BATCH_MAX : 1); ++j)   // member order: each apply may need the pairs the one before inserted
            k_apply_delta<<<(h->V + 255) / 256, 256, 0, h->stream>>>(h->table, h->ctl, h->delta, h->V, 0, 0, 0, 1, 0, j);
        h->tm.kernel_launches += batched ? BATCH_MAX : 1;
    }
    if (h->filt_active) {    // the listed segments may have changed: their signatures from their tokens again
        k_sig_rebuild_cand<<<h->sms * 4, 256, 0, h->stream>>>(h->ctl, h->buf[0], h->buf[1], h->edge[0], h->edge[1], h->sig, h->cand);
        h->tm.kernel_launches++;
    }
}

extern "C" int bpe_train(bpe_handle *h, int32_t num_merges, int32_t first_idx, int32_t *out_pairs, int64_t *out_counts,
                         int32_t *n_done) {
    if (!h || !n_done) return BPE_ERR_ARG;
    if (!h->loaded) return fail(h, BPE_ERR_STATE, "no stream loaded");
    if (num_merges < 0 || first_idx < 0) return fail(h, BPE_ERR_ARG, "num_merges and first_idx must be >= 0");
    if ((u64)first_idx + (u64)num_merges >= 0x7fffffffull) return fail(h, BPE_ERR_ARG, "vocabulary would exceed 2^31-1");
    if (num_merges && (!out_pairs || !out_counts)) return fail(h, BPE_ERR_ARG, "output buffers are NULL");
    if (h->weighted && (h->opt_rescan || h->opt_seg_filter))
        return fail(h, BPE_ERR_STATE, "bpe_train: BPE_OPT_RESCAN and BPE_OPT_SEG_FILTER are not available on a weighted stream");
    h->wt_fresh = false;
    CU(cudaSetDevice(h->device));
    *n_done = 0;
    h->tm.kernel_launches = 0; h->tm.d2h_bytes = 0; h->tm.merge_kernel_ms = 0;
    if (num_merges == 0) return BPE_OK;
    int rc = pull_ctl(h);
    if (rc) return rc;
    // the delta vector is indexed by the ids of a merge's neighbours: it must cover every id of the loaded
    // stream (bpe_load_ids accepts any id < 2^31-1) as well as the ids this call creates
    if ((u64)h->max_id + 1 >= 0x7fffffffull / 2) return fail(h, BPE_ERR_ARG, "bpe_train: ids of the loaded stream are too large for the dense delta vector");
    const u32 V = std::max(std::max((u32)first_idx + (u32)num_merges, h->max_id + 1), h->opt_vocab_cap);
    h->batching = !h->opt_rescan && batch_fits(V);
    if ((rc = ensure_delta(h, V, h->batching ? BATCH_MAX : 1)) || (rc = ensure_log(h, num_merges))) return rc;
    Event ev0, ev1, ev2;
    CU(ev0.create()); CU(ev1.create()); CU(ev2.create());

    // ---- initial statistics (the only full histogram of the run) ----
    CU(cudaEventRecord(ev0, h->stream));
    // only a non-byte stream (bpe_load_ids) or the rescan mode insert without the load check
    u64 cap = auto_table_cap(h, !h->bytes_only ? h->h_ctl->n : 0);
    if (h->opt_rescan && !h->opt_table_log2) {   // every iteration clears and rescans: keep the table moderate
        cap = 1ull << 20;
        while (cap < h->h_ctl->n / 16 && cap < (1ull << 26)) cap <<= 1;
    }
    const bool reuse = h->table_valid && h->table.keys && !h->opt_rescan;  // continuing a previous bpe_train
    if (!reuse && (rc = build_table(h, cap))) return rc;
    h->table_valid = false;  // becomes true again when the loop ends cleanly
    u32 bad = 0;
    if (!reuse && h->bytes_only) CU(cudaMemcpyAsync(&bad, h->d_err, 4, cudaMemcpyDeviceToHost, h->stream));
    if ((rc = pull_ctl(h))) return rc;  // refreshes table_used
    if (bad) return fail(h, BPE_ERR_INTERNAL, "byte stream contains ids >= 256");
    h->h_ctl->iter = 0; h->h_ctl->done = 0; h->h_ctl->first_idx = (u32)first_idx; h->h_ctl->max_iter = (u32)num_merges;
    h->h_ctl->sum_in = 0; h->h_ctl->sum_out = 0;
    h->h_ctl->cand_sum = 0; h->h_ctl->seg_sum = 0;
    h->h_ctl->overflow = 0;
    h->h_ctl->table_limit = (u64)(TABLE_MAX_LOAD * (double)(h->table.mask + 1));
    if ((rc = push_ctl(h))) return rc;
    CU(cudaEventRecord(ev1, h->stream));

    // ---- the merge loop: batches of iterations enqueued back to back, one host sync per batch ----
    int done_iters = 0;
    bool exhausted = false;
    h->filt_active = false;
    if (h->opt_seg_filter == 2 && !h->opt_rescan && (rc = filt_activate(h))) return rc;
    u64 drops_seen = 0;
    while (done_iters < num_merges && !exhausted) {
        const int k = std::min(h->opt_batch, num_merges - done_iters);
        maybe_repack(h);
        for (int i = 0; i < k; ++i) enqueue_iteration(h);
        CU(cudaGetLastError());
        if ((rc = pull_ctl(h))) return rc;
        drain_kernel_events(h);
        if (h->opt_seg_filter == 1 && !h->filt_active && !h->opt_rescan && (int)h->h_ctl->iter > done_iters) {
            // BPE_OPT_SEG_FILTER = 1: once a merge replaces, on average, fewer tokens than a thirty-second of the segments
            // there are, most segments cannot be touched by it: filter from the next batch on (merges only get sparser)
            const u64 drops = h->h_ctl->sum_in - h->h_ctl->sum_out;
            const u64 per_merge = (drops - drops_seen) / (u64)((int)h->h_ctl->iter - done_iters);
            drops_seen = drops;
            if (per_merge * 32 < h->h_ctl->nseg && (rc = filt_activate(h))) return rc;
        }
        if (h->h_ctl->overflow) {
            if (h->opt_rescan) return fail(h, BPE_ERR_CAPACITY, "rescan mode: pair table too small (set BPE_OPT_TABLE_LOG2)");
            if ((rc = handle_overflow(h, h->h_ctl->nk))) return rc;
        }
        done_iters = (int)h->h_ctl->iter;
        exhausted = h->h_ctl->done != 0;
    }
    CU(cudaEventRecord(ev2, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    float ms01 = 0, ms12 = 0;
    cudaEventElapsedTime(&ms01, ev0, ev1);
    cudaEventElapsedTime(&ms12, ev1, ev2);
    h->tm.init_ms = ms01; h->tm.loop_ms = ms12;
    h->tm.tokens_in = h->h_ctl->sum_in; h->tm.tokens_out = h->h_ctl->sum_out;
    h->tm.table_slots = h->table.mask + 1; h->tm.table_used = h->h_ctl->table_used;
    h->tm.filter_candidates = h->h_ctl->cand_sum; h->tm.filter_segments = h->h_ctl->seg_sum;
    if (done_iters > 0) {
        CU(cudaMemcpyAsync(out_pairs, h->log_pairs, (size_t)done_iters * 8, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaMemcpyAsync(out_counts, h->log_counts, (size_t)done_iters * 8, cudaMemcpyDeviceToHost, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        h->tm.d2h_bytes = (u64)done_iters * 16;
    }
    *n_done = done_iters;
    h->filt_active = false;      // the other users of launch_merge (bpe_merge, replay, the step API) do not maintain signatures
    h->table_valid = !h->opt_rescan;
    if (first_idx + done_iters > 256) h->bytes_only = false;
    if (done_iters > 0) h->max_id = std::max(h->max_id, (u32)(first_idx + done_iters - 1));
    return BPE_OK;
}

// debug/test hook: dump the live entries (count > 0) of the incremental table, unordered
extern "C" int bpe_debug_table(bpe_handle *h, int32_t *pairs, int64_t *counts, uint64_t cap, uint64_t *n_pairs) {
    if (!h || !n_pairs) return BPE_ERR_ARG;
    if (!h->table.keys) return fail(h, BPE_ERR_STATE, "no table");
    CU(cudaSetDevice(h->device));
    const u64 tcap = h->table.mask + 1;
    std::vector<u64> keys(tcap), cnt(tcap);
    CU(cudaMemcpyAsync(keys.data(), h->table.keys, tcap * 8, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaMemcpyAsync(cnt.data(), h->table.counts, tcap * 8, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    u64 m = 0;
    for (u64 i = 0; i < tcap; ++i) {
        if (keys[i] == KEY_EMPTY || cnt[i] == 0) continue;
        if (m < cap) { pairs[2 * m] = (int32_t)(keys[i] >> 32); pairs[2 * m + 1] = (int32_t)(keys[i] & 0xffffffffu); counts[m] = (int64_t)cnt[i]; }
        ++m;
    }
    *n_pairs = m;
    return m > cap ? fail(h, BPE_ERR_CAPACITY, "buffers too small") : BPE_OK;
}

#include "encode_host.inl"
#include "step_host.inl"
#include "special_host.inl"
#include "split_host.inl"
#include "encode2_host.inl"
#include "decode_host.inl"
#include "dedup_host.inl"

bpe_handle::~bpe_handle() {   // the members free the device buffers, events and sub-states
    if (h_ctl) cudaFreeHost(h_ctl);
    if (own_stream) cudaStreamDestroy(own_stream);
}
