// tests/emu/cuda_emu.cpp — TEST INFRASTRUCTURE: scheduler, guarded allocator and runtime stubs of the CPU SIMT
// emulator described in cuda_emu.h.
#include "cuda_emu.h"

#include <stdio.h>
#include <sys/mman.h>
#include <time.h>
#include <unistd.h>

#include <atomic>
#include <condition_variable>
#include <map>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#if !defined(__x86_64__)
#error "the fiber switch below is written for x86-64 (System V ABI)"
#endif

// ---- fiber switch: callee-saved registers + stack pointer ---------------------------------------------------------
extern "C" void emu_switch(void **save_sp, void *load_sp);
asm(R"(
.text
.globl emu_switch
.type emu_switch,@function
emu_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size emu_switch,.-emu_switch
)");

namespace emu {

enum { F_RUN, F_WAIT_BAR, F_WAIT_WARP, F_SPIN, F_DONE };
static const size_t STACK_BYTES = 192 * 1024;
static const unsigned MAX_THREADS = 1024;

// one rendezvous of a warp: what its first lane brought (kind, mask, call site), who has arrived, their values
struct WarpSlot {
    uint32_t gen, arrived; uint64_t val[32];
    int kind; uint32_t mask, first; const char *file; int line;
};
struct Warp { WarpSlot slot[2]; uint32_t alive; };

struct Fiber {
    void *sp;
    int state;
    uint32_t bar_gen;       // barrier generation this fiber waits to pass
    uint32_t coll_seq;      // collectives executed so far by this lane
    WarpSlot *wslot; uint32_t wmask; uint32_t wgen;   // what a F_WAIT_WARP fiber waits for
    uint32_t lane, warp;
    ThreadCtx ctx;
};

struct Sched {
    char *stacks = nullptr;            // MAX_THREADS stacks, mapped once per OS thread
    Fiber fib[MAX_THREADS];
    Warp warps[MAX_THREADS / 32];
    void *main_sp = nullptr;
    Fiber *cur = nullptr;
    unsigned nthreads = 0, alive = 0;
    uint32_t bar_gen = 1, bar_arrived = 0;
    const std::function<void()> *body = nullptr;
    void *dyn = nullptr; size_t dyn_cap = 0;
    unsigned long long spins = 0;
    bool in_kernel = false;
    const char *kernel = nullptr;      // name of the running kernel (reports)
    dim3 bid;                          // the running block
};
static thread_local Sched *tl = nullptr;

static Sched *sched() {
    if (!tl) {
        tl = new Sched();
        tl->stacks = (char *)mmap(nullptr, STACK_BYTES * MAX_THREADS, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (tl->stacks == MAP_FAILED) { perror("emu: mmap stacks"); abort(); }
    }
    return tl;
}

ThreadCtx *ctx() { return &tl->cur->ctx; }
void *dyn_smem() { return tl->dyn; }

long long clock() {
    timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
    return (long long)ts.tv_sec * 2000000000ll + (long long)ts.tv_nsec * 2;   // a 2 GHz "SM clock"
}

static void to_main() { Sched *s = tl; emu_switch(&s->cur->sp, s->main_sp); }

static void release_barrier_if_complete(Sched *s) {
    if (s->alive && s->bar_arrived == s->alive) { s->bar_arrived = 0; s->bar_gen++; }
}

static void fiber_entry() {
    Sched *s = tl;
    Fiber *f = s->cur;
    (*s->body)();
    f->state = F_DONE;
    s->alive--;
    s->warps[f->warp].alive &= ~(1u << f->lane);
    release_barrier_if_complete(s);   // the threads still at the barrier no longer wait for this one
    to_main();
    fprintf(stderr, "emu: a finished fiber was resumed\n");
    abort();
}

void sync_threads() {
    Sched *s = tl;
    Fiber *f = s->cur;
    f->bar_gen = s->bar_gen;
    s->bar_arrived++;
    if (s->bar_arrived == s->alive) { s->bar_arrived = 0; s->bar_gen++; return; }   // last one in: nobody waits
    f->state = F_WAIT_BAR;
    to_main();
}

static inline bool slot_ready(const Sched *s, const Fiber *f) {
    const uint32_t need = f->wmask & s->warps[f->warp].alive;
    return f->wslot->gen == f->wgen && (f->wslot->arrived & need) == need;
}

static const char *kind_name(int kind) {
    static const char *const names[] = {"__shfl_sync", "__shfl_up_sync", "__shfl_down_sync", "__shfl_xor_sync", "__ballot_sync", "__all_sync",
                                        "__any_sync", "__reduce_or_sync", "__reduce_max_sync", "__syncwarp", "__match_any_sync"};
    return kind >= 0 && kind <= C_MATCH ? names[kind] : "?";
}

[[noreturn]] static void warp_rule_broken(const char *what, const Sched *s, const Fiber *f, const WarpSlot &sl, int kind, uint32_t mask,
                                          const char *file, int line) {
    fprintf(stderr, "emu: warp collective rule broken (%s) in kernel %s, block (%u,%u,%u), warp %u:\n"
            "  lane %u is at %s(mask 0x%08x) at %s:%d\n"
            "  lane %u arrived first at %s(mask 0x%08x) at %s:%d\n"
            "  (every live lane named in a collective's mask executes that same call: same site, same kind, same mask)\n",
            what, s->kernel ? s->kernel : "?", s->bid.x, s->bid.y, s->bid.z, f->warp, f->lane, kind_name(kind), mask, file, line, sl.first,
            kind_name(sl.kind), sl.mask, sl.file, sl.line);
    abort();
}

[[noreturn]] void activemask_called(const char *file, int line) {
    const Sched *s = tl;
    const Fiber *f = s && s->cur ? s->cur : nullptr;
    fprintf(stderr, "emu: __activemask() called at %s:%d in kernel %s, warp %u, lane %u: the converged set it returns depends on "
            "scheduling; name the lanes that execute the collective instead\n",
            file, line, s && s->kernel ? s->kernel : "?", f ? f->warp : 0u, f ? f->lane : 0u);
    abort();
}

static const uint64_t POISON = 0xCDCDCDCDCDCDCDCDull;   // what a shuffle reads from a lane that is not taking part (guard fill)

uint64_t collective(int kind, uint32_t mask, uint64_t val, uint32_t arg, const char *file, int line) {
    Sched *s = tl;
    Fiber *f = s->cur;
    Warp &w = s->warps[f->warp];
    const uint32_t k = f->coll_seq++;
    WarpSlot &sl = w.slot[k & 1u];
    if (sl.gen != k + 1) {   // first lane of collective number k: what it brought is what the others must bring
        sl.gen = k + 1; sl.arrived = 0;
        sl.kind = kind; sl.mask = mask; sl.file = file; sl.line = line; sl.first = f->lane;
    }
    if (!((mask >> f->lane) & 1u)) warp_rule_broken("the calling lane is not in its own mask", s, f, sl, kind, mask, file, line);
    if (sl.kind != kind) warp_rule_broken("two kinds of collective meet", s, f, sl, kind, mask, file, line);
    if (sl.mask != mask) warp_rule_broken("two masks meet", s, f, sl, kind, mask, file, line);
    if (sl.line != line || strcmp(sl.file, file) != 0) warp_rule_broken("two call sites meet", s, f, sl, kind, mask, file, line);
    sl.val[f->lane] = val;
    sl.arrived |= 1u << f->lane;
    f->wslot = &sl; f->wmask = mask; f->wgen = k + 1;
    while (!slot_ready(s, f)) { f->state = F_WAIT_WARP; to_main(); }
    const uint32_t in = sl.arrived & mask;    // the lanes taking part: every live lane of the mask
    const uint32_t lane = f->lane;
    auto from = [&](uint32_t src) { return (in >> src) & 1u ? sl.val[src] : POISON; };
    switch (kind) {
        case C_SHFL: return from(arg & 31u);
        case C_UP: return lane >= arg ? from(lane - arg) : val;          // no source lane: the caller's own value (CUDA)
        case C_DOWN: return lane + arg < 32 ? from(lane + arg) : val;
        case C_XOR: return from((lane ^ arg) & 31u);
        case C_BALLOT: { uint32_t b = 0; for (int l = 0; l < 32; ++l) if (((in >> l) & 1u) && sl.val[l]) b |= 1u << l; return b; }
        case C_ALL: { for (int l = 0; l < 32; ++l) if (((in >> l) & 1u) && !sl.val[l]) return 0; return 1; }
        case C_ANY: { for (int l = 0; l < 32; ++l) if (((in >> l) & 1u) && sl.val[l]) return 1; return 0; }
        case C_OR: { uint64_t r = 0; for (int l = 0; l < 32; ++l) if ((in >> l) & 1u) r |= sl.val[l]; return r; }
        case C_MAX: { uint64_t r = 0; for (int l = 0; l < 32; ++l) if (((in >> l) & 1u) && sl.val[l] > r) r = sl.val[l]; return r; }
        case C_MATCH: { uint32_t g = 0; for (int l = 0; l < 32; ++l) if (((in >> l) & 1u) && sl.val[l] == val) g |= 1u << l; return g; }
        default: return 0;
    }
}

// Called by every polling load.  Inside a kernel: let the other fibers of the block run (one of them may be the
// producer); a wait that never ends is reported instead of hanging the test.
void spin() {
    Sched *s = tl;
    if (!s || !s->in_kernel) return;
    if (++s->spins > 400000000ull) { fprintf(stderr, "emu: a kernel polled memory 4e8 times without an end (deadlock)\n"); abort(); }
    if ((s->spins & 63u) == 0) { s->cur->state = F_SPIN; to_main(); }
}

static int order_mode() {
    static int v = -1;
    if (v < 0) { const char *e = getenv("EMU_ORDER"); v = !e ? 0 : (e[0] == 'r' && e[1] == 'e') ? 1 : (e[0] == 'r' && e[1] == 'a') ? 2 : 0; }
    return v;
}

static void run_block(Sched *s, const LaunchCfg &cfg, dim3 bid) {
    const unsigned n = cfg.block.x * cfg.block.y * cfg.block.z;
    s->nthreads = n; s->alive = n; s->bar_gen = 1; s->bar_arrived = 0; s->bid = bid;
    const unsigned nw = (n + 31) / 32;
    for (unsigned w = 0; w < nw; ++w) {
        s->warps[w].slot[0].gen = s->warps[w].slot[1].gen = 0;
        const unsigned lanes = (w + 1) * 32 <= n ? 32 : n - w * 32;
        s->warps[w].alive = lanes == 32 ? 0xffffffffu : ((1u << lanes) - 1u);
    }
    for (unsigned t = 0; t < n; ++t) {
        Fiber &f = s->fib[t];
        f.state = F_RUN; f.bar_gen = 0; f.coll_seq = 0; f.lane = t & 31u; f.warp = t >> 5;
        f.ctx.tid = dim3(t % cfg.block.x, (t / cfg.block.x) % cfg.block.y, t / (cfg.block.x * cfg.block.y));
        f.ctx.bid = bid; f.ctx.bdim = cfg.block; f.ctx.gdim = cfg.grid;
        uintptr_t top = ((uintptr_t)(s->stacks + (size_t)(t + 1) * STACK_BYTES)) & ~(uintptr_t)15;
        void **sp = (void **)top;
        *--sp = nullptr;                  // return address of fiber_entry (never used)
        *--sp = (void *)&fiber_entry;     // `ret` of the first switch jumps here
        for (int r = 0; r < 6; ++r) *--sp = nullptr;   // rbp rbx r12 r13 r14 r15
        f.sp = sp;
    }
    // Order in which the runnable threads of the block get the processor.  CUDA promises none: a kernel whose result
    // depends on it has a data race (a missing __syncthreads / __syncwarp).  EMU_ORDER=reverse | random (default: by
    // thread index) lets the test-suite run under other interleavings.
    static thread_local unsigned order[MAX_THREADS];
    static thread_local unsigned long long rng = 0x9e3779b97f4a7c15ull;
    const int mode = order_mode();
    for (unsigned t = 0; t < n; ++t) order[t] = mode == 1 ? n - 1 - t : t;
    unsigned long long idle_rounds = 0;
    while (s->alive) {
        bool progress = false, spinning = false;
        if (mode == 2)
            for (unsigned t = n - 1; t > 0; --t) {
                rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
                const unsigned j = (unsigned)(rng % (t + 1));
                const unsigned x = order[t]; order[t] = order[j]; order[j] = x;
            }
        for (unsigned k = 0; k < n; ++k) {
            const unsigned t = order[k];
            Fiber &f = s->fib[t];
            if (f.state == F_DONE) continue;
            if (f.state == F_WAIT_BAR && f.bar_gen == s->bar_gen) continue;
            if (f.state == F_WAIT_WARP && !slot_ready(s, &f)) continue;
            if (f.state == F_SPIN) spinning = true; else progress = true;
            f.state = F_RUN;
            s->cur = &f;
            emu_switch(&s->main_sp, f.sp);
        }
        if (!progress && !spinning) {
            if (++idle_rounds > 2) {
                fprintf(stderr, "emu: kernel %s, block (%u,%u,%u) is deadlocked: %u threads alive, none can run "
                        "(divergent __syncthreads / collective whose lanes never arrive)\n", s->kernel ? s->kernel : "?", bid.x, bid.y, bid.z,
                        s->alive);
                for (unsigned t = 0; t < n && t < 1024; ++t) {
                    const Fiber &f = s->fib[t];
                    if (f.state == F_WAIT_WARP) {
                        fprintf(stderr, "  thread %u (warp %u, lane %u) waits in %s(mask 0x%08x) at %s:%d\n", t, f.warp, f.lane,
                                kind_name(f.wslot->kind), f.wmask, f.wslot->file, f.wslot->line);
                        break;
                    }
                }
                for (unsigned t = 0; t < n && t < 1024; ++t)
                    if (s->fib[t].state != F_DONE) { fprintf(stderr, "  thread %u state %d\n", t, s->fib[t].state); break; }
                abort();
            }
        } else idle_rounds = 0;
    }
}

// ---- EMU_PAR=n: the blocks of a grid run on n OS threads at the same time ------------------------------------------
// By default the blocks of a launch run one after the other, which hides every race BETWEEN blocks (a slot claimed with
// atomicCAS and read by another block before its payload is written, list appends, tickets, look-back chains, "last block
// out" counters).  With EMU_PAR each calling thread owns a pool of n - 1 workers; every worker has its own scheduler
// (fibers, __shared__ storage: both thread_local) and pulls block indices from a shared counter, lowest first — the order a
// GPU starts blocks in, so a block that waits for a lower-numbered one (decoupled look-back) always finds it started.
static unsigned par_threads() {
    static int v = -1;
    if (v < 0) { const char *e = getenv("EMU_PAR"); v = e ? atoi(e) : 0; if (v < 0) v = 0; if (v > 64) v = 64; }
    return (unsigned)v;
}

struct ParJob {
    const LaunchCfg *cfg = nullptr;
    const char *kernel = nullptr;
    const std::function<void()> *body = nullptr;
    std::atomic<unsigned long long> next{0};
    unsigned long long total = 0;
};

struct ParPool {
    std::mutex mu;
    std::condition_variable cv_go, cv_done;
    std::vector<std::thread> workers;
    ParJob *job = nullptr;
    unsigned long long gen = 0;
    unsigned running = 0;
    bool quit = false;
};

static void par_run_blocks(Sched *s, ParJob *j) {
    const LaunchCfg &cfg = *j->cfg;
    if (cfg.smem > s->dyn_cap) {
        free(s->dyn);
        s->dyn_cap = cfg.smem + 4096;
        if (posix_memalign(&s->dyn, 1024, s->dyn_cap)) abort();
    }
    s->body = j->body;
    s->kernel = j->kernel;
    s->in_kernel = true;
    s->spins = 0;
    for (;;) {
        const unsigned long long b = j->next.fetch_add(1);
        if (b >= j->total) break;
        const unsigned x = (unsigned)(b % cfg.grid.x), y = (unsigned)((b / cfg.grid.x) % cfg.grid.y), z = (unsigned)(b / ((unsigned long long)cfg.grid.x * cfg.grid.y));
        if (s->dyn) memset(s->dyn, 0xCD, cfg.smem);
        run_block(s, cfg, dim3(x, y, z));
    }
    s->in_kernel = false;
    s->cur = nullptr;
}

static void par_worker(ParPool *p) {
    Sched *s = sched();
    unsigned long long seen = 0;
    for (;;) {
        ParJob *j;
        {
            std::unique_lock<std::mutex> lk(p->mu);
            p->cv_go.wait(lk, [&] { return p->quit || p->gen != seen; });
            if (p->quit) return;
            seen = p->gen;
            j = p->job;
        }
        par_run_blocks(s, j);
        {
            std::lock_guard<std::mutex> lk(p->mu);
            if (--p->running == 0) p->cv_done.notify_all();
        }
    }
}

static void launch_parallel(Sched *s, const LaunchCfg &cfg, const char *kernel, const std::function<void()> &body, unsigned long long nblocks,
                            unsigned par) {
    static thread_local ParPool *pool = nullptr;      // one pool per calling thread (= per emulated GPU); lives as long as the process
    if (!pool) {
        pool = new ParPool();
        for (unsigned i = 1; i < par; ++i) pool->workers.emplace_back(par_worker, pool);
    }
    ParJob job;
    job.cfg = &cfg; job.kernel = kernel; job.body = &body; job.total = nblocks;
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        pool->job = &job;
        pool->running = (unsigned)pool->workers.size();
        pool->gen++;
    }
    pool->cv_go.notify_all();
    par_run_blocks(s, &job);                          // the calling thread works too
    std::unique_lock<std::mutex> lk(pool->mu);
    pool->cv_done.wait(lk, [&] { return pool->running == 0; });
    pool->job = nullptr;
}

static std::mutex g_trace_mu;
static std::map<std::string, unsigned long long> g_trace;

static std::map<const void *, int> g_dyn_smem;      // opt-in dynamic shared memory per kernel (default limit: 48 KB)
void set_max_dyn_smem(const void *func, int bytes) {
    std::lock_guard<std::mutex> lk(g_trace_mu);
    g_dyn_smem[func] = bytes;
}

void launch(const LaunchCfg &cfg, const char *kernel, const void *func, const std::function<void()> &body) {
    int smem_limit = 48 * 1024;
    {
        std::lock_guard<std::mutex> lk(g_trace_mu);
        g_trace[kernel] += 1;
        auto it = g_dyn_smem.find(func);
        if (it != g_dyn_smem.end() && it->second > smem_limit) smem_limit = it->second;
    }
    Sched *s = sched();
    const unsigned n = cfg.block.x * cfg.block.y * cfg.block.z;
    if (n == 0 || n > MAX_THREADS) { fprintf(stderr, "emu: bad block size %u\n", n); abort(); }
    // what the CUDA runtime rejects with "invalid configuration argument" / "invalid argument" (it would surface as a
    // failed launch on the GPU; here it stops the test)
    if (cfg.grid.x == 0 || cfg.grid.y == 0 || cfg.grid.z == 0 || cfg.grid.x > 0x7fffffffu || cfg.grid.y > 65535u || cfg.grid.z > 65535u ||
        cfg.block.z > 64u) {
        fprintf(stderr, "emu: invalid launch configuration of %s: grid (%u,%u,%u) block (%u,%u,%u)\n", kernel, cfg.grid.x, cfg.grid.y,
                cfg.grid.z, cfg.block.x, cfg.block.y, cfg.block.z);
        abort();
    }
    if (cfg.smem > (size_t)smem_limit) {
        fprintf(stderr, "emu: %s launched with %zu bytes of dynamic shared memory, limit %d (cudaFuncSetAttribute missing?)\n", kernel,
                cfg.smem, smem_limit);
        abort();
    }
    if (s->in_kernel) { fprintf(stderr, "emu: nested launch\n"); abort(); }
    if (cfg.smem > s->dyn_cap) {
        free(s->dyn);
        s->dyn_cap = cfg.smem + 4096;
        if (posix_memalign(&s->dyn, 1024, s->dyn_cap)) abort();
    }
    const unsigned long long nblocks = (unsigned long long)cfg.grid.x * cfg.grid.y * cfg.grid.z;
    const unsigned par = par_threads();
    if (par > 1 && nblocks > 1) { launch_parallel(s, cfg, kernel, body, nblocks, par); return; }
    s->body = &body;
    s->kernel = kernel;
    s->in_kernel = true;
    s->spins = 0;
    for (unsigned z = 0; z < cfg.grid.z; ++z)
        for (unsigned y = 0; y < cfg.grid.y; ++y)
            for (unsigned x = 0; x < cfg.grid.x; ++x) {
                if (s->dyn) memset(s->dyn, 0xCD, cfg.smem);   // shared memory starts undefined
                run_block(s, cfg, dim3(x, y, z));
            }
    s->in_kernel = false;
    s->cur = nullptr;
}

// ---- guarded device allocator -------------------------------------------------------------------------------------
struct Alloc { void *base; size_t total, user; };   // total == 0: posix_memalign (EMU_GUARD=0)
static std::mutex g_mu;
static std::map<void *, Alloc> g_allocs;
// accounting (emu_alloc_stats): live bytes of the user sizes, their peak, cudaMalloc calls, the armed failure (emu_fail_alloc)
static size_t g_live_bytes = 0, g_peak_bytes = 0;
static unsigned long long g_mallocs = 0, g_fail_at = 0;
static bool guard_on() { static int v = -1; if (v < 0) { const char *e = getenv("EMU_GUARD"); v = !(e && e[0] == '0'); } return v != 0; }

static void account(void *q, const Alloc &a) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_allocs[q] = a;
    g_live_bytes += a.user;
    if (g_live_bytes > g_peak_bytes) g_peak_bytes = g_live_bytes;
}

cudaError_t dev_malloc(void **p, size_t n) {
    const size_t page = 4096;
    const size_t user = (n + 255) & ~(size_t)255;   // cudaMalloc granularity seen by the kernels: 256 B
    {
        std::lock_guard<std::mutex> lk(g_mu);
        ++g_mallocs;
        if (g_fail_at && g_mallocs == g_fail_at) { g_fail_at = 0; return cudaErrorMemoryAllocation; }
    }
    if (!guard_on()) {
        void *q = nullptr;
        if (posix_memalign(&q, 256, user ? user : 256)) return cudaErrorMemoryAllocation;
        memset(q, 0xCD, user ? user : 256);
        account(q, Alloc{q, 0, user});
        *p = q;
        return cudaSuccess;
    }
    const size_t body = (user + page - 1) & ~(page - 1);
    const size_t total = body + page;
    char *base = (char *)mmap(nullptr, total ? total : page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (base == MAP_FAILED) return cudaErrorMemoryAllocation;
    mprotect(base + body, page, PROT_NONE);          // an access past the end of the allocation faults
    char *q = base + (body - user);
    if (user <= (64u << 20)) memset(q, 0xCD, user);  // never-written memory is recognisable (large buffers stay lazy)
    account(q, Alloc{base, total, user});
    *p = q;
    return cudaSuccess;
}

cudaError_t dev_free(void *p) {
    if (!p) return cudaSuccess;
    Alloc a;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_allocs.find(p);
        if (it == g_allocs.end()) { fprintf(stderr, "emu: cudaFree of an unknown pointer %p\n", p); abort(); }
        a = it->second;
        g_allocs.erase(it);
        g_live_bytes -= a.user;
    }
    if (a.total) munmap(a.base, a.total);
    else free(p);
    return cudaSuccess;
}

}  // namespace emu

// ---- runtime stubs ---------------------------------------------------------------------------------------------
static int env_int(const char *name, int dflt) { const char *e = getenv(name); return e ? atoi(e) : dflt; }

cudaError_t cudaGetDeviceCount(int *n) { *n = env_int("EMU_DEVICES", 8); return cudaSuccess; }
cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) {
    memset(p, 0, sizeof(*p));
    snprintf(p->name, sizeof(p->name), "SIMT emulator (CPU, tests/emu)");
    p->major = 9; p->minor = 0;
    p->multiProcessorCount = env_int("EMU_SMS", 2);
    return cudaSuccess;
}
struct emu_event { double t; };
static double now_ms() { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec / 1e6; }
static std::atomic<long long> g_live_events{0};
cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new emu_event{0}; ++g_live_events; return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; --g_live_events; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t = now_ms(); return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) { *ms = (float)(b->t - a->t); return cudaSuccess; }

extern "C" size_t emu_kernel_trace(char *buf, size_t cap) {
    std::lock_guard<std::mutex> lk(emu::g_trace_mu);
    std::string out;
    for (auto &kv : emu::g_trace) { out += kv.first; out += '\n'; }
    emu::g_trace.clear();
    if (cap) { const size_t n = out.size() < cap - 1 ? out.size() : cap - 1; memcpy(buf, out.data(), n); buf[n] = 0; }
    return out.size();
}

extern "C" void emu_alloc_stats(unsigned long long out[5]) {
    std::lock_guard<std::mutex> lk(emu::g_mu);
    out[0] = emu::g_allocs.size(); out[1] = emu::g_live_bytes; out[2] = emu::g_peak_bytes; out[3] = (unsigned long long)g_live_events.load();
    out[4] = emu::g_mallocs;
    emu::g_peak_bytes = emu::g_live_bytes;
}

extern "C" void emu_fail_alloc(unsigned long long k) {
    std::lock_guard<std::mutex> lk(emu::g_mu);
    emu::g_fail_at = k ? emu::g_mallocs + k : 0;
}
