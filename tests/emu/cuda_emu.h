// tests/emu/cuda_emu.h — TEST INFRASTRUCTURE: a CPU SIMT emulator for the kernel SOURCES of minbpe_b200/csrc.
//
// Why: the kernels can only be validated on an H100.  When no GPU is reachable (a build host without one) the next best
// check is to run the very same kernel source — same index arithmetic, same shared-memory protocol, same warp
// collectives, same atomics, same host-side launch sequence — on the CPU and compare the C ABI's results with the
// oracle.  tests/emu/build_emu.py rewrites only the launch syntax (`k<<<g, b, s, st>>>(args)`) and the
// `extern __shared__` declarations, and compiles b200bpe.cu with g++ against this header into
// tests/emu/_build/libb200bpe_emu.so, which exports the same C ABI as libb200bpe.so.
//
// What it is NOT: a CPU fallback of the product.  Nothing in minbpe_b200/ loads it; only tests/test_emu*.py do, in
// a subprocess, through the BPE_LIB_PATH override.  It proves logic, not performance, memory-model behaviour across
// GPUs, or the PTX paths (TMA bulk copies and mbarriers are emulated as immediate copies).
//
// Execution model
//   * one CUDA thread = one fiber (own stack, cooperative switch in ~20 instructions); the fibers of a block share
//     the `__shared__` variables (static thread_local: one block runs at a time per OS thread);
//   * __syncthreads / warp collectives (__syncwarp, __shfl*_sync, __ballot_sync, __all_sync, __any_sync, __reduce_*_sync,
//     __match_any_sync) are rendezvous points: a fiber waits there until the other threads of the block / the other lanes
//     named in the mask that are still alive have arrived — divergence, early exits and data-dependent loops between them
//     behave as on a GPU;
//   * warp collectives are held to the rule the kernels are written to: every live lane named in a collective's mask
//     executes that same call — same call site, same kind, same mask — and the calling lane is in its own mask.  The k-th
//     collective of every lane of a warp is one rendezvous; the first lane there records its site, kind and mask and every
//     later lane is compared with them.  A mismatch stops the kernel with both sites.  __activemask() stops the kernel:
//     without lock-step hardware the converged set has no value, and on a GPU it has one that depends on scheduling.  A
//     shuffle that reads a lane which is not taking part (exited, or outside the mask) gets the 0xCD guard fill;
//   * the threads of a block run in thread-index order between two synchronisation points, or — EMU_ORDER=reverse | random —
//     in another order: a kernel whose result depends on that order has a data race;
//   * blocks of a grid run one after another in blockIdx order (legal: CUDA promises no inter-block progress);
//     spin-waits on memory (`ld.volatile`, `ld.acquire.sys`) yield to the other fibers and give up after a bound;
//   * several OS threads may launch at the same time (one per emulated GPU / rank): peer memory is plain host
//     memory, release/acquire accesses map to C++ atomics;
//   * cudaMalloc places every allocation in front of an inaccessible guard page (EMU_GUARD=0 turns it off) and
//     fills it with 0xCD, so an overrun or a read of never-written memory shows;
//   * the vector types carry their CUDA alignment: a build with EMU_SANITIZE=1 (build_emu.py: UBSan alignment check) traps on
//     every uint2 / uint4 / ulonglong2 access that a GPU would fault on.
#pragma once
#define BPE_SIMT_EMU 1
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <functional>
#include <type_traits>

// ---- CUDA qualifiers -------------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define EMU_NOINLINE __attribute__((noinline))   /* build_emu.py rewrites __noinline__ (libstdc++ spells the attribute that way) */
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static thread_local

// ---- vector types ------------------------------------------------------------------------------------------------
struct uint2 { unsigned int x, y; } __attribute__((aligned(8)));
struct uint4 { unsigned int x, y, z, w; } __attribute__((aligned(16)));
struct ulonglong2 { unsigned long long x, y; } __attribute__((aligned(16)));
static inline uint2 make_uint2(unsigned int x, unsigned int y) { return uint2{x, y}; }
static inline uint4 make_uint4(unsigned int x, unsigned int y, unsigned int z, unsigned int w) { return uint4{x, y, z, w}; }
struct dim3 {
    unsigned int x, y, z;
    dim3(unsigned int a = 1, unsigned int b = 1, unsigned int c = 1) : x(a), y(b), z(c) {}
};

// ---- the running thread ------------------------------------------------------------------------------------------
namespace emu {
struct ThreadCtx { dim3 tid, bid, bdim, gdim; };
ThreadCtx *ctx();                 // the fiber that is running on this OS thread
void sync_threads();              // __syncthreads
enum { C_SHFL, C_UP, C_DOWN, C_XOR, C_BALLOT, C_ALL, C_ANY, C_OR, C_MAX, C_SYNC, C_MATCH };
// one warp collective of the running lane; file:line is its call site
uint64_t collective(int kind, uint32_t mask, uint64_t val, uint32_t arg, const char *file, int line);
[[noreturn]] void activemask_called(const char *file, int line);
void spin();                      // called from every polling load: lets the other fibers run, bounds the wait
void *dyn_smem();                 // base of the block's dynamic shared memory
long long clock();                // monotonic "SM clock"
struct LaunchCfg {
    dim3 grid, block; size_t smem; void *stream;
    LaunchCfg(dim3 g, dim3 b, size_t s = 0, void *st = nullptr) : grid(g), block(b), smem(s), stream(st) {}
};
void launch(const LaunchCfg &cfg, const char *kernel, const void *func, const std::function<void()> &body);
void set_max_dyn_smem(const void *func, int bytes);   // cudaFuncSetAttribute(MaxDynamicSharedMemorySize)
}  // namespace emu
// names of the kernels launched by this process since the last call, one per line (tests/emu/kernel_coverage.py)
extern "C" size_t emu_kernel_trace(char *buf, size_t cap);
// device-memory accounting (tests/test_emu_ownership.py): out[0] live allocations, [1] their bytes, [2] peak live bytes since
// the last call (it restarts at the live bytes), [3] live events, [4] cudaMalloc calls so far
extern "C" void emu_alloc_stats(unsigned long long out[5]);
// the k-th cudaMalloc from now returns cudaErrorMemoryAllocation (k = 0: none)
extern "C" void emu_fail_alloc(unsigned long long k);
#define threadIdx (emu::ctx()->tid)
#define blockIdx (emu::ctx()->bid)
#define blockDim (emu::ctx()->bdim)
#define gridDim (emu::ctx()->gdim)
#define EMU_UNPAREN(...) __VA_ARGS__
#define EMU_STR2(...) #__VA_ARGS__
#define EMU_STR(...) EMU_STR2(__VA_ARGS__)
#define EMU_LAUNCH(K, CFG, ARGS) emu::launch(emu::LaunchCfg CFG, EMU_STR(EMU_UNPAREN K), reinterpret_cast<const void *>(&(EMU_UNPAREN K)), [&]() { EMU_UNPAREN K ARGS; })

static inline void __syncthreads() { emu::sync_threads(); }
#define EMU_SITE const char *file = __builtin_FILE(), int line = __builtin_LINE()   /* the caller's file:line */
#define EMU_AT file, line
static inline void __syncwarp(unsigned mask = 0xffffffffu, EMU_SITE) { emu::collective(emu::C_SYNC, mask, 0, 0, EMU_AT); }
static inline void __threadfence() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
// no kernel may use it: the emulator cannot give it a meaning, and a GPU gives it one that depends on scheduling
static inline unsigned __activemask(EMU_SITE) { emu::activemask_called(EMU_AT); }
static inline long long clock64() { return emu::clock(); }

template <class T> static inline uint64_t emu_bits(T v) { uint64_t b = 0; memcpy(&b, &v, sizeof(T)); return b; }
template <class T> static inline T emu_unbits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }
template <class T> static inline T __shfl_sync(unsigned m, T v, int src, EMU_SITE) { static_assert(sizeof(T) <= 8, ""); return emu_unbits<T>(emu::collective(emu::C_SHFL, m, emu_bits(v), (uint32_t)src, EMU_AT)); }
template <class T> static inline T __shfl_up_sync(unsigned m, T v, unsigned d, EMU_SITE) { return emu_unbits<T>(emu::collective(emu::C_UP, m, emu_bits(v), d, EMU_AT)); }
template <class T> static inline T __shfl_down_sync(unsigned m, T v, unsigned d, EMU_SITE) { return emu_unbits<T>(emu::collective(emu::C_DOWN, m, emu_bits(v), d, EMU_AT)); }
template <class T> static inline T __shfl_xor_sync(unsigned m, T v, int x, EMU_SITE) { return emu_unbits<T>(emu::collective(emu::C_XOR, m, emu_bits(v), (uint32_t)x, EMU_AT)); }
static inline unsigned __ballot_sync(unsigned m, int pred, EMU_SITE) { return (unsigned)emu::collective(emu::C_BALLOT, m, pred != 0, 0, EMU_AT); }
static inline int __all_sync(unsigned m, int pred, EMU_SITE) { return (int)emu::collective(emu::C_ALL, m, pred != 0, 0, EMU_AT); }
static inline int __any_sync(unsigned m, int pred, EMU_SITE) { return (int)emu::collective(emu::C_ANY, m, pred != 0, 0, EMU_AT); }
static inline unsigned __reduce_or_sync(unsigned m, unsigned v, EMU_SITE) { return (unsigned)emu::collective(emu::C_OR, m, v, 0, EMU_AT); }
static inline unsigned __reduce_max_sync(unsigned m, unsigned v, EMU_SITE) { return (unsigned)emu::collective(emu::C_MAX, m, v, 0, EMU_AT); }
// the lanes of the mask that arrived with a key equal to this lane's (a rendezvous like the others)
template <class T> static inline unsigned __match_any_sync(unsigned m, T key, EMU_SITE) {
    static_assert(sizeof(T) <= 8, "");
    return (unsigned)emu::collective(emu::C_MATCH, m, emu_bits(key), 0, EMU_AT);
}

// ---- bit tricks ------------------------------------------------------------------------------------------------
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __clz(unsigned v) { return v ? __builtin_clz(v) : 32; }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { return (unsigned)(((((uint64_t)hi) << 32) | lo) >> (sh & 31u)); }
template <class T> static inline T __ldg(const T *p) { return *p; }

template <class A, class B> static inline typename std::common_type<A, B>::type min(A a, B b) {
    typedef typename std::common_type<A, B>::type R; return (R)a < (R)b ? (R)a : (R)b;
}
template <class A, class B> static inline typename std::common_type<A, B>::type max(A a, B b) {
    typedef typename std::common_type<A, B>::type R; return (R)a > (R)b ? (R)a : (R)b;
}

// ---- atomics (several OS threads = several emulated GPUs may share memory) -------------------------------------------
template <class T, class U> static inline T atomicAdd(T *p, U v) { return __atomic_fetch_add(p, (T)v, __ATOMIC_SEQ_CST); }
template <class T, class U> static inline T atomicOr(T *p, U v) { return __atomic_fetch_or(p, (T)v, __ATOMIC_SEQ_CST); }
template <class T, class U> static inline T atomicMin(T *p, U v) {
    T old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while ((T)v < old && !__atomic_compare_exchange_n(p, &old, (T)v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
template <class T, class U> static inline T atomicMax(T *p, U v) {
    T old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while ((T)v > old && !__atomic_compare_exchange_n(p, &old, (T)v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
template <class T, class U, class W> static inline T atomicCAS(T *p, U cmp, W val) {
    T expected = (T)cmp;
    __atomic_compare_exchange_n(p, &expected, (T)val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
    return expected;
}

// ---- CUDA runtime -----------------------------------------------------------------------------------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorLaunchOutOfResources = 701 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaIpcMemLazyEnablePeerAccess = 1 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum cudaDeviceAttr { cudaDevAttrClockRate = 13 };
typedef void *cudaStream_t;
typedef struct emu_event *cudaEvent_t;
struct cudaIpcMemHandle_t { char reserved[64]; };
struct cudaDeviceProp { char name[256]; int major, minor, multiProcessorCount; };

namespace emu {
cudaError_t dev_malloc(void **p, size_t n);
cudaError_t dev_free(void *p);
}
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t n) { return emu::dev_malloc((void **)p, n); }
static inline cudaError_t cudaFree(void *p) { return emu::dev_free(p); }
template <class T> static inline cudaError_t cudaMallocHost(T **p, size_t n) { *p = (T *)malloc(n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : (e == cudaErrorMemoryAllocation ? "out of memory (emulator)" : "error (emulator)"); }
cudaError_t cudaGetDeviceCount(int *n);
cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int dev);
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr, int) { *v = 2000000; return cudaSuccess; }   // kHz of emu::clock()
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t *s) { *s = malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t *e);
cudaError_t cudaEventDestroy(cudaEvent_t e);
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr);
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b);
template <class F> static inline cudaError_t cudaFuncSetAttribute(F f, cudaFuncAttribute a, int v) {
    if (a == cudaFuncAttributeMaxDynamicSharedMemorySize) {
        if (v > 227 * 1024) return cudaErrorInvalidValue;      // sm_90: 227 KB per CTA
        emu::set_max_dyn_smem(reinterpret_cast<const void *>(f), v);
    }
    return cudaSuccess;
}
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, F, int, size_t) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t *h, void *p) { memset(h, 0, sizeof(*h)); memcpy(h, &p, sizeof(p)); return cudaSuccess; }
static inline cudaError_t cudaIpcOpenMemHandle(void **p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, &h, sizeof(*p)); return cudaSuccess; }
static inline cudaError_t cudaIpcCloseMemHandle(void *) { return cudaSuccess; }
