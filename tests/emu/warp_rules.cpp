// tests/emu/warp_rules.cpp — TEST INFRASTRUCTURE: self-tests of the SIMT emulator's warp collectives (cuda_emu.h).
// tests/test_emu_warp_rules.py compiles this file with cuda_emu.cpp and runs one case per process:
//
//     warp_rules <case>        prints "ok <case> ..." and exits 0, or stops (abort) with the emulator's report
//
// Positive cases check results against a brute-force model of the same warp; negative cases break one rule of the
// collectives each and must stop the kernel with that rule's report (or, for a shuffle from an exited lane, read the
// emulator's poison value).
#include "cuda_emu.h"

#include <stdio.h>

#include <string>
#include <vector>

static const unsigned FULL = 0xffffffffu;
static unsigned lane_of() { return threadIdx.x & 31u; }

// ---- positive cases --------------------------------------------------------------------------------------------------

// out[t] = __match_any_sync over the live lanes of t's warp; a lane with exit_mod != 0 and key % exit_mod == 0 leaves first
__global__ void k_match(const uint32_t *keys, uint32_t *out, unsigned exit_mod) {
    const unsigned t = threadIdx.x;
    const uint32_t key = keys[t];
    if (exit_mod && key % exit_mod == 0) return;
    out[t] = __match_any_sync(FULL, key);
}

// 64-bit keys: equal low words, different high words must not group
__global__ void k_match64(const uint64_t *keys, uint32_t *out) {
    out[threadIdx.x] = __match_any_sync(FULL, keys[threadIdx.x]);
}

// divergent work (per-lane trip counts and branches, no collective inside), then full-mask collectives after reconvergence
__global__ void k_reconverge(const uint32_t *trips, uint32_t *out) {
    const unsigned t = threadIdx.x, lane = lane_of();
    uint32_t acc = 0;
    for (uint32_t i = 0; i < trips[t]; ++i) {
        if ((i + lane) & 1) acc += i * 3u + 1u;
        else acc ^= i << (lane & 7u);
    }
    uint32_t sum = acc;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(FULL, sum, o);
    const uint32_t right = __shfl_sync(FULL, acc, (lane + 1) & 31u);
    const uint32_t up = __shfl_up_sync(FULL, acc, 3);
    const uint32_t down = __shfl_down_sync(FULL, acc, 5);
    const uint32_t odd = __ballot_sync(FULL, acc & 1u);
    out[4 * t + 0] = sum;
    out[4 * t + 1] = right;
    out[4 * t + 2] = up + down;
    out[4 * t + 3] = odd;
}

// ---- negative cases: one broken rule each --------------------------------------------------------------------------

__global__ void k_two_sites() {
    if (lane_of() & 1) __syncwarp();
    else __syncwarp();
}

__global__ void k_two_kinds(uint32_t *out) {
    if (lane_of() < 16) __syncwarp();
    else out[threadIdx.x] = __ballot_sync(FULL, 1);
}

__global__ void k_two_masks(uint32_t *out) {
    const unsigned lane = lane_of();
    out[threadIdx.x] = __shfl_sync(lane < 16 ? FULL : 0xffff0000u, lane, 16);
}

__global__ void k_outside_mask() { __syncwarp(0xfffffffeu); }

__global__ void k_activemask(uint32_t *out) { out[threadIdx.x] = __popc(__activemask()); }

// the shape k_hist_dense had: a full-mask match inside a loop whose trip count differs from lane to lane, then a barrier
__global__ void k_loop_match(const uint32_t *trips, uint32_t *out) {
    uint32_t n = 0;
    for (uint32_t i = 0; i < trips[threadIdx.x]; ++i) n += __popc(__match_any_sync(FULL, i & 3u));
    __syncthreads();
    out[threadIdx.x] = n;
}

// lanes 16..31 exit; lanes 0..15 read lane + 16
__global__ void k_shfl_exited(uint32_t *out) {
    const unsigned lane = lane_of();
    if (lane >= 16) return;
    out[threadIdx.x] = __shfl_sync(FULL, 1000u + lane, lane + 16);
}

// ---- driver --------------------------------------------------------------------------------------------------------

static uint64_t rng_state = 0x2545f4914f6cdd1dull;
static uint32_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return (uint32_t)(rng_state >> 11); }

static int fails = 0;
#define CHECK(cond, ...) do { if (!(cond)) { if (fails++ < 10) { fprintf(stderr, "warp_rules: "); fprintf(stderr, __VA_ARGS__); fprintf(stderr, "\n"); } } } while (0)

// brute force: the lanes of t's warp that are live (alive[]) and hold t's key
template <class K>
static uint32_t group_of(const std::vector<K> &keys, const std::vector<bool> &alive, unsigned t) {
    const unsigned w0 = t & ~31u;
    uint32_t g = 0;
    for (unsigned l = 0; l < 32 && w0 + l < keys.size(); ++l)
        if (alive[w0 + l] && keys[w0 + l] == keys[t]) g |= 1u << l;
    return g;
}

// n threads in one block; keys from an alphabet of `alphabet` values; exit_mod as in k_match
static void run_match(unsigned n, unsigned alphabet, unsigned exit_mod, int rounds) {
    for (int r = 0; r < rounds; ++r) {
        std::vector<uint32_t> keys(n), out(n, 0xdeadbeefu);
        std::vector<bool> alive(n);
        for (unsigned t = 0; t < n; ++t) {
            keys[t] = rnd() % alphabet;
            if (r & 1) keys[t] |= 0x80000000u;      // high keys (0xffffffff-like empty keys of the kernels)
            alive[t] = !(exit_mod && keys[t] % exit_mod == 0);
        }
        const uint32_t *kp = keys.data();
        uint32_t *op = out.data();
        EMU_LAUNCH((k_match), (dim3(1), dim3(n)), (kp, op, exit_mod));
        for (unsigned t = 0; t < n; ++t)
            if (alive[t]) CHECK(out[t] == group_of(keys, alive, t), "n %u round %d thread %u: match 0x%08x, want 0x%08x", n, r, t, out[t], group_of(keys, alive, t));
    }
}

static void case_match_full() { run_match(256, 2, 0, 4); run_match(256, 7, 0, 4); run_match(256, 64, 0, 4); run_match(32, 1, 0, 1); }
static void case_match_partial() { run_match(80, 3, 0, 4); run_match(33, 2, 0, 4); run_match(200, 9, 0, 4); }
static void case_match_exited() { run_match(256, 5, 5, 4); run_match(256, 12, 3, 4); run_match(112, 4, 2, 4); }

static void case_match_64bit() {
    const unsigned n = 128;
    std::vector<uint64_t> keys(n);
    std::vector<uint32_t> out(n);
    std::vector<bool> alive(n, true);
    for (unsigned t = 0; t < n; ++t) keys[t] = ((uint64_t)(rnd() % 3) << 32) | (rnd() % 2);
    const uint64_t *kp = keys.data();
    uint32_t *op = out.data();
    EMU_LAUNCH((k_match64), (dim3(1), dim3(n)), (kp, op));
    for (unsigned t = 0; t < n; ++t) CHECK(out[t] == group_of(keys, alive, t), "thread %u: match 0x%08x, want 0x%08x", t, out[t], group_of(keys, alive, t));
}

static void case_reconverge() {
    const unsigned n = 256;
    std::vector<uint32_t> trips(n), out(4 * n), acc(n);
    for (unsigned t = 0; t < n; ++t) trips[t] = rnd() % 40;
    for (unsigned t = 0; t < n; ++t) {
        const unsigned lane = t & 31u;
        uint32_t a = 0;
        for (uint32_t i = 0; i < trips[t]; ++i) {
            if ((i + lane) & 1) a += i * 3u + 1u;
            else a ^= i << (lane & 7u);
        }
        acc[t] = a;
    }
    const uint32_t *tp = trips.data();
    uint32_t *op = out.data();
    EMU_LAUNCH((k_reconverge), (dim3(2), dim3(n)), (tp, op));
    for (unsigned t = 0; t < n; ++t) {
        const unsigned w0 = t & ~31u, lane = t & 31u;
        uint32_t sum = 0, odd = 0;
        for (unsigned l = 0; l < 32; ++l) { sum += acc[w0 + l]; odd |= (acc[w0 + l] & 1u) << l; }
        const uint32_t up = lane >= 3 ? acc[t - 3] : acc[t], down = lane + 5 < 32 ? acc[t + 5] : acc[t];
        CHECK(out[4 * t] == sum, "thread %u: xor-reduce %u, want %u", t, out[4 * t], sum);
        CHECK(out[4 * t + 1] == acc[w0 + ((lane + 1) & 31u)], "thread %u: shfl %u", t, out[4 * t + 1]);
        CHECK(out[4 * t + 2] == up + down, "thread %u: shfl up + down %u, want %u", t, out[4 * t + 2], up + down);
        CHECK(out[4 * t + 3] == odd, "thread %u: ballot 0x%08x, want 0x%08x", t, out[4 * t + 3], odd);
    }
}

static std::vector<uint32_t> g_out(1024), g_trips(1024);

static void case_two_sites() { EMU_LAUNCH((k_two_sites), (dim3(1), dim3(64)), ()); }
static void case_two_kinds() { uint32_t *op = g_out.data(); EMU_LAUNCH((k_two_kinds), (dim3(1), dim3(64)), (op)); }
static void case_two_masks() { uint32_t *op = g_out.data(); EMU_LAUNCH((k_two_masks), (dim3(1), dim3(64)), (op)); }
static void case_outside_mask() { EMU_LAUNCH((k_outside_mask), (dim3(1), dim3(64)), ()); }
static void case_activemask() { uint32_t *op = g_out.data(); EMU_LAUNCH((k_activemask), (dim3(1), dim3(64)), (op)); }
static void case_loop_match() {
    for (unsigned t = 0; t < 64; ++t) g_trips[t] = 1 + (t & 31u) / 8;   // 1..4 trips, differing inside each warp
    const uint32_t *tp = g_trips.data();
    uint32_t *op = g_out.data();
    EMU_LAUNCH((k_loop_match), (dim3(1), dim3(64)), (tp, op));
}
static void case_shfl_exited() {
    uint32_t *op = g_out.data();
    EMU_LAUNCH((k_shfl_exited), (dim3(1), dim3(64)), (op));
    for (unsigned t = 0; t < 64; ++t)
        if ((t & 31u) < 16) printf("thread %u read 0x%08x\n", t, op[t]);
}

int main(int argc, char **argv) {
    struct Case { const char *name; void (*run)(); };
    static const Case cases[] = {
        {"match_full", case_match_full}, {"match_partial", case_match_partial}, {"match_exited", case_match_exited},
        {"match_64bit", case_match_64bit}, {"reconverge", case_reconverge},
        {"two_sites", case_two_sites}, {"two_kinds", case_two_kinds}, {"two_masks", case_two_masks},
        {"outside_mask", case_outside_mask}, {"activemask", case_activemask}, {"loop_match", case_loop_match},
        {"shfl_exited", case_shfl_exited},
    };
    if (argc != 2) { fprintf(stderr, "usage: warp_rules <case>\n"); return 2; }
    for (const Case &c : cases)
        if (std::string(argv[1]) == c.name) {
            c.run();
            if (fails) { fprintf(stderr, "warp_rules: %s: %d mismatches\n", c.name, fails); return 1; }
            printf("ok %s\n", c.name);
            return 0;
        }
    fprintf(stderr, "warp_rules: unknown case %s\n", argv[1]);
    return 2;
}
