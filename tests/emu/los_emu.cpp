// tests/emu/los_emu.cpp -- TEST INFRASTRUCTURE. Runs the device source of k_los_level and k_los_b
// (permafrost-engine_b200/csrc/pfnav_los_kernel.cuh, unmodified) as ONE warp on 32 CPU threads, so that the level-parallel
// LOS pass, its certificate and the replay fallback are checked against the plain-C port in the CPU test suite too. The
// CUDA keywords, intrinsics and warp collectives the header uses are defined as plain C++; every collective is a pthread
// barrier. This is not a product path: nothing in libpfnav.so links or calls it, and it is built only by
// tests/test_los_level_emu.py (also with -DLOS_LEVEL_NO_CERTIFICATE or -DLOS_LEVEL_ALWAYS_REPLAY).
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <thread>
#include <vector>
#include "../../include/pfnav.h"

#define __device__
#define __global__
#define __forceinline__ inline
#define __restrict__
#define __shared__
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define pf_globaltimer() 0ull

struct uint4 { uint32_t x, y, z, w; };
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
struct emu_dim3 { unsigned x, y, z; };
static thread_local emu_dim3 threadIdx;
static pthread_barrier_t g_barrier;
static uint64_t g_xchg[32];
alignas(16) uint8_t smem_raw[1 << 15];

static inline void __syncwarp() { pthread_barrier_wait(&g_barrier); }
static inline void __threadfence() {}
static inline void __nanosleep(unsigned) {}
template <class T> static inline T __ldg(const T *p) { return *p; }
template <class T> static inline T __ldcg(const T *p) { return *p; }

// every lane publishes a value, then reads the one of lane `src(lane)`
template <class F> static inline uint64_t exchange(uint64_t v, F src)
{
    g_xchg[threadIdx.x] = v;
    pthread_barrier_wait(&g_barrier);
    const int s = src((int)threadIdx.x);
    const uint64_t r = (s >= 0 && s < 32) ? g_xchg[s] : v;
    pthread_barrier_wait(&g_barrier);
    return r;
}
static inline int __shfl_sync(unsigned, int v, int src) { return (int)exchange((uint32_t)v, [=](int) { return src; }); }
static inline unsigned __shfl_up_sync(unsigned, unsigned v, int d) { return (unsigned)exchange(v, [=](int l) { return l - d; }); }
static inline int __shfl_up_sync(unsigned, int v, int d) { return (int)exchange((uint32_t)v, [=](int l) { return l - d; }); }
static inline unsigned __shfl_down_sync(unsigned, unsigned v, int d) { return (unsigned)exchange(v, [=](int l) { return l + d; }); }
template <class F> static inline uint64_t reduce(uint64_t v, F op)
{
    g_xchg[threadIdx.x] = v;
    pthread_barrier_wait(&g_barrier);
    uint64_t r = g_xchg[0];
    for (int k = 1; k < 32; k++) r = op(r, g_xchg[k], k);
    pthread_barrier_wait(&g_barrier);
    return r;
}
static inline unsigned __ballot_sync(unsigned, int p)
{
    return (unsigned)reduce(p ? 1 : 0, [](uint64_t a, uint64_t b, int k) { return a | (b << k); });
}
static inline int __any_sync(unsigned, int p) { return __ballot_sync(0, p) != 0; }
static inline unsigned __reduce_add_sync(unsigned, unsigned v) { return (unsigned)reduce(v, [](uint64_t a, uint64_t b, int) { return a + b; }); }
static inline int __popcll(uint64_t v) { return __builtin_popcountll(v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline unsigned atomicAdd(unsigned *p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicOr(unsigned *p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline int atomicMax(int *p, int v)
{
    int old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
template <class C> static inline uint32_t bytecmp(uint32_t a, uint32_t b, C c)
{
    uint32_t r = 0;
    for (int k = 0; k < 4; k++)
        if (c((a >> (8 * k)) & 0xFFu, (b >> (8 * k)) & 0xFFu)) r |= 0xFFu << (8 * k);
    return r;
}
static inline uint32_t __vcmpeq4(uint32_t a, uint32_t b) { return bytecmp(a, b, [](uint32_t x, uint32_t y) { return x == y; }); }
static inline uint32_t __vcmpne4(uint32_t a, uint32_t b) { return bytecmp(a, b, [](uint32_t x, uint32_t y) { return x != y; }); }
static inline uint32_t __vcmpgtu4(uint32_t a, uint32_t b) { return bytecmp(a, b, [](uint32_t x, uint32_t y) { return x > y; }); }

#include "../../permafrost-engine_b200/csrc/pfnav_los_kernel.cuh"

static_assert(sizeof(LosSmemB) <= sizeof(smem_raw), "one warp's shared memory");

// cost / blk / fmask: row-major layer images [layer][H64][W64], exactly what the device holds (fmask may be NULL when no
// request is attacking); reqs: n requests sorted so that prev_index < own index; fields: n x 4096 output bytes; trace:
// n x 4 words (may be NULL). variant: 2 = k_los_level, 1 = k_los_b.
extern "C" int emu_los_fields(const uint8_t *cost, const uint16_t *blk, const uint16_t *fmask, const uint16_t *enemies, int H64,
                              int W64, float map_x, float map_z, const pfnav_los_req *reqs, int n, uint8_t *fields,
                              unsigned long long *trace, int variant)
{
    for (int i = 0; i < n; i++)
        if (reqs[i].prev_index >= i) return -1;
    FlowGrids g;
    memset(&g, 0, sizeof(g));
    g.cost = cost; g.blk = blk; g.fmask = fmask; g.W64 = W64; g.H64 = H64;
    for (int f = 0; f < 16; f++) g.enemies[f] = enemies ? enemies[f] : 0;
    const LosMapInfo mi{map_x, map_z};
    unsigned counter = 0;
    std::vector<int> done(n > 0 ? n : 1, 0);
    pthread_barrier_init(&g_barrier, nullptr, 32);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < 32; t++)
        th.emplace_back([&, t]() {
            threadIdx = {t, 0, 0};
            if (variant == 2) k_los_level(g, mi, reqs, n, fields, nullptr, &counter, done.data(), trace);
            else k_los_b(g, mi, reqs, n, fields, nullptr, &counter, done.data(), trace);
        });
    for (auto &t : th) t.join();
    pthread_barrier_destroy(&g_barrier);
    return 0;
}
