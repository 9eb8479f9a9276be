// tests/emu/arrival_emu.cpp -- TEST INFRASTRUCTURE. Runs the device source of the whole-layer search tier
// (mq_layer_search in permafrost-engine_b200/csrc/pfnav_layer_search.cuh, unmodified) as one CTA of nt CPU threads, so
// that its level-synchronous replays of N_ClosestPathable and n_closest_island_tiles are checked against the host routine
// (pfnav_route_arrival_consts) in the CPU test suite. The CUDA keywords and intrinsics the header uses are defined as
// plain C++; __syncthreads is a pthread barrier. This is not a product path: nothing in libpfnav.so links or calls it, and
// it is built only by tests/test_arrival_search_emu.py.
#include <pthread.h>
#include <stdint.h>
#include <stddef.h>
#include <math.h>
#include <algorithm>
#include <thread>
#include <vector>
#include "../../include/pfnav.h"

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __restrict__
#define __shared__ static
#define __launch_bounds__(...)
using std::max;
using std::min;

struct emu_dim3 { unsigned x, y, z; };
static thread_local emu_dim3 threadIdx;
static const emu_dim3 blockIdx = {0, 0, 0}, blockDim = {32, 1, 1}, gridDim = {1, 1, 1};
static pthread_barrier_t g_barrier;
static inline void __syncwarp() { pthread_barrier_wait(&g_barrier); }
static inline void __syncthreads() { pthread_barrier_wait(&g_barrier); }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline void atomicOr(uint32_t *p, uint32_t v) { __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline void atomicAdd(int *p, int v) { __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline void atomicMin(int *p, int v)
{
    int cur = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (v < cur && !__atomic_compare_exchange_n(p, &cur, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
}
struct float2 { float x, y; };
static inline float2 make_float2(float x, float y) { return {x, y}; }

#include "../../permafrost-engine_b200/csrc/pfnav_map_view.cuh"
#include "../../permafrost-engine_b200/csrc/pfnav_query_kernel.cuh"
#include "../../permafrost-engine_b200/csrc/pfnav_layer_search.cuh"

static mq_layer_shared g_L;

// cost / blk / gisl: row-major layer images [layer][H64][W64], exactly what the device holds (gisl may be NULL when
// every search is CLOSEST_PATHABLE). Search i starts at the in-map tile (tr[i], tc[i]) of `layer`; cp[i] selects
// N_ClosestPathable (out_tile[i]: row * W64 + col, or -1) or n_closest_island_tiles (list[i][256] tile centres, out_n[i]).
extern "C" int emu_layer_search(const uint8_t *cost, const uint16_t *blk, const uint16_t *gisl, int chunk_w, int chunk_h,
                                float map_x, float map_z, int layer, const int32_t *cp, const int32_t *tr, const int32_t *tc,
                                int n, int nt, int32_t *out_tile, float *list, int32_t *out_n)
{
    if (nt < 1 || nt > MQ_LAYER_THREADS) return -1;
    const MapView m = {cost, blk, chunk_w * 64, chunk_h * 64, chunk_w, chunk_h, map_x, map_z};
    std::vector<int32_t> scratch(mq_layer_scratch_words(m.W64, m.H64));
    pthread_barrier_init(&g_barrier, nullptr, nt);
    std::vector<std::thread> th;
    for (int t = 0; t < nt; t++)
        th.emplace_back([&, t]() {
            threadIdx = {(unsigned)t, 0, 0};
            for (int i = 0; i < n; i++) {
                mq_layer_search(g_L, scratch.data(), m, gisl, layer, cp[i] != 0, tr[i], tc[i],
                                (float2 *)(list + (size_t)i * MQ_LIST_MAX * 2), t, nt);
                if (t == 0) { out_tile[i] = g_L.tile; out_n[i] = cp[i] ? 0 : g_L.n; }
                __syncthreads();
            }
        });
    for (auto &t : th) t.join();
    pthread_barrier_destroy(&g_barrier);
    return 0;
}
