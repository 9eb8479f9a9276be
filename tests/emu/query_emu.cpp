// tests/emu/query_emu.cpp -- TEST INFRASTRUCTURE. Runs the device source of pfnav_map_query's search kernel
// (permafrost-engine_b200/csrc/pfnav_query_kernel.cuh, unmodified) as ONE warp on 32 CPU threads, so that the window
// replays of N_ClosestPathable and n_closest_island_tiles are checked against the host routine (pfnav_route_arrival_consts)
// in the CPU test suite too. The CUDA keywords the header uses are defined as plain C++; __syncwarp is a pthread barrier.
// This is not a product path: nothing in libpfnav.so links or calls it, and it is built only by
// tests/test_map_query_emu.py.
#include <pthread.h>
#include <stdint.h>
#include <stddef.h>
#include <math.h>
#include <algorithm>
#include <thread>
#include <vector>
#include "../../include/pfnav.h"

#define __device__
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

#include "../../permafrost-engine_b200/csrc/pfnav_map_view.cuh"
#include "../../permafrost-engine_b200/csrc/pfnav_query_kernel.cuh"

static mq_shared g_S;

// cost / blk / gisl: row-major layer images [layer][H64][W64], exactly what the device holds (gisl may be NULL when
// no query is MAXIMALLY_CLOSE); q: n CLOSEST_PATHABLE / MAXIMALLY_CLOSE queries. Per query: out (the kernel's result),
// fallback (1 = the replay left the 128 x 128 window), and for MAXIMALLY_CLOSE the listed tiles as absolute (row, col)
// pairs, mc_rc[i][256][2] with mc_n[i] entries (-1 when the query never reached a replay).
extern "C" int emu_map_search(const uint8_t *cost, const uint16_t *blk, const uint16_t *gisl, int chunk_w, int chunk_h,
                              float map_x, float map_z, const pfnav_map_query_req *q, int n, pfnav_map_query_result *out,
                              uint8_t *fallback, int32_t *mc_rc, int32_t *mc_n)
{
    const MapView m = {cost, blk, chunk_w * 64, chunk_h * 64, chunk_w, chunk_h, map_x, map_z};
    pthread_barrier_init(&g_barrier, nullptr, 32);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < 32; t++)
        th.emplace_back([=]() {
            threadIdx = {t, 0, 0};
            for (int i = 0; i < n; i++) {
                if (t == 0) { g_S.n = -1; g_S.dim = 0; }
                __syncwarp();
                mq_search(g_S, m, gisl, q[i], out + i, fallback + i, (int)t);
                if (t == 0) {
                    const bool listed = q[i].kind == PFNAV_QUERY_MAXIMALLY_CLOSE && g_S.dim > 0;
                    mc_n[i] = listed ? g_S.n : -1;
                    for (int k = 0; listed && k < g_S.n; k++) {
                        mc_rc[((size_t)i * MQ_LIST_MAX + k) * 2] = g_S.r0 + g_S.list[k] / g_S.dim;
                        mc_rc[((size_t)i * MQ_LIST_MAX + k) * 2 + 1] = g_S.c0 + g_S.list[k] % g_S.dim;
                    }
                }
                __syncwarp();
            }
        });
    for (auto &t : th) t.join();
    pthread_barrier_destroy(&g_barrier);
    return 0;
}
