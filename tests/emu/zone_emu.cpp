// tests/emu/zone_emu.cpp -- TEST INFRASTRUCTURE. Runs the device source of k_zone_seed_bits
// (permafrost-engine_b200/csrc/pfnav_zone_kernel.cuh, unmodified) as ONE warp on 32 CPU threads, so that the seed
// flood's replay of the reference's heap order is checked against the host flood (pfnav_zone_seeds) in the CPU test
// suite too. The CUDA keywords and warp intrinsics the header uses are defined as plain C++; __syncwarp is a pthread
// barrier. This is not a product path: nothing in libpfnav.so links or calls it, and it is built only by
// tests/test_zone_seed_emu.py.
#include <pthread.h>
#include <stdint.h>
#include <stddef.h>
#include <thread>
#include <vector>

#define __device__
#define __global__
#define __forceinline__ inline
#define __restrict__
#define __shared__
#define __launch_bounds__(...)

struct uint4 { uint32_t x, y, z, w; };
struct emu_dim3 { unsigned x, y, z; };
static thread_local emu_dim3 threadIdx;
static const emu_dim3 blockIdx = {0, 0, 0}, gridDim = {1, 1, 1};
static pthread_barrier_t g_barrier;
static int g_shfl;
alignas(16) uint32_t zs_smem[128 * 128 + 1 + 3 * 128 * 128 / 32];

static inline void __syncwarp() { pthread_barrier_wait(&g_barrier); }
static inline int __shfl_sync(unsigned, int v, int src)
{
    if ((int)threadIdx.x == src) g_shfl = v;
    pthread_barrier_wait(&g_barrier);
    const int r = g_shfl;
    pthread_barrier_wait(&g_barrier);
    return r;
}

#include "../../permafrost-engine_b200/csrc/pfnav_zone_kernel.cuh"

// cost / blk: row-major layer images [layer][H64][W64], exactly what the device holds; jobs: n zone_job records;
// bits: n * dim * dim / 32 words
extern "C" int emu_zone_seed_bits(const uint8_t *cost, const uint16_t *blk, int H64, int W64, int dim, const zone_job *jobs, int n,
                                  uint32_t *bits)
{
    if (dim * dim > 128 * 128) return -1;
    pthread_barrier_init(&g_barrier, nullptr, 32);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < 32; t++)
        th.emplace_back([=]() {
            threadIdx = {t, 0, 0};
            k_zone_seed_bits(cost, blk, H64, W64, dim, jobs, n, bits);
        });
    for (auto &t : th) t.join();
    pthread_barrier_destroy(&g_barrier);
    return 0;
}
