// tests/emu/repair_emu.cpp -- TEST INFRASTRUCTURE. Runs the device source of the kind-0 repair seed flood
// (permafrost-engine_b200/csrc/pfnav_repair_kernel.cuh, unmodified) as one 64-thread CTA on CPU threads, so that the
// seeds k_repair_chain builds are checked against the host's breadth-first search (pfnav_repair_seeds) in the CPU test
// suite. __syncthreads is a pthread barrier. Nothing in libpfnav.so links or calls it; only
// tests/test_repair_seed_emu.py builds it.
#include <pthread.h>
#include <stdint.h>
#include <stddef.h>
#include <thread>
#include <vector>

#define __device__
#define __restrict__

struct emu_dim3 { unsigned x, y, z; };
static thread_local emu_dim3 threadIdx;
static pthread_barrier_t g_barrier;
static inline void __syncthreads() { pthread_barrier_wait(&g_barrier); }

#include "../../permafrost-engine_b200/csrc/pfnav_repair_kernel.cuh"

// cost / blk: the row-major layer image [H64][W64]; starts: n start tiles (r << 6 | c inside chunk (chunk_r, chunk_c));
// out: n * 64 seed rows
extern "C" int emu_repair_seeds(const uint8_t *cost, const uint16_t *blk, int W64, int chunk_r, int chunk_c,
                                const int32_t *starts, int n, uint64_t *out)
{
    const unsigned nthreads = 64;
    pthread_barrier_init(&g_barrier, nullptr, nthreads);
    repair_seed_smem s;
    uint64_t seed[64];
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nthreads; t++)
        th.emplace_back([&, t]() {
            threadIdx = {t, 0, 0};
            for (int i = 0; i < n; i++) {
                repair_nearest_pathable_seeds(cost, blk, 0, W64, chunk_r, chunk_c, starts[i], s, seed);
                out[(size_t)i * 64 + t] = seed[t];
                __syncthreads();
            }
        });
    for (auto &t : th) t.join();
    pthread_barrier_destroy(&g_barrier);
    return 0;
}
