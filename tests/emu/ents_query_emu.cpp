// tests/emu/ents_query_emu.cpp -- TEST INFRASTRUCTURE. Runs the device source of the position index walk and of
// pfnav_ents_in_circles' count and write passes (permafrost-engine_b200/csrc/pfnav_ents_query_kernel.cuh, unmodified) as
// ONE warp on 32 CPU threads, so that every answer is checked against the plain-C port (pfo_ents_in_circle) in the CPU
// test suite. The CUDA keywords, intrinsics and warp collectives the header uses are defined as plain C++; every
// collective is a barrier of the warp's 32 threads. The index is built here as k_cell_* builds it (cells in row-major
// order, descending uid inside a cell) and the answer lengths are scanned serially; the device scans them with the
// index's exclusive scan (k_cell_scan or the k_cell_scan_* launches, both on pf_block_excl_scan). This is not a
// product path: nothing in libpfnav.so links or calls it, and it is built only by tests/test_ents_query_emu.py.
#include <math.h>
#include <atomic>
#include <sched.h>
#include <stdlib.h>
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <thread>
#include <vector>
#include "../../include/pfnav.h"

#define __device__
#define __global__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)

struct pf_record {          // pfnav_internal.cuh
    float px, pz, vx, vz, radius;
    uint32_t state_flags;
};
static_assert(sizeof(pf_record) == 24, "pf_record");

struct WarpCtx {
    std::atomic<int> count{0}, gen{0};
    uint32_t xchg[32];
};
static inline void warp_barrier(WarpCtx *w)
{
    const int g = w->gen.load(std::memory_order_acquire);
    if (w->count.fetch_add(1, std::memory_order_acq_rel) == 31) {
        w->count.store(0, std::memory_order_relaxed);
        w->gen.store(g + 1, std::memory_order_release);
        return;
    }
    for (int k = 0; w->gen.load(std::memory_order_acquire) == g; k++)
        if (k > 64) sched_yield();
}
struct emu_dim3 { unsigned x, y, z; };
static thread_local emu_dim3 threadIdx;
static const emu_dim3 blockIdx = {0, 0, 0}, blockDim = {32, 1, 1}, gridDim = {1, 1, 1};
static WarpCtx *g_warp;
static int g_walk = -1;                      // the last walk's way (PF_WALK_TRACE)

static inline void __syncwarp() { warp_barrier(g_warp); }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline int __float2int_rn(float x) { return (int)lrintf(x); }      // the default rounding: to nearest, ties to even
static inline int __shfl_sync(unsigned, int v, int src)
{
    g_warp->xchg[threadIdx.x] = (uint32_t)v;
    warp_barrier(g_warp);
    const int r = (int)g_warp->xchg[src];
    warp_barrier(g_warp);
    return r;
}
static inline unsigned __ballot_sync(unsigned, int p)
{
    g_warp->xchg[threadIdx.x] = p ? 1 : 0;
    warp_barrier(g_warp);
    unsigned r = 0;
    for (int k = 0; k < 32; k++) r |= g_warp->xchg[k] << k;
    warp_barrier(g_warp);
    return r;
}
#define PF_WALK_TRACE(kind, lane) do { if ((lane) == 0) g_walk = (kind); } while (0)

#include "../../permafrost-engine_b200/csrc/pfnav_ents_query_kernel.cuh"

// pos_xz / state_flags: the population's records (uid order) on a chunk_w x chunk_h map at (map_x, map_z); q: nq queries.
// filter_garr: the population holds a GARRISONED entity (what the context's any_garrisoned says).
// Out: offsets[nq + 1] and ids (room for `cap`; returns -1 without writing ids when the total exceeds it), and per query
// raw[i] (the raw cut), walk[i] (-1 no walk, else PF_WALK_TRACE's kind of the count pass) and scr[i] (the garrison
// scratch the write pass used, 0 = none).
extern "C" int emu_ents_query(const float *pos_xz, const uint32_t *state_flags, size_t n, int chunk_w, int chunk_h,
                              float map_x, float map_z, const pfnav_ents_query *q, int nq, int filter_garr, uint32_t *offsets,
                              uint32_t *ids, size_t cap, uint32_t *raw, int32_t *walk, uint32_t *scr)
{
    std::vector<pf_record> rec(n);
    for (size_t i = 0; i < n; i++) rec[i] = {pos_xz[2 * i], pos_xz[2 * i + 1], 0.0f, 0.0f, 0.0f, state_flags[i]};
    // the index geometry of agents_upload_impl (G_Pos_Init + bg_init), and the index k_cell_* builds
    const float W = (float)(chunk_w * 256), H = (float)(chunk_h * 256);
    const float cx = map_x - W / 2.0f, cz = map_z + H / 2.0f;
    GridView g;
    g.origin_x = (int32_t)lrintf((cx - W / 2.0f) * 256.0f);
    g.origin_y = (int32_t)lrintf((cz - H / 2.0f) * 256.0f);
    g.grid_w = max(1, (int)(((uint32_t)((int32_t)lrintf((cx + W / 2.0f) * 256.0f) - g.origin_x) + 4095u) >> 12));
    g.grid_h = max(1, (int)(((uint32_t)((int32_t)lrintf((cz + H / 2.0f) * 256.0f) - g.origin_y) + 4095u) >> 12));
    const size_t ncells = (size_t)g.grid_w * g.grid_h;
    std::vector<uint32_t> start(ncells + 1, 0), fill(ncells, 0), sid(n);
    std::vector<int32_t> six(n), siy(n);
    std::vector<int> cell(n);
    for (size_t i = 0; i < n; i++) {
        cell[i] = cell_of(bg_scale(rec[i].pz), g.origin_y, g.grid_h) * g.grid_w + cell_of(bg_scale(rec[i].px), g.origin_x, g.grid_w);
        start[cell[i] + 1]++;
    }
    for (size_t c = 0; c < ncells; c++) start[c + 1] += start[c];
    for (size_t k = n; k-- > 0;) {
        const uint32_t s = start[cell[k]] + fill[cell[k]]++;
        sid[s] = (uint32_t)k; six[s] = bg_scale(rec[k].px); siy[s] = bg_scale(rec[k].pz);
    }
    g.cell_start = start.data(); g.cell_count = nullptr; g.ix = six.data(); g.iy = siy.data(); g.id = sid.data();

    std::vector<uint32_t> surv(nq), soff(nq + 1, 0);
    static WarpCtx warp;                     // one call at a time
    g_warp = &warp;
    auto run = [&](auto &&body) {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < 32; t++)
            th.emplace_back([&, t]() { threadIdx = {t, 0, 0}; body(t); });
        for (auto &t : th) t.join();
    };
    // count pass, then the scans (serial here)
    run([&](uint32_t lane) {
        for (int i = 0; i < nq; i++) {
            if (lane == 0) g_walk = -1;
            __syncwarp();
            uint32_t r, s;
            eq_count(g, rec.data(), q[i], filter_garr, lane, &r, &s);
            if (lane == 0) { raw[i] = r; surv[i] = s; walk[i] = g_walk; scr[i] = filter_garr && r != s ? r : 0u; }
            __syncwarp();
        }
    });
    offsets[0] = 0;
    for (int i = 0; i < nq; i++) { offsets[i + 1] = offsets[i] + surv[i]; soff[i + 1] = soff[i] + scr[i]; }
    if (offsets[nq] > cap) return -1;
    std::vector<uint32_t> scratch(soff[nq] + 1);
    run([&](uint32_t lane) {
        for (int i = 0; i < nq; i++)
            eq_write(g, rec.data(), q[i], lane, ids + offsets[i], scr[i] ? scratch.data() + soff[i] : nullptr);
    });
    return 0;
}
