// tests/emu/clearpath_emu.cpp -- TEST INFRASTRUCTURE. Runs the device source of ClearPath
// (permafrost-engine_b200/csrc/pfnav_clearpath_kernel.cuh, unmodified) as ONE warp on 32 CPU threads, so that the first
// solve, the one-pass retry emulation with its literal replay, and the two-phase split are checked bit for bit against the
// plain-C port in the CPU test suite. The CUDA keywords, intrinsics and warp collectives the header uses are defined as
// plain C++; every collective is a barrier of the warp's 32 threads. Barrier and exchange state belong to one warp
// instance, so several batches can run at once from different host threads. This is not a product path: nothing in
// libpfnav.so links or calls it, and it is built only by tests/test_clearpath_emu.py (with -ffp-contract=off, the CPU
// counterpart of the TU's -fmad=false).
//
// The block of k_agent_velocity that drives ClearPath (first solve, retry, literal replay, counters) stays inline in the
// kernel (pfnav_agents.cu: as a function it reorders the MODE 2 schedule); emu_solve below restates THAT BLOCK ONLY.
// Everything it calls comes from the header.
#include <math.h>
#include <atomic>
#include <pthread.h>
#include <sched.h>
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <thread>
#include <vector>
#include "../../include/pfnav.h"

#define __device__
#define __forceinline__ inline
#define __align__(n) __attribute__((aligned(n)))

struct float2 { float x, y; };
// a sense-reversing barrier of the warp's 32 threads: spins briefly, then yields (far cheaper than a futex barrier when
// 32 threads share a few cores)
struct WarpCtx {
    std::atomic<int> count{0}, gen{0};
    uint64_t xchg[32];
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
static thread_local WarpCtx *g_warp;

static inline void __syncwarp() { warp_barrier(g_warp); }
static inline float __int_as_float(int v) { float f; memcpy(&f, &v, 4); return f; }
static inline int __float_as_int(float f) { int v; memcpy(&v, &f, 4); return v; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline int __popc(uint32_t v) { return __builtin_popcount(v); }
static inline int __ffs(uint32_t v) { return __builtin_ffs((int)v); }

// every lane publishes a value, then reads the one of lane `src(lane)`
template <class F> static inline uint64_t exchange(uint64_t v, F src)
{
    g_warp->xchg[threadIdx.x] = v;
    warp_barrier(g_warp);
    const int s = src((int)threadIdx.x);
    const uint64_t r = (s >= 0 && s < 32) ? g_warp->xchg[s] : v;
    warp_barrier(g_warp);
    return r;
}
static inline int __shfl_sync(unsigned, int v, int src) { return (int)(uint32_t)exchange((uint32_t)v, [=](int) { return src; }); }
static inline float __shfl_sync(unsigned, float v, int src) { return __int_as_float(__shfl_sync(0u, __float_as_int(v), src)); }
static inline int __shfl_xor_sync(unsigned, int v, int m) { return (int)(uint32_t)exchange((uint32_t)v, [=](int l) { return l ^ m; }); }
static inline float __shfl_xor_sync(unsigned, float v, int m) { return __int_as_float(__shfl_xor_sync(0u, __float_as_int(v), m)); }
static inline unsigned __ballot_sync(unsigned, int p)
{
    g_warp->xchg[threadIdx.x] = p ? 1 : 0;
    warp_barrier(g_warp);
    unsigned r = 0;
    for (int k = 0; k < 32; k++) r |= (unsigned)g_warp->xchg[k] << k;
    warp_barrier(g_warp);
    return r;
}
static inline int __any_sync(unsigned, int p) { return __ballot_sync(0u, p) != 0; }
static inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }

#include "../../permafrost-engine_b200/csrc/pfnav_clearpath_kernel.cuh"

// Restatement of the ClearPath block of k_agent_velocity<MODE> (pfnav_agents.cu, "G_ClearPath_NewVelocity
// (clearpath.c:694)"), MODE 0 or 2; prep is the agent's phase-A record (MODE 2 only). Returns the velocity before
// v2_truncate; n_rays / found / exact: the first solve's ray count and outcome, the one-pass emulation's exact flag.
template <int MODE>
static v2 emu_solve(VelSmem &s, const cp_ent self, const v2 vpref, int ndyn, int nstat, uint32_t lane, const pf_prep *prep,
                    unsigned long long *stats, int &n_rays_out, bool &found_out, bool &exact_out)
{
    v2 new_vel = {0.0f, 0.0f};
    {
        v2 r;
        int n_rays = 0;
        bool found, exact = true;
        if (MODE == 2 && prep->nx != PF_PREP_OVERFLOW)
            found = clearpath_finish(s, self, vpref, ndyn, nstat, lane, prep->xp, (int)prep->nx, r, n_rays);
        else
            found = clearpath_new_velocity(s, self, vpref, ndyn, nstat, lane, r, n_rays);
        n_rays_out = n_rays; found_out = found;
        if (found) new_vel = r;
        else {
            if (lane == 0) { atomicAdd(stats + 0, 1ull); if (ndyn > 0 && nstat > 0) atomicAdd(stats + 1, 1ull); }
            new_vel = clearpath_retry(s, self, vpref, ndyn, nstat, n_rays, lane, exact);
            if (!exact) {
                new_vel = {0.0f, 0.0f};
                unsigned long long solves = 0;
                while (true) {
                    remove_furthest(s, self.pos, ndyn, nstat, lane);
                    if (!(ndyn > 0 && nstat > 0)) break;
                    int nr2;
                    solves++;
                    if (clearpath_new_velocity(s, self, vpref, ndyn, nstat, lane, r, nr2)) { new_vel = r; break; }
                }
                if (lane == 0) { atomicAdd(stats + 2, 1ull); atomicAdd(stats + 3, solves); }
            }
        }
        exact_out = exact;
    }
    return new_vel;
}

static void load_lists(VelSmem &s, const float *dyn5, int ndyn, const float *stat5, int nstat, uint32_t lane)
{
    for (int k = lane; k < ndyn; k += 32) s.dyn[k] = cp_ent{{dyn5[5 * k], dyn5[5 * k + 1]}, {dyn5[5 * k + 2], dyn5[5 * k + 3]}, dyn5[5 * k + 4]};
    for (int k = lane; k < nstat; k += 32) s.stat[k] = cp_ent{{stat5[5 * k], stat5[5 * k + 1]}, {stat5[5 * k + 2], stat5[5 * k + 3]}, stat5[5 * k + 4]};
    __syncwarp();
}

// One case on one warp. mode 0: the single pass (k_agent_velocity<0>); mode 2: phase A (clearpath_collect, as
// k_agent_velocity<1> stores it) into a pf_prep, then phase B (k_agent_velocity<2>) on a shared-memory image that phase A
// did not leave behind. out2: the velocity after v2_truncate(max_len); stats4 += the kernel's counters; info4: {first
// solve found, exact, n_rays, phase A's nx (its raw count, > PF_PREP_XP_CAP = overflow; -1 in mode 0)}.
static void warp_case(VelSmem &s, pf_prep &prep, const float *self5, const float *vpref2, const float *dyn5, int ndyn,
                      const float *stat5, int nstat, int mode, float max_len, float *out2, unsigned long long *stats4,
                      int *info4, uint32_t lane)
{
    const cp_ent self = {{self5[0], self5[1]}, {self5[2], self5[3]}, self5[4]};
    const v2 vpref = {vpref2[0], vpref2[1]};
    int n_rays = 0, nx = -1;
    bool found = false, exact = true;
    v2 v;
    if (lane == 0) memset(&s, 0xA5, sizeof(s));
    __syncwarp();
    load_lists(s, dyn5, ndyn, stat5, nstat, lane);
    if (mode == 2) {
        nx = clearpath_collect(s, self, ndyn, nstat, lane, prep.xp);
        if (lane == 0) {
            prep.ndyn = (uint32_t)ndyn; prep.nstat = (uint32_t)nstat;
            prep.nx = nx > PF_PREP_XP_CAP ? PF_PREP_OVERFLOW : (uint32_t)nx;
        }
        __syncwarp();
        if (lane == 0) memset(&s, 0x5A, sizeof(s));
        __syncwarp();
        load_lists(s, dyn5, ndyn, stat5, nstat, lane);
        v = emu_solve<2>(s, self, vpref, ndyn, nstat, lane, &prep, stats4, n_rays, found, exact);
    } else {
        v = emu_solve<0>(s, self, vpref, ndyn, nstat, lane, nullptr, stats4, n_rays, found, exact);
    }
    v = v2_truncate(v, max_len);
    if (lane == 0) {
        out2[0] = v.x; out2[1] = v.z;
        info4[0] = found; info4[1] = exact; info4[2] = n_rays; info4[3] = nx;
    }
    __syncwarp();
}

// n cases on one warp of 32 threads; dyn5 / stat5: [n][32][5] {px, pz, vx, vz, radius}; stats4 / info4: [n][4]
extern "C" int emu_clearpath_batch(int n, const float *self5, const float *vpref2, const float *dyn5, const int *ndyn,
                                   const float *stat5, const int *nstat, int mode, const float *max_len, float *out2,
                                   unsigned long long *stats4, int *info4)
{
    if (mode != 0 && mode != 2) return -1;
    for (int i = 0; i < n; i++)
        if (ndyn[i] < 0 || ndyn[i] > PFNAV_MAX_NEIGHBOURS || nstat[i] < 0 || nstat[i] > PFNAV_MAX_NEIGHBOURS) return -1;
    WarpCtx ctx;
    VelSmem *s = (VelSmem *)aligned_alloc(16, (sizeof(VelSmem) + 15) / 16 * 16);
    pf_prep *prep = (pf_prep *)aligned_alloc(16, (sizeof(pf_prep) + 15) / 16 * 16);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < 32; t++)
        th.emplace_back([&, t]() {
            threadIdx = {t, 0, 0};
            g_warp = &ctx;
            for (int i = 0; i < n; i++)
                warp_case(*s, *prep, self5 + 5 * i, vpref2 + 2 * i, dyn5 + (size_t)160 * i, ndyn[i], stat5 + (size_t)160 * i,
                          nstat[i], mode, max_len[i], out2 + 2 * i, stats4 + 4 * i, info4 + 4 * i, t);
        });
    for (auto &t : th) t.join();
    free(s); free(prep);
    return 0;
}

// the single-case form: dyn5 / stat5 hold ndyn / nstat records; stats8: the kernel's counters are added to [0..3]
extern "C" int emu_clearpath(const float *self5, const float *vpref2, const float *dyn5, int ndyn, const float *stat5,
                             int nstat, int mode, float max_len, float *out2, unsigned long long *stats8, int *info)
{
    if (ndyn < 0 || ndyn > PFNAV_MAX_NEIGHBOURS || nstat < 0 || nstat > PFNAV_MAX_NEIGHBOURS) return -1;
    float d[160] = {0}, st[160] = {0};
    memcpy(d, dyn5, sizeof(float) * 5 * ndyn);
    memcpy(st, stat5, sizeof(float) * 5 * nstat);
    unsigned long long c[4] = {0, 0, 0, 0};
    const int r = emu_clearpath_batch(1, self5, vpref2, d, &ndyn, st, &nstat, mode, &max_len, out2, c, info);
    for (int k = 0; k < 4; k++) stats8[k] += c[k];
    return r;
}

// ---- single-thread entries (no warp collectives) ----
// vo_contains on a table of ONE obstacle: rays4 = {px, pz, dx, dz} of its left (even) and right (odd) ray
extern "C" void emu_vo_contains(const float *rays4, const float *pts2, long n, uint8_t *out)
{
    static thread_local VelSmem s;
    for (int k = 0; k < 2; k++) {
        s.rpx[k] = rays4[4 * k]; s.rpz[k] = rays4[4 * k + 1]; s.rdx[k] = rays4[4 * k + 2]; s.rdz[k] = rays4[4 * k + 3];
        s.rsl[k] = line_slope(v2{s.rdx[k], s.rdz[k]});
    }
    for (long i = 0; i < n; i++) out[i] = vo_contains(s, 0, v2{pts2[2 * i], pts2[2 * i + 1]});
}

extern "C" void emu_quot_lt0(const float *a, const float *b, long n, uint8_t *out)
{
    for (long i = 0; i < n; i++) out[i] = quot_lt0(a[i], b[i]);
}

// line_isect_s with the slopes line_slope gives: lines4 = [n][2][4] {px, pz, dx, dz}; out3 = {ok, x, z}
extern "C" void emu_line_isect_s(const float *lines4, long n, float *out3)
{
    for (long i = 0; i < n; i++) {
        const float *l = lines4 + 8 * i;
        v2 p = {0.0f, 0.0f};
        const bool ok = line_isect_s(v2{l[0], l[1]}, line_slope(v2{l[2], l[3]}), v2{l[4], l[5]}, line_slope(v2{l[6], l[7]}), p);
        out3[3 * i] = ok ? 1.0f : 0.0f; out3[3 * i + 1] = p.x; out3[3 * i + 2] = p.z;
    }
}

// retry_better(T, dist, p, best) on a best {bT, bdist, bid, bp}: out2 = {returned better, tie flag afterwards}
extern "C" void emu_retry_better(int T, float dist, float px, float pz, int bT, float bdist, int bid, float bpx, float bpz, int *out2)
{
    retry_best b;
    b.T = bT; b.dist = bdist; b.id = bid; b.p = v2{bpx, bpz}; b.tie = 0;
    out2[0] = retry_better(T, dist, v2{px, pz}, b);
    out2[1] = b.tie;
}
