// pfnav_scan.cuh -- the CTA exclusive scan and the ordered compaction that the device lists of libpfnav.so are built
// with (sm_90a): the spatial index, the flock member lists, the work list, the event list, the repair representatives,
// the blocker ops and the island ids.
// Needs: <stdint.h>, <algorithm>, the CUDA runtime.
#pragma once

// Exclusive scan of v over the calling CTA (blockDim.x a multiple of 32, <= 1024; every thread calls it).
// warp_tot: blockDim.x / 32 shared T; total: the CTA's sum. Safe to call again in a loop without an extra barrier.
template <typename T> __device__ __forceinline__ T pf_block_excl_scan(T v, T *warp_tot, T &total)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    T x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const T y = __shfl_up_sync(0xFFFFFFFFu, x, o); if (lane >= o) x += y; }
    __syncthreads();                        // the previous call's warps may still be reading warp_tot
    if (lane == 31) warp_tot[wid] = x;
    __syncthreads();
    // every warp scans the warp totals itself: nothing is written back, so two barriers are enough
    const T w = lane < nw ? warp_tot[lane] : T(0);
    T s = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const T y = __shfl_up_sync(0xFFFFFFFFu, s, o); if (lane >= o) s += y; }
    total = __shfl_sync(0xFFFFFFFFu, s, 31);
    return __shfl_sync(0xFFFFFFFFu, s - w, wid) + x - v;
}

// ---- ordered compaction: F::emit(i, slot) for the items i in [lo, hi) with F::keep(i), slots in item order ----
// Block b of nb owns the items [lo + b * per, lo + (b + 1) * per), per a multiple of PF_COMPACT_THREADS, nb <= 1024
// (pf_compact_grid_of). k_compact_count stores every warp's ballot of keep at bal[(i - lo) >> 5] and the block's count
// at part[b]; k_compact_offsets (one CTA) turns part[0 .. nb) into offsets and writes the number kept to *count;
// k_compact_write emits the items of the set ballot bits behind their block's offset, so keep runs once per item.
// Scratch: nb part words and ceil((hi - lo) / 32) ballot words.
#define PF_COMPACT_THREADS 1024

struct pf_compact_grid { int nb, per; };
inline pf_compact_grid pf_compact_grid_of(int n)
{
    const int nb = std::min(1024, (n + PF_COMPACT_THREADS - 1) / PF_COMPACT_THREADS);
    return {nb, nb ? ((n + nb - 1) / nb + PF_COMPACT_THREADS - 1) / PF_COMPACT_THREADS * PF_COMPACT_THREADS : 0};
}

template <typename F>
__global__ void __launch_bounds__(PF_COMPACT_THREADS) k_compact_count(F f, int lo, int hi, int per, uint32_t *__restrict__ bal,
                                                                      uint32_t *__restrict__ part)
{
    __shared__ uint32_t warp_tot[PF_COMPACT_THREADS / 32];
    const int b0 = lo + blockIdx.x * per, b1 = min(b0 + per, hi);
    uint32_t c = 0;
    for (int base = b0; base < b1; base += PF_COMPACT_THREADS) {
        const int i = base + threadIdx.x;
        const bool k = i < b1 && f.keep(i);
        const unsigned m = __ballot_sync(0xFFFFFFFFu, k);
        if ((threadIdx.x & 31) == 0 && i < b1) bal[(i - lo) >> 5] = m;
        c += k;
    }
    uint32_t total;
    pf_block_excl_scan(c, warp_tot, total);
    if (threadIdx.x == 0) part[blockIdx.x] = total;
}

// a template like the other two stages, so that only the translation units that compact compile it
template <typename F>
__global__ void __launch_bounds__(PF_COMPACT_THREADS) k_compact_offsets(uint32_t *__restrict__ part, int nb,
                                                                        uint32_t *__restrict__ count)
{
    __shared__ uint32_t warp_tot[PF_COMPACT_THREADS / 32];
    const uint32_t v = (int)threadIdx.x < nb ? part[threadIdx.x] : 0;
    uint32_t total;
    const uint32_t e = pf_block_excl_scan(v, warp_tot, total);
    if ((int)threadIdx.x < nb) part[threadIdx.x] = e;
    if (threadIdx.x == 0) *count = total;
}

template <typename F>
__global__ void __launch_bounds__(PF_COMPACT_THREADS) k_compact_write(F f, int lo, int hi, int per, const uint32_t *__restrict__ bal,
                                                                      const uint32_t *__restrict__ part)
{
    __shared__ uint32_t warp_tot[PF_COMPACT_THREADS / 32];
    const int b0 = lo + blockIdx.x * per, b1 = min(b0 + per, hi);
    const int wid = threadIdx.x >> 5;
    uint32_t out = part[blockIdx.x];
    for (int base = b0; base < b1; base += PF_COMPACT_THREADS) {
        const unsigned m = base + (wid << 5) < b1 ? bal[((base - lo) >> 5) + wid] : 0u;
        const uint32_t k = (m >> (threadIdx.x & 31)) & 1u;
        uint32_t total;
        const uint32_t slot = out + pf_block_excl_scan(k, warp_tot, total);
        if (k) f.emit(base + threadIdx.x, slot);
        out += total;
    }
}
