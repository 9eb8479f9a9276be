// pfnav_digest.cu -- pfnav_state_digest and pfnav_state_digest_read: the state digests of pfnav_digest_host.h computed on
// the device (sm_90a) and read back as a few dozen bytes. The job forms (pfnav_group_state_digest, pfnav_mgpu_state_digest)
// are in pfnav_mgpu.cu.
//
// Every kernel adds wrapping 64-bit sums into the context's digest record with atomics, so the bits do not depend on the
// launch configuration or the order in which CTAs finish:
//   k_digest_rows     population and block array: grid-stride over the own uids, one row per thread. The row's 16-byte
//                     words are read straight from each table in the order pf_ckpt_word_source gives (the checkpoint
//                     header owns the row layout) and chained in registers. A warp's 32 uids lie in one block
//                     (block_log2 >= 6): a warp reduce, then one atomic per (CTA, block) and one per CTA for the total.
//   k_digest_records  records: grid-stride over the whole record column, one record per thread, one atomic per CTA.
//   k_digest_pool     the pool's device sum: one CTA per slot (grid-stride, as k_pool_pack), its 8 KB of flow and LOS bytes
//                     when its `has` byte is set, and its device touch stamp; one atomic per CTA.
//   k_map_digest      (pfnav_pool.cu) the committed map's block sum.
//   k_digest_finish   one thread: folds in the parts the host holds -- the flock chain of the flock table pfnav_agents_save
//                     writes, the map digest's geometry and enemy table, the chain over the pool's host bookkeeping.
#include "pfnav_internal.cuh"
#include <string.h>

enum { DG_POP = 0, DG_FLOCKS = 1, DG_REC = 2, DG_MAP = 3, DG_POOL = 4 };
#define DG_THREADS 256

// what k_digest_finish folds in, taken on the host at the call
struct pf_digest_fin {
    uint64_t flocks, pool_host;
    int nlayers, chunk_w, chunk_h;
    float map_x, map_z;
    uint16_t enemies[16];
};

__device__ __forceinline__ uint64_t dg_lo(const uint4 &v) { return (uint64_t)v.x | (uint64_t)v.y << 32; }
__device__ __forceinline__ uint64_t dg_hi(const uint4 &v) { return (uint64_t)v.z | (uint64_t)v.w << 32; }

__device__ __forceinline__ uint64_t dg_warp_sum(uint64_t v)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

// the sum of every thread's v over the CTA (DG_THREADS threads), in thread 0; called by the whole CTA
__device__ __forceinline__ uint64_t dg_cta_sum(uint64_t v, uint64_t *ws)
{
    v = dg_warp_sum(v);
    if (pf_lane() == 0) ws[threadIdx.x >> 5] = v;
    __syncthreads();
    uint64_t t = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < DG_THREADS / 32; w++) t += ws[w];
    __syncthreads();
    return t;
}

__global__ void __launch_bounds__(DG_THREADS) k_digest_rows(pf_ckpt_src src, pf_ckpt_row row, uint32_t tables, uint32_t lo,
                                                            uint32_t hi, int k, unsigned long long *__restrict__ total,
                                                            unsigned long long *__restrict__ blocks)
{
    __shared__ uint64_t ws[DG_THREADS / 32];
    const uint32_t step = gridDim.x * DG_THREADS;
    // CTAs start on multiples of DG_THREADS, so every warp's 32 uids share one block
    for (uint32_t base = (lo & ~(uint32_t)(DG_THREADS - 1)) + blockIdx.x * DG_THREADS; base < hi; base += step) {
        const uint32_t u = base + threadIdx.x;
        uint64_t h = 0;
        if (u >= lo && u < hi) {
            h = pf_digest_row_begin(u, tables);
            for (uint32_t q = 0; q < row.words; q++) {
                int t;
                uint32_t w;
                pf_ckpt_word_source(row, tables, q, &t, &w);
                // selects, not an indexed parameter array: a dynamic index would put src in local memory
                const uint4 *b = t == 0 ? src.p[0] : t == 1 ? src.p[1] : t == 2 ? src.p[2] : t == 3 ? src.p[3] : src.p[4];
                const uint32_t n = t == 0 ? src.words[0] : t == 1 ? src.words[1] : t == 2 ? src.words[2] : t == 3 ? src.words[3] : src.words[4];
                const uint4 v = __ldg(b + (size_t)u * n + w);
                h = pf_digest_word(h, dg_lo(v), dg_hi(v));
            }
        }
        h = dg_warp_sum(h);
        if (pf_lane() == 0) ws[threadIdx.x >> 5] = h;
        __syncthreads();
        const uint32_t wi = threadIdx.x;
        if (wi < DG_THREADS / 32 && base + 32 * wi < hi) {
            // the first warp of each run of warps in one block adds the run's sum
            const uint32_t bw = (base + 32 * wi) >> k;
            if (wi == 0 || ((base + 32 * (wi - 1)) >> k) != bw) {
                uint64_t s = 0;
                for (uint32_t j = wi; j < DG_THREADS / 32 && base + 32 * j < hi && ((base + 32 * j) >> k) == bw; j++) s += ws[j];
                if (s) atomicAdd(blocks + bw, (unsigned long long)s);
            }
            if (wi == 0) {
                uint64_t s = 0;
                for (int j = 0; j < DG_THREADS / 32; j++) s += ws[j];
                if (s) atomicAdd(total, (unsigned long long)s);
            }
        }
        __syncthreads();
    }
}

// pf_record is 24 bytes, 8-byte aligned: three 8-byte words per uid
__global__ void __launch_bounds__(DG_THREADS) k_digest_records(const uint2 *__restrict__ rec, uint32_t n,
                                                               unsigned long long *__restrict__ out)
{
    __shared__ uint64_t ws[DG_THREADS / 32];
    uint64_t s = 0;
    for (uint32_t u = blockIdx.x * DG_THREADS + threadIdx.x; u < n; u += gridDim.x * DG_THREADS) {
        const uint2 a = __ldg(rec + 3 * (size_t)u), b = __ldg(rec + 3 * (size_t)u + 1), c = __ldg(rec + 3 * (size_t)u + 2);
        s += pf_digest_record(u, (uint64_t)a.x | (uint64_t)a.y << 32, (uint64_t)b.x | (uint64_t)b.y << 32,
                              (uint64_t)c.x | (uint64_t)c.y << 32);
    }
    s = dg_cta_sum(s, ws);
    if (threadIdx.x == 0 && s) atomicAdd(out, (unsigned long long)s);
}

__global__ void __launch_bounds__(DG_THREADS) k_digest_pool(const uint4 *__restrict__ flow, const uint4 *__restrict__ los,
                                                            const uint8_t *__restrict__ has, const uint32_t *__restrict__ touch,
                                                            int max, unsigned long long *__restrict__ out)
{
    __shared__ uint64_t ws[DG_THREADS / 32];
    uint64_t acc = 0;                         // thread 0: this CTA's slot terms
    for (int s = blockIdx.x; s < max; s += gridDim.x) {
        if (has[s]) {                         // the same for the whole CTA
            const size_t at = (size_t)s * 256;
            uint64_t v = 0;
            for (int w = threadIdx.x; w < 512; w += DG_THREADS) {
                const uint4 x = w < 256 ? __ldg(flow + at + w) : __ldg(los + at + w - 256);
                v += pf_digest_field_word((uint32_t)w, dg_lo(x), dg_hi(x));
            }
            v = dg_cta_sum(v, ws);
            if (threadIdx.x == 0) acc += pf_digest_slot((uint32_t)s, v);
        }
        if (threadIdx.x == 0) acc += pf_digest_touch((uint32_t)s, touch[s]);
    }
    if (threadIdx.x == 0 && acc) atomicAdd(out, (unsigned long long)acc);
}

__global__ void k_digest_finish(unsigned long long *rec, uint32_t what, pf_digest_fin f)
{
    if (what & PFNAV_DIGEST_FLOCKS) rec[DG_FLOCKS] = f.flocks;
    if (what & PFNAV_DIGEST_MAP) rec[DG_MAP] = pf_digest_fold(rec[DG_MAP], f.nlayers, f.chunk_w, f.chunk_h, f.map_x, f.map_z, f.enemies);
    if (what & PFNAV_DIGEST_POOL) rec[DG_POOL] = pf_digest_step(f.pool_host, rec[DG_POOL]);
}

void pf_digest_free(pfnav_ctx *ctx)
{
    if (ctx->digest_done) cudaEventDestroy(ctx->digest_done);
    if (ctx->h_digest) cudaFreeHost(ctx->h_digest);
    ctx->digest_done = nullptr; ctx->h_digest = nullptr; ctx->h_digest_cap = 0; ctx->digest_valid = false;
}

int pf_digest_check(pfnav_ctx *ctx, uint32_t what, int block_log2)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(what && !(what & ~PFNAV_DIGEST_ALL), "what: no component, or unknown component bits");
    if (what & PFNAV_DIGEST_POPULATION)
        PF_ARG(block_log2 >= PF_DIGEST_BLOCK_MIN && block_log2 <= PF_DIGEST_BLOCK_MAX, "block_log2 outside 6..20");
    if (what & (PFNAV_DIGEST_POPULATION | PFNAV_DIGEST_FLOCKS | PFNAV_DIGEST_RECORDS))
        PF_ARG(ctx->d_agents, "no population uploaded");
    if (what & PFNAV_DIGEST_MAP) PF_ARG(ctx->d_cost, "map not created");
    if (what & PFNAV_DIGEST_POOL) PF_ARG(ctx->pool.d_slot, "pool not created");
    return PFNAV_OK;
}

// the CTAs of a grid-stride pass over n items: at most 8 resident CTAs per SM, the count the items need below that
static int dg_grid(const pfnav_ctx *ctx, size_t n)
{
    return (int)std::max<size_t>(1, std::min<size_t>((n + DG_THREADS - 1) / DG_THREADS, (size_t)ctx->sm_count * 8));
}

int pf_digest_launch(pfnav_ctx *ctx, uint32_t what, int block_log2, cudaStream_t st, int world, int rank)
{
    PF_CUDA(cudaSetDevice(ctx->device));
    const bool pop = what & PFNAV_DIGEST_POPULATION;
    const size_t nblocks = pop ? pf_digest_nblocks(ctx->n_agents, block_log2) : 0;
    const size_t nrec = (size_t)world * PF_DIGEST_REC, words = nrec + nblocks;
    // the previous digest's copy may still read the device buffer and write the pinned one
    if (ctx->digest_valid) PF_CUDA(cudaStreamWaitEvent(st, ctx->digest_done, 0));
    ctx->digest_valid = false;
    if (int rc = ctx->d_digest.reserve(words)) return rc;
    if (ctx->h_digest_cap < words) {
        if (ctx->digest_done) PF_CUDA(cudaEventSynchronize(ctx->digest_done));
        const size_t want = std::max(words, 2 * ctx->h_digest_cap);
        if (ctx->h_digest) PF_CUDA(cudaFreeHost(ctx->h_digest));
        ctx->h_digest = nullptr; ctx->h_digest_cap = 0;
        PF_CUDA(cudaMallocHost(&ctx->h_digest, want * sizeof(uint64_t)));
        ctx->h_digest_cap = want;
    }
    if (!ctx->digest_done) PF_CUDA(cudaEventCreateWithFlags(&ctx->digest_done, cudaEventDisableTiming));
    if (what & PFNAV_DIGEST_POOL) {
        // ordered as the pool's other readers: after the forked field work and a pending clear
        PF_CUDA(pf_fields_join(ctx, st));
        PF_CUDA(pf_pool_refresh(ctx, st));
    }
    unsigned long long *d = ctx->d_digest.p, *rec = d + (size_t)rank * PF_DIGEST_REC, *blocks = d + nrec;
    PF_CUDA(cudaMemsetAsync(d, 0, words * sizeof(uint64_t), st));
    const uint32_t tables = pf_ckpt_tables(ctx);
    const size_t lo = ctx->shard_lo, hi = ctx->shard_hi;
    if (pop && hi > lo) {
        k_digest_rows<<<dg_grid(ctx, hi - (lo & ~(size_t)(DG_THREADS - 1))), DG_THREADS, 0, st>>>(
            pf_ckpt_sources(ctx), pf_ckpt_row_of(tables), tables, (uint32_t)lo, (uint32_t)hi, block_log2, rec + DG_POP, blocks);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    if ((what & PFNAV_DIGEST_RECORDS) && ctx->n_agents) {
        k_digest_records<<<dg_grid(ctx, ctx->n_agents), DG_THREADS, 0, st>>>((const uint2 *)ctx->d_records.p,
                                                                             (uint32_t)ctx->n_agents, rec + DG_REC);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    if (what & PFNAV_DIGEST_MAP)
        if (int rc = pf_map_digest_launch(ctx, st, rec + DG_MAP)) return rc;
    pf_digest_fin fin;
    memset(&fin, 0, sizeof(fin));
    if (what & PFNAV_DIGEST_POOL) {
        const pf_pool &P = ctx->pool;
        // the host part of the segment pfnav_pool_save would write (its map digest word is not hashed)
        std::vector<int32_t> stored;
        const pf_pool_layout L = pf_pool_seg_plan(P, ctx->aux, stored);
        std::vector<uint8_t> head(L.dtouch);
        pf_pool_seg_write(P, ctx->aux, {ctx->chunk_w, ctx->chunk_h, ctx->nlayers, P.ndests, P.max, 0}, ctx->tick_no, stored, L,
                          head.data());
        fin.pool_host = pf_digest_pool_host(head.data(), L.dtouch);
        k_digest_pool<<<(unsigned)std::max(1, std::min(P.max, ctx->sm_count * 8)), DG_THREADS, 0, st>>>(
            (const uint4 *)P.d_flow, (const uint4 *)P.d_los, P.d_has, P.d_touch, P.max, rec + DG_POOL);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    if (what & PFNAV_DIGEST_FLOCKS) fin.flocks = pf_digest_flocks(ctx->h_flocks.data(), ctx->h_flocks.size());
    fin.nlayers = ctx->nlayers; fin.chunk_w = ctx->chunk_w; fin.chunk_h = ctx->chunk_h;
    fin.map_x = ctx->map_x; fin.map_z = ctx->map_z;
    memcpy(fin.enemies, ctx->enemies, sizeof(fin.enemies));
    k_digest_finish<<<1, 1, 0, st>>>(rec, what, fin);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    pfnav_digest &I = ctx->digest_info;
    memset(&I, 0, sizeof(I));
    I.what = what; I.block_log2 = pop ? block_log2 : 0; I.tables = tables; I.hz = ctx->hz;
    I.n_total = ctx->n_agents; I.lo = lo; I.hi = hi; I.nblocks = nblocks;
    ctx->digest_world = world; ctx->digest_rank = rank;
    return PFNAV_OK;
}

int pf_digest_finish(pfnav_ctx *ctx, cudaStream_t st)
{
    const size_t words = (size_t)ctx->digest_world * PF_DIGEST_REC + ctx->digest_info.nblocks;
    PF_CUDA(cudaMemcpyAsync(ctx->h_digest, ctx->d_digest.p, words * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaEventRecord(ctx->digest_done, st));
    ctx->digest_valid = true;
    return PFNAV_OK;
}

extern "C" int pfnav_state_digest(pfnav_ctx *ctx, uint32_t what, int block_log2, void *stream)
{
    if (int rc = pf_digest_check(ctx, what, block_log2)) return rc;
    cudaStream_t st = pf_stream(ctx, stream);
    if (int rc = pf_digest_launch(ctx, what, block_log2, st, 1, 0)) return rc;
    return pf_digest_finish(ctx, st);
}

extern "C" int pfnav_state_digest_read(pfnav_ctx *ctx, pfnav_digest *out, uint64_t *blocks, size_t cap, size_t *nblocks)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(out, "out == NULL");
    PF_ARG(!blocks || nblocks, "nblocks == NULL with a block array");
    if (!ctx->digest_valid) {
        pfnav_set_error("pfnav_state_digest_read: no digest was queued (pfnav_state_digest / pfnav_mgpu_state_digest)");
        return PFNAV_ERR_STATE;
    }
    const pfnav_digest &I = ctx->digest_info;
    if (nblocks) *nblocks = (size_t)I.nblocks;
    if (blocks && cap < I.nblocks) {
        pfnav_set_error("pfnav_state_digest_read: the block array holds %llu entries, cap %zu", (unsigned long long)I.nblocks, cap);
        return PFNAV_ERR_NOMEM;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaEventSynchronize(ctx->digest_done));
    const int world = ctx->digest_world;
    const uint64_t *h = ctx->h_digest, *own = h + (size_t)ctx->digest_rank * PF_DIGEST_REC;
    pfnav_digest d = I;
    d.population = own[DG_POP]; d.flocks = own[DG_FLOCKS]; d.records = own[DG_REC]; d.map = own[DG_MAP]; d.pool = own[DG_POOL];
    if (world > 1) {
        // an NCCL job's records: the population summed, the replicated components rank 0's with the ranks that differ
        d.population = 0;
        for (int r = 0; r < world; r++) {
            const uint64_t *x = h + (size_t)r * PF_DIGEST_REC, bit = 1ull << std::min(r, 63);
            d.population += x[DG_POP];
            if (x[DG_FLOCKS] != h[DG_FLOCKS]) d.differ_flocks |= bit;
            if (x[DG_REC] != h[DG_REC]) d.differ_records |= bit;
            if (x[DG_MAP] != h[DG_MAP]) d.differ_map |= bit;
        }
        d.flocks = h[DG_FLOCKS]; d.records = h[DG_REC]; d.map = h[DG_MAP];
    }
    if (blocks && I.nblocks) memcpy(blocks, h + (size_t)world * PF_DIGEST_REC, (size_t)I.nblocks * sizeof(uint64_t));
    *out = d;
    return PFNAV_OK;
}
