// pfnav_inputs.cu -- the engine's inputs beyond point seeking as deltas on the device-resident tables (sm_90a).
//
// pfnav_agents_input_deltas writes fields of the movestate_ext table and whole formation records for a subset of the
// population: pfnav_inputs_host.h validates the records and folds those of one uid into one record, which goes through
// the request staging, and k_apply_input_deltas writes them with one thread per folded record. A member of a multi-GPU
// job takes the job's whole batch (pf_input_job_check / pf_input_job_apply, for pfnav_mgpu.cu) and writes the records of
// its own uids.
#include "pfnav_internal.cuh"
#include <string.h>

static_assert(sizeof(pfnav_input_delta) == 128, "pfnav_input_delta must be 128 bytes");
static_assert(offsetof(pfnav_input_delta, formation) == 64, "pfnav_input_delta.formation at offset 64");

// One thread per folded record (one per uid). The 64-byte ext record is read and written in four 16-byte accesses
// around pf_input_apply; the formation record is stored whole. The host refuses the ext bits without an ext table and
// creates the formation table before a FORMATION record, so the pointers are valid when used.
__global__ void __launch_bounds__(128) k_apply_input_deltas(const pfnav_input_delta *__restrict__ deltas, int n,
                                                            pfnav_movestate_ext *__restrict__ exts,
                                                            pfnav_formation_in *__restrict__ forms)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    union { pfnav_input_delta r; uint4 v[8]; } d;
    const uint4 *src = reinterpret_cast<const uint4 *>(deltas + i);
#pragma unroll
    for (int k = 0; k < 8; k++) d.v[k] = src[k];
    const uint32_t uid = d.r.uid, mask = d.r.mask;
    union { pfnav_movestate_ext e; uint4 v[4]; } x;
    union { pfnav_formation_in f; uint4 v[4]; } f;
    uint4 *ext = reinterpret_cast<uint4 *>(exts + uid);
    if (mask & PF_INPUT_EXT) {
#pragma unroll
        for (int k = 0; k < 4; k++) x.v[k] = ext[k];
    }
    pf_input_apply(&x.e, &f.f, d.r);
    if (mask & PF_INPUT_EXT) {
#pragma unroll
        for (int k = 0; k < 4; k++) ext[k] = x.v[k];
    }
    if (mask & PFNAV_INPUT_FORMATION) {
        uint4 *form = reinterpret_cast<uint4 *>(forms + uid);
#pragma unroll
        for (int k = 0; k < 4; k++) form[k] = f.v[k];
    }
}

// Everything after validation, on `st`: the formation table when the batch needs one that does not exist (as
// pfnav_agents_upload_formation of all-zero records leaves it), then the folded records through the request staging.
static int input_apply(pfnav_ctx *ctx, cudaStream_t st, const std::vector<pfnav_input_delta> &merged, bool any_form)
{
    int rc;
    if (any_form && !ctx->d_formation) {
        if ((rc = ctx->d_formation.reserve(ctx->n_agents))) return rc;
        PF_CUDA(cudaMemsetAsync(ctx->d_formation, 0, ctx->n_agents * sizeof(pfnav_formation_in), st));
    }
    if (merged.empty()) return PFNAV_OK;
    const size_t bytes = merged.size() * sizeof(pfnav_input_delta);
    pf_stage S;
    if ((rc = pf_stage_begin(ctx, st, bytes, bytes, false, &S))) return rc;
    memcpy(S.host, merged.data(), bytes);
    if ((rc = pf_stage_upload(ctx, st, S, bytes))) return rc;
    k_apply_input_deltas<<<((int)merged.size() + 127) / 128, 128, 0, st>>>((const pfnav_input_delta *)S.dev, (int)merged.size(),
                                                                          ctx->d_ms_ext, ctx->d_formation);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return pf_stage_done(ctx, st);
}

extern "C" int pfnav_agents_input_deltas(pfnav_ctx *ctx, const pfnav_input_delta *d, size_t n, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_agents, "agents not uploaded");
    if (ctx->mgpu || ctx->shard_lo > 0 || ctx->shard_hi < ctx->n_agents) {
        pfnav_set_error("pfnav_agents_input_deltas: the context is part of a multi-GPU job (pfnav_mgpu_input_deltas / "
                        "pfnav_group_input_deltas keep the members' sets of tables equal)");
        return PFNAV_ERR_STATE;
    }
    PF_ARG(d || n == 0, "d == NULL");
    PF_ARG(n < (1u << 31), "n");
    const pf_input_limits L = {ctx->shard_lo, ctx->shard_hi, ctx->d_ms_ext != nullptr};
    std::vector<pfnav_input_delta> merged;
    const char *err = pf_input_merge(d, n, L, merged);
    PF_ARG(!err, err);
    if (merged.empty()) return PFNAV_OK;
    bool any_form = false;
    for (const pfnav_input_delta &m : merged) any_form |= (m.mask & PFNAV_INPUT_FORMATION) != 0;
    PF_CUDA(cudaSetDevice(ctx->device));
    return input_apply(ctx, pf_stream(ctx, stream), merged, any_form);
}

int pf_input_job_check(pfnav_ctx *ctx, const pfnav_input_delta *d, size_t n, pf_input_job &J)
{
    PF_ARG(ctx->d_agents, "agents not uploaded");
    PF_ARG(d || n == 0, "d == NULL");
    PF_ARG(n < (1u << 31), "n");
    const pf_input_limits L = {0, ctx->n_agents, ctx->d_ms_ext != nullptr};
    const char *err = pf_input_job_plan(d, n, L, ctx->shard_lo, ctx->shard_hi, J.own, J.any_form);
    PF_ARG(!err, err);
    return PFNAV_OK;
}

int pf_input_job_apply(pfnav_ctx *ctx, const pf_input_job &J, cudaStream_t st)
{
    return input_apply(ctx, st, J.own, J.any_form);
}

extern "C" int pfnav_agents_read_formation(pfnav_ctx *ctx, pfnav_formation_in *out, size_t maxout)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_agents && ctx->d_formation, "no formation table");
    PF_ARG(out || maxout == 0, "out == NULL");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());
    const size_t n = std::min(maxout, ctx->shard_hi - ctx->shard_lo);       // this context's own entity range
    if (n) PF_CUDA(cudaMemcpy(out, ctx->d_formation + ctx->shard_lo, n * sizeof(pfnav_formation_in), cudaMemcpyDeviceToHost));
    return PFNAV_OK;
}
