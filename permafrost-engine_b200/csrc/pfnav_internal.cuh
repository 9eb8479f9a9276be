// pfnav_internal.cuh -- shared declarations of libpfnav.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <algorithm>
#include <chrono>
#include <memory>
#include <set>
#include <string>
#include <utility>
#include <vector>
#include "../../include/pfnav.h"
#include "pfnav_pool_host.h"
#include "pfnav_commands_host.h"
#include "pfnav_inputs_host.h"
#include "pfnav_waves_host.h"
#include "pfnav_resident_host.h"
#include "pfnav_checkpoint_host.h"
#include "pfnav_digest_host.h"

#define PFNAV_VERSION 100

#define PF_CUDA(call)                                                                       \
    do {                                                                                    \
        cudaError_t _e = (call);                                                            \
        if (_e != cudaSuccess) {                                                            \
            pfnav_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,                   \
                            cudaGetErrorString(_e));                                        \
            return PFNAV_ERR_CUDA;                                                          \
        }                                                                                   \
    } while (0)

#define PF_NEED_DEVICE(ctx)                                                                         \
    do {                                                                                            \
        if ((ctx)->device < 0) {                                                                    \
            pfnav_set_error("%s: host-only context has no compute path (no CPU fallback)", __func__); \
            return PFNAV_ERR_NO_DEVICE;                                                             \
        }                                                                                           \
    } while (0)

#define PF_ARG(cond, msg)                                                                   \
    do {                                                                                    \
        if (!(cond)) {                                                                      \
            pfnav_set_error("%s:%d: bad argument: %s", __FILE__, __LINE__, msg);            \
            return PFNAV_ERR_ARG;                                                           \
        }                                                                                   \
    } while (0)

// A device array that grows on demand; it owns its pointer and its capacity in elements. reserve(n) keeps the array when
// it holds n elements. Otherwise it waits for the current device and frees the array, if there is one (a launch still in
// flight may read it), then allocates max(n, 2 * capacity) elements (the first allocation is exact); the old content is
// gone. A failed allocation leaves (nullptr, 0) and returns PFNAV_ERR_NOMEM. *grew, when given, tells whether the array
// was reallocated. A pointer stays null until the first reserve, so an optional input can use null as "absent". The
// owner is destroyed after cudaSetDevice of its device.
template <typename T>
struct pf_dbuf {
    T *p = nullptr;
    size_t cap = 0;
    pf_dbuf() = default;
    pf_dbuf(const pf_dbuf &) = delete;
    pf_dbuf &operator=(const pf_dbuf &) = delete;
    ~pf_dbuf() { release(); }
    operator T *() const { return p; }
    void release()
    {
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
    }
    int reserve(size_t n, bool *grew = nullptr)
    {
        if (grew) *grew = false;
        if (n <= cap) return PFNAV_OK;
        const size_t want = std::max(n, 2 * cap);
        if (p) {
            PF_CUDA(cudaDeviceSynchronize());
            release();
        }
        if (cudaMalloc(&p, want * sizeof(T)) != cudaSuccess) {
            cudaGetLastError();
            p = nullptr;
            pfnav_set_error("cudaMalloc of %zu bytes failed", want * sizeof(T));
            return PFNAV_ERR_NOMEM;
        }
        cap = want;
        if (grew) *grew = true;
        return PFNAV_OK;
    }
};
// Reserve n elements in every buffer of a group that shares one length. If an allocation fails the whole group is
// released, so a group is either complete or empty.
template <typename... B>
static int pf_dbuf_reserve_all(size_t n, B &...bufs)
{
    int rc = PFNAV_OK;
    ((rc = rc ? rc : bufs.reserve(n)), ...);
    if (rc) (bufs.release(), ...);
    return rc;
}

// one used (flock, layer) pair of the arrival constants and its flock's target
struct pf_arrival_pair { int32_t flock, layer; float tx, tz; };

// 24-byte neighbour record: exactly what one agent needs to know about another
// (SURVEY.md 8e). This is also the unit of the per-tick NCCL all-gather.
struct __align__(8) pf_record {
    float    px, pz;
    float    vx, vz;
    float    radius;
    uint32_t state_flags;     // state << 24 | (flags & 0xFFFFFF)
};
static_assert(sizeof(pf_record) == 24, "pf_record must be 24 bytes");
struct pf_prep;                          // pfnav_clearpath_kernel.cuh

struct pfnav_ctx {
    int device = 0;
    int sm_count = 0;
    uint64_t launches = 0;
    bool use_tma = true;
    bool tma_ok = false;

    // ---- map state (row-major images per layer: [layer][H*64][W*64]) ----
    int chunk_w = 0, chunk_h = 0, nlayers = 0;
    int W64 = 0, H64 = 0;
    float map_x = 0.f, map_z = 0.f;
    uint8_t  *d_cost = nullptr;      // u8
    uint16_t *d_blk = nullptr;       // u16 blockers refcounts
    uint16_t *d_liid = nullptr;      // u16 local islands
    // per-faction blocker refcounts (chunk->factions, nav_data.h): host counts per layer (allocated on first
    // use, [chunk][15][4096]) and a device bit mask per tile (bit f <=> factions[f] > 0) for the "attacking"
    // passability rule field_tile_passable_no_enemies (field.c:179)
    uint16_t *d_fmask = nullptr;
    std::vector<std::vector<uint8_t>> h_fac;     // [layer]
    std::vector<uint16_t> h_fmask;               // [layer][chunk][4096]
    uint16_t enemies[16] = {0};                  // enemies[f] = factions at war with f (G_GetEnemyFactions)
    bool faction_enabled = false;
    int req_faction = 0xF;                       // faction of the path request being planned (n_request_path's faction_id)
    uint8_t  *d_unit = nullptr;      // [layer][chunk] 1 if every passable cost in the chunk == 1
    std::vector<uint8_t> h_unit;     // host mirror
    CUtensorMap tmap_cost, tmap_blk; // rank-3 {x, y, layer}, box 64x64x1
    pf_dbuf<uint8_t> d_stage;                                  // upload staging
    pf_dbuf<unsigned long long> d_los_trace; size_t los_trace_n = 0; bool los_trace_on = false;   // 4 words per request
    int los_variant = 2;
    pf_dbuf<int> d_los_sched;                                  // LOS scheduler: work counter + per-request done flags
    cudaEvent_t ev_los_sched = nullptr;                        // recorded after every LOS launch: the next one waits for it
    // host mirrors (chunk-blocked, [layer][chunk][64][64]) for the host-side planner
    std::vector<uint8_t>  h_cost;
    std::vector<uint16_t> h_blk, h_liid;
    struct portal_t { int16_t chunk_r, chunk_c, r0, c0, r1, c1; int32_t conn_chunk, conn_idx; };
    std::vector<std::vector<std::vector<portal_t>>> portals;   // [layer][chunk][idx]
    // host-side derived state, owned by the context (no process-global tables: contexts on different threads are independent)
    void *route_state = nullptr;                               // pfnav_route.cu: std::vector<pfnav_route_layer>
    void *route_dev_state = nullptr;                           // pfnav_route.cu: device copies of the routing tables (k_portal_graph_path_warp)
    pf_dbuf<uint16_t> d_gisl;                                  // pfnav_route.cu: global islands, [layer][H64][W64] (pfnav_map_query)
    pf_dbuf<uint8_t> d_mq_buf;                                 // pfnav_query.cu: the inputs and outputs of one query batch
    pf_dbuf<int32_t> d_layer_scratch;                          // pfnav_map_query's whole-layer tier: mq_layer_cta_words per CTA
    std::set<std::pair<int, int>> dirty, fdirty;               // pfnav_blockers.cu: (layer, chunk) occupancy / faction mask changed
    void *blk_state = nullptr;                                 // pfnav_blockers.cu: queued blocker ops + device-side refcount state

    // ---- field pool (pfnav_pool.cu, pfnav_pool_host.h) ----
    pf_pool pool;
    // The plan of the last goal batch stays resident in the staging device buffer: re-requesting the same goals on an
    // unchanged map (map_epoch) relaunches the kernels without re-planning or re-uploading anything.
    uint64_t map_epoch = 0;
    struct goal_batch_t {
        bool valid = false; uint64_t epoch = 0; int layer = 0; std::vector<int32_t> dests, targets;
        pf_waves waves;
    } goal_batch;
    uint32_t tick_no = 1;                         // advanced by pfnav_agents_tick
    // TARGET_ENEMIES / TARGET_ENTITY destinations (pfnav_pool_request_entity_fields): what their repairs start from
    using aux_target = pf_aux_target;
    std::vector<aux_target> aux;

    // ---- agents ----
    size_t n_agents = 0, n_flocks = 0;
    int hz = 20;
    // per-entity arrays (pf_agents_reserve)
    pf_dbuf<pfnav_agent> d_agents;        // AoS input as uploaded
    pf_dbuf<pf_record> d_records;         // 24-B records (uid order)
    pf_dbuf<uint32_t> d_flock_members;    // agent ids grouped by flock, ascending uid
    pf_dbuf<int32_t> d_flock_of;          // [n_agents] flock id column (all-gathered with the records)
    // flock table (pf_flocks_reserve)
    pf_dbuf<pfnav_flock> d_flocks;
    pf_dbuf<uint32_t> d_flock_start;      // [nflocks+1] offsets into d_flock_members
    pf_dbuf<pfnav_formation_in> d_formation;    // optional formation inputs, uid order
    pf_dbuf<pfnav_movestate_ext> d_ms_ext;      // optional: the movestate beyond point seeking
    pf_dbuf<uint8_t> d_enter;             // ENTER_ENTITY_RANGE candidates (pfnav_agents_compute_updates)
    pf_dbuf<uint32_t> d_facts;            // {max radius bits, any garrisoned}
    // multi-GPU: this context owns the entity index range [shard_lo, shard_hi) of the population (pfnav_mgpu.cu)
    size_t shard_lo = 0, shard_hi = 0;
    void *mgpu = nullptr;                 // pf_mgpu: NCCL communicator or in-process group membership
    bool members_stale = false;           // flock member lists must be rebuilt at the next gather
    pf_dbuf<float2> d_cohesion;           // per-agent cohesion force (pre-pass)
    pf_dbuf<float2> d_member_pos;         // positions in flock-member order
    pf_dbuf<pf_prep> d_prep;              // phase-A results of the two-phase velocity update
    bool two_phase = true, two_phase_force = false;
    int phase_a_ctas_per_sm = 0;
    // spatial index (bitmap_grid.h equivalent)
    int grid_w = 0, grid_h = 0; int32_t origin_x = 0, origin_y = 0;
    pf_dbuf<uint32_t> d_cell_count, d_cell_start, d_cell_fill;      // cell index: ncells + 1 each
    pf_dbuf<int32_t> d_sorted_ix, d_sorted_iy;                       // per-entity (pf_agents_reserve)
    pf_dbuf<uint32_t> d_sorted_id;
    pf_dbuf<int32_t> d_sorted_flock;                                 // flock id of every index entry (windowed cohesion)
    // records written since the last index build (pfnav_ents_in_circles refuses then): set by the record writers,
    // cleared by build_index
    bool index_stale = false;
    pf_dbuf<uint32_t> d_eq_ids;                                      // pfnav_ents_in_circles: the answers, then the garrison scratch
    pf_dbuf<uint32_t> d_coh_fallback;
    pf_dbuf<uint32_t> d_scan_part;                                   // block sums of the cell-count scan
    pf_dbuf<unsigned long long> d_cp_stats;                          // ClearPath event counters (pfnav_agents_clearpath_stats)
    pf_dbuf<float4> d_coh_part;                                      // windowed cohesion: partial sums of split runs, [nsplit][n]
    std::vector<uint32_t> h_flock_start;
    int cohesion_mode = 0;
    // work list + outputs (pf_work_reserve)
    size_t n_work = 0;
    pf_dbuf<uint32_t> d_work;
    pf_dbuf<float2> d_vel_out, d_vpref_out, d_vdes_out;
    pf_dbuf<uint8_t> d_los_out;
    pf_dbuf<uint32_t> d_work_count;
    // state update (entity_compute_update)
    pf_dbuf<pfnav_movestate> d_movestate; bool movestate_set = false;
    pf_dbuf<pfnav_patch> d_patches;
    pf_dbuf<uint8_t> d_arrival;                              // [nflocks][nlayers] pf_arrival_dev + tile lists
    uint64_t arrival_epoch = ~0ull; bool arrival_valid = false;
    std::vector<uint8_t> flock_layer_used;                   // [nflocks][12]
    std::vector<pf_arrival_pair> arrival_pairs;              // the used pairs of the last build, slot order
    pf_dbuf<int32_t> d_arrival_scratch;                      // the arrival and ENTER_ENTITY_RANGE tiers' own whole-layer
                                                             // scratch: compute_updates runs on its caller's stream,
                                                             // unordered with pfnav_map_query
    std::vector<pfnav_flock> h_flocks;
    float max_radius = 0.0f;
    bool has_unsupported_state = false;
    bool any_garrisoned = false;                             // G_Pos_EntsInCircleFrom filters + reorders (position.c:100)
    pf_dbuf<uint32_t> d_nb_scratch;
    cudaEvent_t update_done = nullptr;
    bool updates_unapplied = false;                          // set by pfnav_agents_compute_updates, cleared by the apply
    // pfnav_agents_collect_events (pfnav_events.cu): the list of the last collect, its block offsets, count and ballot
    // words, the count's pinned copy and the event recorded behind it; the read's pinned staging. events_valid is
    // cleared by the calls that renumber the population.
    pf_dbuf<pfnav_event> d_events; pf_dbuf<uint32_t> d_event_aux;
    uint32_t *h_event_count = nullptr; cudaEvent_t events_done = nullptr; bool events_valid = false;
    pfnav_event *h_events = nullptr; size_t h_events_cap = 0;
    // pfnav_state_digest (pfnav_digest.cu): the device records of the last digest ([world][PF_DIGEST_REC] words: the own
    // record at rank, the peers' after an NCCL all-gather) and its block array behind them, their pinned copy, the event
    // recorded behind the copy, and what the read reports from the call
    pf_dbuf<unsigned long long> d_digest;
    uint64_t *h_digest = nullptr; size_t h_digest_cap = 0; cudaEvent_t digest_done = nullptr; bool digest_valid = false;
    pfnav_digest digest_info = {}; int digest_world = 1, digest_rank = 0;
    cudaStream_t tick_stream = nullptr;
    cudaEvent_t tick_done = nullptr;
    // LOS chains of a goal batch run on their own stream so that the parts of the tick that do not read
    // fields (all-gather, position index, cohesion) overlap the latency-bound LOS dependency chain
    cudaStream_t field_stream = nullptr, flow_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_los = nullptr, ev_flow = nullptr;
    // measured durations of the previous LOS batch and the previous velocity update steer the two-phase choice
    cudaEvent_t ev_vel0 = nullptr, ev_vel1 = nullptr;
    bool vel_timed = false; float last_los_ms = -1.0f, last_vel_ms = -1.0f;
    bool los_inflight = false;

    // pfnav_plan.cu: the buffers of the request staging (pf_stage_*), and the persistent host threads and per-goal
    // scratch of the goal planner
    void *stager = nullptr;
    void *planner = nullptr;
    // pfnav_pool_repair_batch (pfnav_agents.cu): misses, representatives, their hash table and the gather, grown on demand;
    // the serial pfnav_pool_repair keeps its misses here too
    pf_dbuf<uint8_t> d_rep_buf;
    int repair_stats[6] = {0, 0, 0, 0, 0, 0};                  // the last call: representatives per phase, rounds ended per rule
    // blocking table of pfnav_agents_upload_blocking (uid order, blocking_n records, of which the own range
    // [shard_lo, shard_hi) was uploaded; 0 = none uploaded) and the uid list of pfnav_agents_set_blocking
    pf_dbuf<pfnav_blocking> d_blocking; size_t blocking_n = 0; bool blocking_any_fac = false;
    pf_dbuf<uint32_t> d_block_uids;
    pf_dbuf<uint8_t> d_ckpt;                  // pfnav_agents_save / pfnav_pool_save / _restore: the packed rows or fields
    // pfnav_agents_commands (pfnav_commands.cu): (flock, layer) of every own entity, filled by every full upload, and the device
    // scratch of a batch (merged deltas, per-warp flock histograms, block sums of the work compaction), grown on demand
    pf_cmd_mirror cmd_mirror;
    pf_dbuf<uint8_t> d_cmd_buf;
    // goal, zone and entity-field batches of a multi-GPU job (pfnav_mgpu_request_goals_ex, ..._zones,
    // ..._entity_fields_batch): the staging buffer of the fields built for the job, 4096-byte blocks (a zone or entity
    // batch keeps its copy list behind them), grown on demand; the last call's owner of every goal or request and the
    // requests this member built
    pf_dbuf<uint8_t> d_job_stage;
    std::vector<int32_t> job_owner; int job_built[2] = {0, 0};

    // ---- optional per-kernel timing (pfnav_profile_enable) ----
    bool profiling = false;
    struct prof_rec { int slot; cudaEvent_t a, b; };
    std::vector<prof_rec> prof_pending;
    // host wall-clock segments of pfnav_pool_clear / pfnav_pool_request_goals_ex (pfnav_profile_read_host)
    double host_ms[8] = {0}; uint32_t host_count[8] = {0};
};

// Every entry point that takes a `void *stream`: NULL names the context's own non-blocking stream
// (never the legacy default stream, which would not be ordered against it).
static inline cudaStream_t pf_stream(pfnav_ctx *ctx, void *stream)
{
    return stream ? (cudaStream_t)stream : ctx->tick_stream;
}

// order `st` after the LOS work forked onto field_stream (no-op when none was forked)
static inline cudaError_t pf_fields_join(pfnav_ctx *ctx, cudaStream_t st)
{
    if (!ctx->los_inflight) return cudaSuccess;
    cudaError_t e = cudaStreamWaitEvent(st, ctx->ev_flow, 0);
    if (e != cudaSuccess) return e;
    return cudaStreamWaitEvent(st, ctx->ev_los, 0);
}
// host-side wait for the forked LOS work (setup-time entry points that use blocking copies)
static inline cudaError_t pf_fields_sync(pfnav_ctx *ctx)
{
    if (!ctx->los_inflight) return cudaSuccess;
    cudaError_t e = cudaEventSynchronize(ctx->ev_flow);
    if (e == cudaSuccess) e = cudaEventSynchronize(ctx->ev_los);
    if (e == cudaSuccess) ctx->los_inflight = false;
    return e;
}
// per (flock, layer) constants of arrived() (movement.c:2170), see pfnav_route.cu
#define PF_ARRIVAL_MC_MAX 256           /* FIELD_RES_R*2 + FIELD_RES_C*2 (nav.c:4721) */
struct pf_arrival_consts {
    int32_t nearest_ok; float nearest[2]; int32_t mc_n;
    float mc[PF_ARRIVAL_MC_MAX][2];
};
// which: the searches to run; PF_ARRIVAL_MC needs pfnav_route_build(layer)
enum { PF_ARRIVAL_NEAREST = 1, PF_ARRIVAL_MC = 2 };
// The device table of arrived()'s constants: [nflocks][nlayers] records, each used pair's list of mc_n tile centres at
// mc_off in the float2 array that follows (a 256-entry slot per used pair).
struct pf_arrival_dev { int32_t nearest_ok; float nearest[2]; int32_t mc_n; int32_t mc_off; int32_t _pad[3]; };
// pfnav_query.cu: the constants of npairs (flock, layer) pairs into d_arr / d_tiles on `st`; d_flags: 2 bytes per pair
int pf_arrival_search(pfnav_ctx *ctx, cudaStream_t st, const pf_arrival_pair *d_pairs, int npairs, pf_arrival_dev *d_arr,
                      float2 *d_tiles, uint8_t *d_flags);
int pfnav_arrival_consts(pfnav_ctx *ctx, int layer, float tx, float tz, pf_arrival_consts *out,
                         int which = PF_ARRIVAL_NEAREST | PF_ARRIVAL_MC);

// STATE_ENTER_ENTITY_RANGE (movement.c:2569-2603): an item whose stop depends on N_IsMaximallyClose(new_pos, target, 0)
// -- not within target_range, new tile 4-adjacent to an impassable or blocked one -- leaves k_entity_update as one of these
// records with the end of its update undecided; pf_enter_range_search decides it on the device. Each record owns the patch
// of its work item, so the order of the records does not matter.
struct pf_enter_cand { uint32_t wi; int32_t layer; float nx, nz, tx, tz, prev_x, prev_z; };
// The end of the ENTER_ENTITY_RANGE update: stop (WAITING), or re-issue the order when the target moved more than 5 wu
// since target_prev_pos (v2_len of the difference, as the rest of k_entity_update).
__device__ __forceinline__ void pf_enter_range_tail(pfnav_patch &p, bool stop, float tx, float tz, float prev_x, float prev_z)
{
    if (stop) { p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_WAITING; p.next_block = 1; return; }
    const float dx = tx - prev_x, dz = tz - prev_z;
    if (sqrtf(dx * dx + dz * dz) > 5.0f) {
        p.flags |= PFNAV_UPDATE_SET_DEST | PFNAV_UPDATE_SET_TARGET_PREV;
        p.next_dest[0] = tx; p.next_dest[1] = tz; p.next_attack = 0;
        p.next_target_prev[0] = tx; p.next_target_prev[1] = tz;
    }
}
// pfnav_query.cu: decide the candidates k_entity_update appended (count[0] of them, at most nwork) on `st` and finish
// their patches. count[1] and flagged[0 .. nwork) are the search's own; both counts are zero before k_entity_update.
int pf_enter_range_search(pfnav_ctx *ctx, cudaStream_t st, const pf_enter_cand *d_cand, uint32_t *d_count,
                          uint32_t *d_flagged, int nwork, pfnav_patch *d_patches);
// the device image of the global islands of `layer` ([H64][W64] u16, uploaded by pfnav_route_build), or nullptr when
// the layer's routing structure is not built (pfnav_route.cu)
const uint16_t *pfnav_route_dev_islands(const pfnav_ctx *ctx, int layer);

// One repair of the flow-field repair chain (k_repair_chain, pfnav_fields.cu): applied to field `slot` when its turn
// comes if the direction of `tile` is FD_NONE then, or always (`always`). kind 0 builds its seeds on the device from
// start tile `arg`; kind 1 reads mask row block `mask` (64 x u64).
struct pf_chain_item {
    pfnav_field_req q;
    int32_t slot, tile, kind, arg, always, mask;
};
// The seeds of item `it` (q, kind and arg set; pfnav_route.cu): kind 0 checks its start tile, kind 1 appends its mask
// (pfnav_repair_seeds) to `masks` and sets it.mask. Returns the error and changes nothing when the repair cannot run.
int pf_chain_item_seeds(pfnav_ctx *ctx, pf_chain_item &it, std::vector<uint64_t> &masks);
// Launch chain items on `st`: items grouped by slot (one CTA per group, items in order) into `fields`, 4096 bytes per
// slot: the pool's d_flow, or, when host_fields > 0, that many host fields, staged with the items and copied back on
// `st`. The repairs applied are added to *d_count when it is given. The item and mask arrays are copied on `st` before
// the call returns.
int pfnav_repair_chain_launch(pfnav_ctx *ctx, cudaStream_t st, const std::vector<pf_chain_item> &items,
                              const std::vector<uint64_t> &masks, uint8_t *fields, size_t host_fields, uint32_t *d_count);

// Staged path requests against the pool (pfnav_route.cu), shared by pfnav_pool_request_paths and pfnav_pool_repair_batch:
// begin plans requests i = 0 .. n-1 (each on its own layer) up front; probe emits request i against the pool mirrors as
// they are now without changing anything; commit reserves and stages the probed emission (PFNAV_ERR_NOMEM: nothing
// changed); flush launches what is staged on the stream and uploads the slot table and `has` bytes.
struct pf_path_batch;
struct pf_path_probe {
    int nf = 0, nl = 0, ok = 0; uint32_t dest_id = 0;
    bool would_evict = false;                 // the reservation needs more slots than are free
    std::vector<int32_t> write_slots;         // slots already mapped that the emission writes
};
int  pf_path_batch_begin(pfnav_ctx *ctx, int n, const int32_t *dests, const int32_t *layers, const float *src_xz,
                         const float *dst_xz, cudaStream_t st, pf_path_batch **out);
bool pf_path_batch_planned(const pf_path_batch *B, int i);     // false: the layer is not routed or a point is off the map
int  pf_path_batch_probe(pf_path_batch *B, int i, pf_path_probe *out);
int  pf_path_batch_commit(pf_path_batch *B, std::vector<int32_t> *out_slots);   // out: the slots written
int  pf_path_batch_flush(pf_path_batch *B);
void pf_path_batch_end(pf_path_batch *B);

int pfnav_fmask_push_chunk(pfnav_ctx *ctx, int layer, int chunk);
int pfnav_blockers_flush(pfnav_ctx *ctx);                        // pfnav_blockers.cu: apply the queued blocker operations now
int pfnav_blockers_factions_uploaded(pfnav_ctx *ctx, int layer); // pfnav_blockers.cu: host faction counts of a layer were replaced
// Blocker ops decided on the device (pfnav_blockers.cu). A producer kernel handles `nitems` items in blocks of
// PF_OPS_BLOCK threads; item i writes its 0..2 ops to ops[2i], ops[2i + 1] and desc[i] = nops | wide(op 0) << 2 | wide(op 1)
// << 3 (wide: the circle exceeds the bit window of k_blockers_circles, pf_op_wide), and the block's thread 0 writes
// bsum[block] = its narrow count | wide count << 32. pf_blocker_ops_stage sizes the staging for nitems and the op buffer
// for 2 * nitems more pending ops; pf_blocker_ops_append compacts the staged ops in item order behind the pending ones
// (on `st`, no host wait). pfnav_map_commit applies them.
#define PF_OPS_BLOCK 256
struct pf_op_stage { pfnav_blocker_op *ops; uint8_t *desc; unsigned long long *bsum; };
int pf_blocker_ops_stage(pfnav_ctx *ctx, size_t nitems, pf_op_stage *out);
int pf_blocker_ops_append(pfnav_ctx *ctx, cudaStream_t st, size_t nitems, bool any_fac);
// The exchange of device-decided ops between the members of a job (pfnav_mgpu.cu). pf_blocker_ops_view waits for the
// device and describes the member's pending ops: the count pair on the device, the leading `sent` ops every member
// already holds, and whether any op may carry a faction. pf_blocker_ops_reserve makes room for `need` ops in each buffer
// (keeping the pending ones; the pointers may change). pf_blocker_ops_exchanged: the buffers now hold cnt = {narrow,
// wide} ops, all of them held by every member.
struct pf_ops_view { pfnav_blocker_op *narrow, *wide; uint32_t *d_cnt; uint32_t sent[2]; bool fac; };
int pf_blocker_ops_view(pfnav_ctx *ctx, pf_ops_view *out);
int pf_blocker_ops_reserve(pfnav_ctx *ctx, size_t need, pf_ops_view *out);
int pf_blocker_ops_exchanged(pfnav_ctx *ctx, const uint32_t cnt[2], bool any_fac);
bool pf_mgpu_shares_blockers(const pfnav_ctx *ctx);             // pfnav_mgpu.cu: member of a job that opted in
bool pf_blocker_ops_unexchanged(pfnav_ctx *ctx);                // pfnav_blockers.cu: ops decided since the last exchange
bool pf_blocker_ops_pending(pfnav_ctx *ctx);                    // pfnav_blockers.cu: device-decided ops not yet committed
// pfnav_blockers.cu: the next pfnav_map_commit has work left: device-decided or host-queued blocker ops, or dirty chunks
bool pf_map_uncommitted(pfnav_ctx *ctx);
void pf_mgpu_rank_world(const pfnav_ctx *ctx, int *rank, int *world);    // pfnav_mgpu.cu: 0 / 1 outside a job
__host__ __device__ __forceinline__ bool pf_op_wide(float range) { return !(range >= 0.0f && (int)ceilf(range / 4) <= 12); }

int pfnav_aux_chunk_seeds(pfnav_ctx *ctx, int dest, int chunk_r, int chunk_c, std::vector<int> &out);     // pfnav_region.cu
// The inputs of an entity-field batch named by uid (pfnav_*_request_entity_fields_resident; pfnav_region.cu): checks the
// arguments (pf_resident_check), refuses stale records (PFNAV_ERR_STATE), resolves the named uids from the context's
// records with k_resident_footprints on `st` (one host wait) and merges them (pf_resident_merge). m == 0 resolves
// nothing. Changes nothing but the request staging.
int pf_resident_resolve(pfnav_ctx *ctx, cudaStream_t st, const pfnav_entity_field_req *reqs, size_t m,
                        const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents, const uint32_t *seeker_uids,
                        size_t nseekers, pf_resident_batch &B);
// PFNAV_ERR_STATE, with the message "<what> by uid: ...", when records were written after the last index build.
int pf_resident_fresh(pfnav_ctx *ctx, const char *what);
// The calls whose positions may name resident entities (pfnav_pool_request_paths_resident, pfnav_map_query_resident,
// pfnav_group_arrival_velocity_resident; pfnav_region.cu): pf_resident_points_check against the context's population
// (PFNAV_ERR_ARG), then, when n > 0, pf_resident_fresh (PFNAV_ERR_STATE). Changes nothing.
int pf_resident_points_begin(pfnav_ctx *ctx, const char *what, size_t n, const uint32_t *uids_a, bool given_a,
                             const uint32_t *uids_b, bool given_b, pf_resident_points &P);
// k_resident_xz on `st` for P's pairs, staged at d_pairs by P.pack: the x, z of each named record over buf[entry * stride
// + off0] (the first array's pairs) or buf[entry * stride + off1] (the second's). Nothing when P names nothing.
int pf_resident_xz_launch(pfnav_ctx *ctx, cudaStream_t st, const uint8_t *d_pairs, const pf_resident_points &P, int stride,
                          int off0, int off1, float *buf);

// ---- pfnav_pool.cu: the device pool, and the pool mutators of a context, each of which drops the resident goal plan
// Bring the device copies of the pool up to date after pfnav_pool_clear: empty slot table, no `has` bytes, zero touch
// stamps, ordered on `st` after the forked field work (which may still write the pool). Every entry point that reads
// or writes the device pool calls this first, on the stream it runs on.
cudaError_t pf_pool_refresh(pfnav_ctx *ctx, cudaStream_t st);
int pf_pool_free(pfnav_ctx *ctx);                          // forget every slot: pfnav_destroy, pfnav_map_create, pfnav_pool_create
// pfnav_pool_host.h's reservation, with the device's touch stamps when it must evict
int pf_pool_reserve(pfnav_ctx *ctx, const size_t *keys, size_t n, int32_t *slots_out, bool *out_evicted);
int32_t pf_pool_zone_take(pfnav_ctx *ctx, size_t key);     // the zone rule: the key's slot, -1 when the pool is full
void pf_pool_drop(pfnav_ctx *ctx, int dest, int chunk);    // pfnav_map_commit: the map changed under the key's fields
// copy the slot table and the `has` bytes into `host` (pinned, pool.table_bytes() long) and enqueue their two copies to
// the device on `st`; the caller records the event that guards the reuse of `host` after them
int pf_pool_stage_table(pfnav_ctx *ctx, uint8_t *host, cudaStream_t st);
void pf_planner_destroy(pfnav_ctx *ctx);                         // pfnav_plan.cu: join the goal planner threads

// ---- pfnav_plan.cu: request staging. A batch built on the host goes through the next of two pinned buffers into the
// context's one device buffer, which the batch's kernels then read. The blocking calls on host arrays (pfnav_flow_fields_update
// and the like) also write their outputs behind their inputs there and copy them back before they return.
//   pf_stage_begin  S->host: host_bytes, then the pool's slot table and `has` bytes when `table`, once the copy that last
//                   read the pinned buffer is done. S->dev: dev_bytes (none when 0), with `st` ordered after the buffer's
//                   last readers: the forked field work (pf_fields_join) and the stream-ordered reader that called
//                   pf_stage_done. Growing it waits for both on the host. Drops the resident goal plan, which lives there.
//   pf_stage_upload copies host[0, bytes) to S.dev on `st`, then the table when asked for; guards the pinned buffer.
//   pf_stage_done   after the last kernel on `st` that reads S.dev; forked readers are joined instead.
struct pf_stage { uint8_t *host = nullptr, *dev = nullptr, *table = nullptr; int ri = 0; };
int pf_stage_begin(pfnav_ctx *ctx, cudaStream_t st, size_t host_bytes, size_t dev_bytes, bool table, pf_stage *S);
int pf_stage_upload(pfnav_ctx *ctx, cudaStream_t st, const pf_stage &S, size_t bytes);
int pf_stage_done(pfnav_ctx *ctx, cudaStream_t st);
void pf_stage_free(pfnav_ctx *ctx);                              // pfnav_destroy, after the device is idle
// a packed batch (pfnav_waves_host.h) at `dev`: every flow wave on `flow_st`, one launch each, then its LOS requests in
// one launch on `los_st`, into the fields (pool or staging blocks) their destinations name
int pf_waves_launch(pfnav_ctx *ctx, const uint8_t *dev, const pf_waves &W, uint8_t *flow_fields, uint8_t *los_fields,
                    cudaStream_t flow_st, cudaStream_t los_st);

// One member's part of a goal batch of a multi-GPU job (pfnav_plan.cu; the transports are in pfnav_mgpu.cu).
//   pf_job_plan   plans the batch on the member's planner threads and describes what pfnav_pool_request_goals_ex would
//                 write, changing nothing: lack[g * chunks + c] (bit 0 flow, bit 1 LOS: the member lacks that field of
//                 goal g), the solo counts and whether the member's reservation would succeed. The merged plan stays in
//                 the member's planner until pf_job_launch.
//   pf_job_launch takes `uni`, the OR of every member's lack bytes: assigns every goal with a field in `uni` to one
//                 owner, lays the owners' fields out in the staging buffer (segment of rank r: blocks [seg[r], seg[r+1])),
//                 reserves the member's slots exactly as the solo call does, uploads its slot table and `has` bytes,
//                 and builds the fields of the goals `rank` owns into its segment; `st` is joined after the builds.
//   pf_job_scatter (after the exchange of the segments) copies every field the member lacks from the staging buffer
//                 into its pool slot, on `st`, and makes the next pool reader wait for it.
// Zone and entity-field batches (kind PF_JOB_ZONES / PF_JOB_ENTITY) take the same three steps: pf_job_plan validates
// and takes the verdict of the member's reservation (pf_aux_job_plan, pfnav_region.cu: pf_pool_zone_fits, or
// pf_pool_fits of each request; no lack record: every member writes every key the arguments name), pf_job_launch
// reserves, lays out the owners' fields (pf_job_layout) and builds the member's own (pf_aux_job_launch), pf_job_scatter
// copies.
enum { PF_JOB_GOALS = 0, PF_JOB_ZONES = 1, PF_JOB_ENTITY = 2 };
struct pf_job {
    int kind = PF_JOB_GOALS;
    int ngoals = 0, layer = 0; uint32_t flags = 0;
    const int32_t *dests = nullptr, *targets = nullptr;
    size_t m = 0;                                   // zone / entity-field requests
    const pfnav_zone_req *zreqs = nullptr; const pfnav_entity_field_req *ereqs = nullptr;
    const pfnav_footprint *ents = nullptr; size_t nents = 0; const int32_t *chunks_rc = nullptr; size_t nchunks = 0;
    std::vector<int32_t> nfields;                   // zones: fields per request (pf_job_launch)
    std::shared_ptr<void> aux;                      // pfnav_region.cu: the validated batch, from pf_job_plan to pf_job_launch
    bool fits = true; int nf = 0, nl = 0;           // pf_job_plan
    std::vector<uint8_t> lack;
    std::vector<size_t> seg;                        // pf_job_launch: world + 1 block offsets
    const void *d_items = nullptr; int nitems = 0;  // the member's copies from staging into its pool
    int refused = 0;                                // the member's verdict before planning (a resident batch it could not resolve)
};
int pf_job_plan(pfnav_ctx *ctx, pf_job &J);
int pf_job_launch(pfnav_ctx *ctx, pf_job &J, const uint8_t *uni, int world, int rank, cudaStream_t st);
int pf_job_scatter(pfnav_ctx *ctx, pf_job &J, cudaStream_t st);
int pf_job_check_state(pfnav_ctx *ctx);
int pf_aux_job_plan(pfnav_ctx *ctx, pf_job &J);
int pf_aux_job_launch(pfnav_ctx *ctx, pf_job &J, int world, int rank, cudaStream_t st);
// one field copy of k_field_copy: block src of the source buffer of its kind (0 flow, 1 LOS) to block dst
struct pf_field_copy { int32_t src, dst, kind; };
//   pf_job_layout  owners and staging blocks of a zone or entity-field batch: field f of the batch (in the order the
//                  serial calls write them) is written by request freq[f] to key fkey[f] and costs fcost[f]. A key
//                  belongs to the request that writes it last; a request costs what its last-written keys cost. The most
//                  expensive request first, to the member with the least cost so far, ties to the lower rank; sets
//                  ctx->job_owner (-1: the request writes no key last) and J.seg; blk[f]: the field's staging block, -1
//                  when a later field writes its key.
//   pf_job_stage   grows the staging buffer to the job's blocks with `items` behind them and uploads the items, the
//                  member's slot table and its `has` bytes on `st` (J.d_items, J.nitems for pf_job_scatter).
void pf_job_layout(pfnav_ctx *ctx, pf_job &J, const std::vector<int32_t> &freq, const std::vector<size_t> &fkey,
                   const std::vector<int64_t> &fcost, int world, std::vector<int32_t> &blk);
int pf_job_stage(pfnav_ctx *ctx, pf_job &J, const std::vector<pf_field_copy> &items, int world, cudaStream_t st);
enum { PF_PROF_FLOW = 0, PF_PROF_LOS = 1, PF_PROF_INDEX = 2, PF_PROF_VDES = 3, PF_PROF_COHESION = 4,
       PF_PROF_VELOCITY = 5, PF_PROF_UPDATE = 6, PF_PROF_APPLY = 7, PF_PROF_SLOTS = 8 };

// host segments of a cold goal batch (pfnav_profile_read_host): 0 pfnav_pool_clear, 1 waits on events / streams,
// 2 planning, 3 merge + dependency sort, 4 pf_pool_reserve, 5 packing, 6 H2D enqueue, 7 kernel launches
enum { PF_HPROF_CLEAR = 0, PF_HPROF_WAIT = 1, PF_HPROF_PLAN = 2, PF_HPROF_MERGE = 3, PF_HPROF_RESERVE = 4,
       PF_HPROF_PACK = 5, PF_HPROF_UPLOAD = 6, PF_HPROF_LAUNCH = 7, PF_HPROF_SLOTS = 8 };

// lap timer over consecutive host segments: lap(slot) books the time since the previous lap; off unless profiling
struct pf_host_timer {
    pfnav_ctx *ctx; std::chrono::steady_clock::time_point t;
    explicit pf_host_timer(pfnav_ctx *c) : ctx(c) { if (ctx->profiling) t = std::chrono::steady_clock::now(); }
    void lap(int slot)
    {
        if (!ctx->profiling) return;
        const auto now = std::chrono::steady_clock::now();
        ctx->host_ms[slot] += std::chrono::duration<double, std::milli>(now - t).count();
        ctx->host_count[slot]++;
        t = now;
    }
};

// RAII helper: brackets the launches of one kernel group with events when profiling is on
struct pf_prof_scope {
    pfnav_ctx *ctx; cudaStream_t st; int slot; cudaEvent_t a = nullptr, b = nullptr;
    pf_prof_scope(pfnav_ctx *c, cudaStream_t s, int sl) : ctx(c), st(s), slot(sl)
    {
        if (!ctx->profiling) return;
        cudaEventCreate(&a); cudaEventCreate(&b);
        cudaEventRecord(a, st);
    }
    ~pf_prof_scope()
    {
        if (!a) return;
        cudaEventRecord(b, st);
        ctx->prof_pending.push_back({slot, a, b});
    }
};

// ---- pfnav_fields.cu ----
int pfnav_fields_init(pfnav_ctx *ctx);
void pfnav_fields_free(pfnav_ctx *ctx);

int pfnav_flow_launch(pfnav_ctx *ctx, const pfnav_field_req *d_reqs, size_t n, uint8_t *d_inout_fields,
                      const int32_t *d_out_slot, void *stream);
int pfnav_los_launch(pfnav_ctx *ctx, const pfnav_los_req *d_reqs, size_t n, uint8_t *d_out_fields,
                     const int32_t *d_out_slot, void *stream);

// ---- pfnav_agents.cu ----
void pfnav_agents_free(pfnav_ctx *ctx);
int pfnav_agents_init(pfnav_ctx *ctx);
int pfnav_agents_finish_snapshot(pfnav_ctx *ctx, cudaStream_t st, bool members);
// max_radius and any_garrisoned from the records of the whole population (k_population_facts); waits for `st`
int pfnav_agents_refresh_facts(pfnav_ctx *ctx, cudaStream_t st);
// the one sizing of each group of arrays that share a length (pf_dbuf_reserve_all): the flock table for nflocks flocks
// (d_flocks nflocks + 1, d_flock_start nflocks + 2), and the work list and its outputs for nwork items with the 4-word
// d_work_count. A failed work list also empties the list (n_work = 0), so no tick reads the released arrays.
int pf_flocks_reserve(pfnav_ctx *ctx, size_t nflocks);
int pf_work_reserve(pfnav_ctx *ctx, size_t nwork);
// the spatial index of the current records (pfnav_agents_rebuild_index), on `st`
int build_index(pfnav_ctx *ctx, cudaStream_t st);
// entity_block (mode 1) / entity_unblock (mode 0) of the n uids at d_uids (unique) through k_blocking_decide, appended to
// the device-decided ops that pfnav_map_commit applies; d_patches != nullptr: the rules of PFNAV_APPLY_BLOCKERS instead
int blocking_emit(pfnav_ctx *ctx, cudaStream_t st, const uint32_t *d_uids, int n, const pfnav_patch *d_patches, int mode);
// pfnav_agents_restore: the incref of every restored row of [lo, lo + n) that holds a block (pf_ckpt_restore_op), in uid
// order, through k_blocking_restore_decide into the same op buffer
int blocking_restore_emit(pfnav_ctx *ctx, cudaStream_t st, size_t lo, int n);
// ---- pfnav_checkpoint.cu: a restore in steps, so that a group checks the segments once and every member before any
// member changes ----
// ready: a device context with a map. check: the member's own state against segments pf_ckpt_check accepted (route
// builds of the layers in use, shared blockers in a job), changing nothing; [*lo, *hi): the range the context takes.
// apply: the uploads of the range's records and the ops of its blocking rows, on `st`.
int pf_ckpt_restore_ready(pfnav_ctx *ctx);
int pf_ckpt_restore_check(pfnav_ctx *ctx, const pf_ckpt_set &S, size_t *lo, size_t *hi);
int pf_ckpt_restore_apply(pfnav_ctx *ctx, const pf_ckpt_set &S, size_t lo, size_t hi, cudaStream_t st);
// ---- pfnav_events.cu ----
void pf_events_free(pfnav_ctx *ctx);                             // pfnav_destroy, after the device is idle
// ---- pfnav_digest.cu: pfnav_state_digest in steps, so that the NCCL form all-gathers the records in between ----
// check: the arguments against the context, changing nothing. launch: the digest kernels on `st`, writing the own record
// at rank of a world-record area and the block array. finish: the copy of the records and blocks to the pinned buffer and
// the event behind it. A digest record holds PF_DIGEST_REC words: population, flocks, records, map, pool, 0, 0, 0.
#define PF_DIGEST_REC 8
int pf_digest_check(pfnav_ctx *ctx, uint32_t what, int block_log2);
int pf_digest_launch(pfnav_ctx *ctx, uint32_t what, int block_log2, cudaStream_t st, int world, int rank);
int pf_digest_finish(pfnav_ctx *ctx, cudaStream_t st);
void pf_digest_free(pfnav_ctx *ctx);                             // pfnav_destroy, after the device is idle
// ---- pfnav_checkpoint.cu / pfnav_pool.cu: what the digest shares with the saves ----
uint32_t pf_ckpt_tables(const pfnav_ctx *ctx);                   // the PF_CKPT_* tables pfnav_agents_save writes
// the per-entity tables a row is packed from, as 16-byte words: table t (pf_ckpt_word_source's t) holds words[t] words
// per uid; a table the context does not hold is null
struct pf_ckpt_src { const uint4 *p[5]; uint32_t words[5]; };
pf_ckpt_src pf_ckpt_sources(const pfnav_ctx *ctx);
// k_map_digest on `st`: the wrapping sum of the block terms added to *d_sum (pf_digest_fold finishes it)
int pf_map_digest_launch(pfnav_ctx *ctx, cudaStream_t st, unsigned long long *d_sum);

// ---- pfnav_commands.cu: a job member's part of a command batch (pfnav_mgpu.cu runs the verdict exchange) ----
// pf_cmd_job_check validates the batch against the member's state and plans it, changing nothing (the error is set);
// pf_cmd_job_apply applies a checked batch on `st` (the caller has selected the member's device).
struct pf_cmd_job {
    std::vector<pfnav_agent_delta> own;
    std::vector<pf_cmd_foreign> foreign;
    std::vector<pf_cmd_change> changes;
    const pfnav_flock *flocks = nullptr; size_t nflocks = 0;
};
int pf_cmd_job_check(pfnav_ctx *ctx, const pfnav_agent_delta *deltas, size_t n, const pfnav_flock *flocks, size_t nflocks,
                     pf_cmd_job &J);
int pf_cmd_job_apply(pfnav_ctx *ctx, const pf_cmd_job &J, cudaStream_t st);

// ---- pfnav_inputs.cu: a job member's part of an input batch (pfnav_mgpu.cu runs the verdict exchange) ----
// pf_input_job_check validates the whole batch against the population and keeps the folded records of the member's own
// range, changing nothing (the error is set); pf_input_job_apply writes them on `st`, creating the formation table first
// when the batch carries PFNAV_INPUT_FORMATION and the member has none. pf_input_tables: the tables a batch may write,
// as the verdict's bits (1 movestate_ext, 2 formation).
struct pf_input_job {
    std::vector<pfnav_input_delta> own;
    bool any_form = false;
};
int pf_input_job_check(pfnav_ctx *ctx, const pfnav_input_delta *d, size_t n, pf_input_job &J);
int pf_input_job_apply(pfnav_ctx *ctx, const pf_input_job &J, cudaStream_t st);
static inline uint32_t pf_input_tables(const pfnav_ctx *ctx)
{
    return (ctx->d_ms_ext != nullptr ? 1u : 0u) | (ctx->d_formation != nullptr ? 2u : 0u);
}

// ---- pfnav_commands.cu: a job member's part of a population change (pfnav_mgpu.cu runs the verdict exchange and moves
// the segments between the stages) ----
// One block of rows of every table a population change writes, in a member's command scratch; row 0 has the new uid
// `first`. Tables that do not exist are null.
struct pf_pop_rows {
    pfnav_agent *agents = nullptr; pf_record *rec = nullptr; int32_t *flock = nullptr; pfnav_movestate *ms = nullptr;
    pfnav_movestate_ext *ext = nullptr; pfnav_formation_in *form = nullptr; pfnav_blocking *blk = nullptr;
    size_t first = 0;
    int device = 0;
};
struct pf_pop_member {
    pf_pop_job J;
    pf_pop_tables T = {};
    const pfnav_agent *add = nullptr; const pfnav_movestate *add_ms = nullptr; const pfnav_movestate_ext *add_ext = nullptr;
    const pfnav_formation_in *add_form = nullptr; const pfnav_blocking *add_blk = nullptr; size_t nadd = 0;
    const pfnav_flock *flocks = nullptr; size_t nflocks = 0;
    pf_pop_rows own;                     // the member's survivors, new uids [keep_lo[rank], keep_lo[rank + 1])
    std::vector<pf_pop_rows> from;       // per sender: the block holding its segment for this member (own for itself)
    std::vector<pf_pop_rows> pair;       // receive_all: one block per (sender, receiver) segment, [s * world + r]
    pf_record *c_rec = nullptr; int32_t *c_flock = nullptr;       // the compacted columns of the whole new population
    uint8_t *stage = nullptr;            // the staged inputs, at these offsets
    size_t s_removed = 0, s_key = 0, s_agents = 0, s_ms = 0, s_ext = 0, s_form = 0, s_blk = 0, s_fac = 0;
    pf_cmd_mirror mirror;                // the mirror of the new range, committed by pf_pop_job_commit
};
// pf_pop_job_check: validation and plan, changing nothing (the error is set). pf_pop_job_stage (on `st`): the scratch, the
// blocks released by the member's removed entities, its survivors compacted into `own`, the replicated record and flock
// columns compacted in the scratch; receive_all also lays out `pair` (the NCCL form receives every segment). Between
// stage and write every `from` block must be final. pf_pop_job_write: the tables at their new length and the member's
// new range written from `from`, its appended entities and the compacted columns. pf_pop_job_commit: the host facts,
// member lists and population facts; the scratch is reused from here on, so no peer may still read `own`.
int pf_pop_job_check(pfnav_ctx *ctx, const uint32_t *remove_uids, size_t nremove, const pfnav_agent *add,
                     const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext, const pfnav_formation_in *add_form,
                     const pfnav_blocking *add_blk, size_t nadd, const pfnav_flock *flocks, size_t nflocks, int world, int rank,
                     pf_pop_member &M);
int pf_pop_job_stage(pfnav_ctx *ctx, pf_pop_member &M, bool receive_all, cudaStream_t st);
int pf_pop_job_write(pfnav_ctx *ctx, pf_pop_member &M, cudaStream_t st);
int pf_pop_job_commit(pfnav_ctx *ctx, pf_pop_member &M, cudaStream_t st);

// ---- device helpers shared by kernels ----
__device__ __forceinline__ uint32_t pf_lane() { return threadIdx.x & 31; }

// entity footprint -> tiles (pfnav_blockers.cu), for the TARGET_ENTITY / TARGET_ENEMIES frontiers
int pfnav_footprint_tiles(const pfnav_ctx *ctx, const pfnav_footprint *e, int rings, int32_t *out_rc);
