// pfnav_commands_host.h -- the host side of pfnav_agents_commands and the write rule its kernel applies, CUDA-free:
// delta validation, per-uid merging in array order, the navigation layer rule and the (flock, layer) mirror that keeps
// flock_layer_used equal to a fresh upload's; and the split of a multi-GPU job's batch into a member's own and foreign
// parts. tests/emu/commands_emu.cpp and tests/emu/commands_job_emu.cpp build this header with g++.
#pragma once
#include <math.h>
#include <stdint.h>
#include <unordered_map>
#include <vector>
#include "../../include/pfnav.h"

#ifdef __CUDACC__
#define PF_HD __host__ __device__ __forceinline__
#else
#define PF_HD inline
#endif

#define PF_DELTA_PUBLIC 0x3FFu
// Merged records only. A PFNAV_DELTA_CLEAR_HIST delta is resolved against the flags the entity has at that point of the
// batch: known from an earlier PFNAV_DELTA_FLAGS of the batch (CLEAR_NOW when not COMBAT_HELD, nothing when held), or
// else the flags the entity has on the device before the batch (CLEAR_ORIG: the kernel decides).
#define PF_DELTA_CLEAR_NOW  (1u << 30)
#define PF_DELTA_CLEAR_ORIG (1u << 31)

// Entity_NavLayerWithRadius (entity.c:554) in two parts: layer = base(flags) + size class(radius)
static inline int pf_layer_base(uint32_t flags) { return (flags & PFNAV_FLAG_WATER) ? 4 : (flags & PFNAV_FLAG_AIR) ? 8 : 0; }
static inline int pf_layer_class(float r) { return r >= 15.0f ? 3 : r >= 10.0f ? 2 : r >= 5.0f ? 1 : 0; }

// One delta (public or merged) on one entity, fields in the order of the mask bits. ms / ex may be NULL when the delta
// carries no bit that writes them.
PF_HD void pf_delta_apply(pfnav_agent *a, pfnav_movestate *ms, pfnav_movestate_ext *ex, const pfnav_agent_delta &d)
{
    const uint32_t flags0 = a->flags;
    if (d.mask & PFNAV_DELTA_STATE) a->state = d.state;
    if (d.mask & PFNAV_DELTA_FLOCK) a->flock = d.flock;
    if (d.mask & PFNAV_DELTA_AUX_DEST) a->aux_dest1 = d.aux_dest1;
    if (d.mask & PFNAV_DELTA_FLAGS) a->flags = d.flags & 0xFFFFFFu;
    if (d.mask & PFNAV_DELTA_SPEEDS) { a->max_speed = d.max_speed; a->speed = d.speed; }
    if (d.mask & PFNAV_DELTA_RADIUS) a->radius = d.radius;
    if (d.mask & PFNAV_DELTA_VELOCITY) { a->velocity[0] = d.velocity[0]; a->velocity[1] = d.velocity[1]; }
    if (d.mask & PFNAV_DELTA_POSITION) {
        a->pos[0] = a->prev_pos[0] = d.position[0]; a->pos[1] = a->prev_pos[1] = d.position[1];
        ms->next_pos[0] = d.position[0]; ms->next_pos[2] = d.position[1];
        ms->step = 0.0f; ms->left = 0;
    }
    const bool clear = (d.mask & PF_DELTA_CLEAR_NOW) || ((d.mask & PF_DELTA_CLEAR_ORIG) && !(flags0 & PFNAV_FLAG_COMBAT_HELD)) ||
                       ((d.mask & PFNAV_DELTA_CLEAR_HIST) && !(a->flags & PFNAV_FLAG_COMBAT_HELD));
    if (clear)
        for (int i = 0; i < PFNAV_VEL_HIST_LEN; i++) { ms->vel_hist[i][0] = 0.0f; ms->vel_hist[i][1] = 0.0f; }
    if (d.mask & PFNAV_DELTA_TARGET) { ex->surround_target_uid = d.target_uid; ex->target_range = d.target_range; }
}

struct pf_cmd_limits {
    size_t lo, hi, n_agents;      // own range, population
    size_t nflocks;               // length of the flock table after the call
    bool have_ms, have_ext;       // movestate / movestate_ext tables uploaded
};

// the checks of one delta that need nothing but the delta; NULL when it passes
static inline const char *pf_delta_check(const pfnav_agent_delta &d, const pf_cmd_limits &L)
{
    if (d.uid < L.lo || d.uid >= L.hi) return "delta uid outside this context's own entity range";
    if (d.mask & ~PF_DELTA_PUBLIC) return "unknown delta mask bit";
    if ((d.mask & PFNAV_DELTA_STATE) && d.state > PFNAV_STATE_ARRIVING_TO_CELL) return "delta state outside enum pfnav_move_state";
    if ((d.mask & PFNAV_DELTA_FLOCK) && (d.flock < -1 || d.flock >= (int64_t)L.nflocks)) return "delta flock index outside the flock table";
    if ((d.mask & PFNAV_DELTA_SPEEDS) && !(isfinite(d.max_speed) && isfinite(d.speed))) return "delta speeds not finite";
    if ((d.mask & PFNAV_DELTA_RADIUS) && !isfinite(d.radius)) return "delta radius not finite";
    if ((d.mask & PFNAV_DELTA_VELOCITY) && !(isfinite(d.velocity[0]) && isfinite(d.velocity[1]))) return "delta velocity not finite";
    if ((d.mask & PFNAV_DELTA_POSITION) && !(isfinite(d.position[0]) && isfinite(d.position[1]))) return "delta position not finite";
    if ((d.mask & (PFNAV_DELTA_POSITION | PFNAV_DELTA_CLEAR_HIST)) && !L.have_ms)
        return "PFNAV_DELTA_POSITION / PFNAV_DELTA_CLEAR_HIST need pfnav_agents_upload_movestate";
    if (d.mask & PFNAV_DELTA_TARGET) {
        if (!L.have_ext) return "PFNAV_DELTA_TARGET needs pfnav_agents_upload_movestate_ext";
        if (!isfinite(d.target_range)) return "delta target_range not finite";
        if (d.target_uid != PFNAV_NULL_UID && d.target_uid >= L.n_agents) return "delta target_uid outside the population";
    }
    return nullptr;
}

// Validate every delta and fold the deltas of one uid, in array order, into one record (first-occurrence order), so that
// one thread owns each entity. Applying `out` equals applying `d` one by one. Returns NULL, or what was wrong (out is
// then meaningless).
static inline const char *pf_cmd_merge(const pfnav_agent_delta *d, size_t n, const pf_cmd_limits &L, std::vector<pfnav_agent_delta> &out)
{
    out.clear();
    std::unordered_map<uint32_t, uint32_t> at;
    at.reserve(n * 2);
    for (size_t i = 0; i < n; i++) {
        const pfnav_agent_delta &s = d[i];
        if (const char *e = pf_delta_check(s, L)) return e;
        auto it = at.find(s.uid);
        if (it == at.end()) {
            it = at.emplace(s.uid, (uint32_t)out.size()).first;
            pfnav_agent_delta z = {};
            z.uid = s.uid;
            out.push_back(z);
        }
        pfnav_agent_delta &m = out[it->second];
        if (s.mask & PFNAV_DELTA_STATE) m.state = s.state;
        if (s.mask & PFNAV_DELTA_FLOCK) m.flock = s.flock;
        if (s.mask & PFNAV_DELTA_AUX_DEST) m.aux_dest1 = s.aux_dest1;
        if (s.mask & PFNAV_DELTA_FLAGS) m.flags = s.flags & 0xFFFFFFu;
        if (s.mask & PFNAV_DELTA_SPEEDS) { m.max_speed = s.max_speed; m.speed = s.speed; }
        if (s.mask & PFNAV_DELTA_RADIUS) m.radius = s.radius;
        if (s.mask & PFNAV_DELTA_VELOCITY) { m.velocity[0] = s.velocity[0]; m.velocity[1] = s.velocity[1]; }
        if (s.mask & PFNAV_DELTA_POSITION) { m.position[0] = s.position[0]; m.position[1] = s.position[1]; }
        if (s.mask & PFNAV_DELTA_TARGET) { m.target_uid = s.target_uid; m.target_range = s.target_range; }
        m.mask |= s.mask & ~PFNAV_DELTA_CLEAR_HIST;
        if (s.mask & PFNAV_DELTA_CLEAR_HIST) {
            if (!(m.mask & PFNAV_DELTA_FLAGS)) m.mask |= PF_DELTA_CLEAR_ORIG;
            else if (!(m.flags & PFNAV_FLAG_COMBAT_HELD)) m.mask |= PF_DELTA_CLEAR_NOW;
        }
    }
    return nullptr;
}

// (flock, layer) of every own entity and the entities per (flock, layer): filled at upload, updated by the command
// batches (nothing else changes an entity's flock, flags or radius). used() is the flock_layer_used table a fresh upload
// of the population would compute.
struct pf_cmd_mirror {
    std::vector<int32_t> flock;
    std::vector<uint8_t> layer;
    std::vector<uint32_t> count;          // [nflocks][PFNAV_NAV_LAYER_MAX]
    size_t nflocks = 0;

    void reset(size_t n, size_t nf)
    {
        flock.assign(n, -1); layer.assign(n, 0); count.assign(nf * PFNAV_NAV_LAYER_MAX, 0); nflocks = nf;
    }
    void set(size_t i, int32_t f, int l)      // upload: entity i of the own range, not counted before
    {
        flock[i] = f; layer[i] = (uint8_t)l;
        if (f >= 0) count[(size_t)f * PFNAV_NAV_LAYER_MAX + l]++;
    }
    void used(std::vector<uint8_t> &out) const
    {
        out.resize(count.size());
        for (size_t k = 0; k < count.size(); k++) out[k] = count[k] ? 1 : 0;
    }
};

struct pf_cmd_change { uint32_t idx; int32_t flock; uint8_t layer; };     // idx: index into the own range

// What the merged batch does to the mirror, changing nothing: every entity's resulting layer must exist, and no entity
// may keep a flock index the new table no longer has. Returns NULL or what was wrong.
static inline const char *pf_cmd_plan(const pf_cmd_mirror &M, size_t lo, const std::vector<pfnav_agent_delta> &merged,
                                      size_t nflocks_new, int nlayers, std::vector<pf_cmd_change> &out)
{
    out.clear();
    int64_t stranded = 0;
    for (size_t f = nflocks_new; f < M.nflocks; f++)
        for (int l = 0; l < PFNAV_NAV_LAYER_MAX; l++) stranded += M.count[f * PFNAV_NAV_LAYER_MAX + l];
    for (const pfnav_agent_delta &m : merged) {
        if (!(m.mask & (PFNAV_DELTA_FLOCK | PFNAV_DELTA_FLAGS | PFNAV_DELTA_RADIUS))) continue;
        const size_t i = m.uid - lo;
        const int base = (m.mask & PFNAV_DELTA_FLAGS) ? pf_layer_base(m.flags) : (M.layer[i] & ~3);
        const int cls = (m.mask & PFNAV_DELTA_RADIUS) ? pf_layer_class(m.radius) : (M.layer[i] & 3);
        if (base + cls >= nlayers) return "a delta gives an entity a navigation layer that was not created (radius/flags)";
        const int32_t f = (m.mask & PFNAV_DELTA_FLOCK) ? m.flock : M.flock[i];
        if (M.flock[i] >= (int64_t)nflocks_new && f < (int64_t)nflocks_new) stranded--;
        if (f != M.flock[i] || base + cls != M.layer[i]) out.push_back({(uint32_t)i, f, (uint8_t)(base + cls)});
    }
    if (stranded > 0) return "the new flock table is shorter than the flock index some entity keeps";
    return nullptr;
}

static inline void pf_cmd_commit(pf_cmd_mirror &M, const std::vector<pf_cmd_change> &changes, size_t nflocks_new)
{
    // a shrinking table drops its tail only after the entities that leave it are taken out of its counts
    if (nflocks_new > M.nflocks) M.count.resize(nflocks_new * PFNAV_NAV_LAYER_MAX, 0);
    for (const pf_cmd_change &c : changes) {
        if (M.flock[c.idx] >= 0) M.count[(size_t)M.flock[c.idx] * PFNAV_NAV_LAYER_MAX + M.layer[c.idx]]--;
        M.flock[c.idx] = c.flock; M.layer[c.idx] = c.layer;
        if (c.flock >= 0) M.count[(size_t)c.flock * PFNAV_NAV_LAYER_MAX + c.layer]++;
    }
    M.count.resize(nflocks_new * PFNAV_NAV_LAYER_MAX);         // a dropped tail holds no entity (pf_cmd_plan)
    M.nflocks = nflocks_new;
}

// ---- the job form (pfnav_mgpu_commands / pfnav_group_commands) ----
// Every member gets the job's whole batch. It applies the merged records of the uids it owns as the solo call does, and
// for every other uid writes only what no tick step changes -- the flock column entry and the neighbour record's radius
// and low 24 flag bits (k_make_records and k_entity_apply copy those from the agent unchanged) -- so that its flock
// column, radii and flag bits equal the owners' after the call. Position, velocity and state of other members' entities
// arrive with the next gather.
#define PF_DELTA_FOREIGN (PFNAV_DELTA_FLOCK | PFNAV_DELTA_RADIUS | PFNAV_DELTA_FLAGS)
struct pf_cmd_foreign { uint32_t uid, mask; int32_t flock; float radius; uint32_t flags; };     // mask: PF_DELTA_FOREIGN bits

PF_HD void pf_foreign_apply(const pf_cmd_foreign &f, int32_t &flock, float &radius, uint32_t &state_flags)
{
    if (f.mask & PFNAV_DELTA_FLOCK) flock = f.flock;
    if (f.mask & PFNAV_DELTA_RADIUS) radius = f.radius;
    if (f.mask & PFNAV_DELTA_FLAGS) state_flags = (state_flags & 0xFF000000u) | (f.flags & 0xFFFFFFu);
}

// A member's part of a job batch, changing nothing: validation of every delta against the population (L.lo = 0,
// L.hi = n_total), merging, the split into the merged records of the own range [lo, hi) and the foreign part of the
// others, and pf_cmd_plan of the own records on the member's mirror (layers and stranded flock indices, which only the
// owner can check). Returns NULL or what was wrong.
static inline const char *pf_cmd_job_plan(const pfnav_agent_delta *d, size_t n, const pf_cmd_limits &L, size_t lo, size_t hi,
                                          const pf_cmd_mirror &M, int nlayers, std::vector<pfnav_agent_delta> &own,
                                          std::vector<pf_cmd_foreign> &foreign, std::vector<pf_cmd_change> &changes)
{
    std::vector<pfnav_agent_delta> merged;
    own.clear(); foreign.clear(); changes.clear();
    if (const char *e = pf_cmd_merge(d, n, L, merged)) return e;
    for (const pfnav_agent_delta &m : merged) {
        if (m.uid >= lo && m.uid < hi) own.push_back(m);
        else if (m.mask & PF_DELTA_FOREIGN) foreign.push_back({m.uid, m.mask & PF_DELTA_FOREIGN, m.flock, m.radius, m.flags});
    }
    return pf_cmd_plan(M, lo, own, L.nflocks, nlayers, changes);
}
