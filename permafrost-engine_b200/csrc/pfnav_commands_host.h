// pfnav_commands_host.h -- the host side of pfnav_agents_commands and the write rule its kernel applies, CUDA-free:
// delta validation, per-uid merging in array order, the navigation layer rule and the (flock, layer) mirror that keeps
// flock_layer_used equal to a fresh upload's; and the split of a multi-GPU job's batch into a member's own and foreign
// parts; and the validation, numbering rule and mirror update of pfnav_agents_change_population, and its job form's
// ranges, segments and member mirror. tests/emu/commands_emu.cpp, tests/emu/commands_job_emu.cpp,
// tests/emu/population_emu.cpp and tests/emu/population_job_emu.cpp build this header with g++.
#pragma once
#include <math.h>
#include <algorithm>
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

// The per-entity checks of an agent record that pfnav_agents_upload and pfnav_agents_change_population both make: its
// flock index below the length of the flock table it will be read against, and its navigation layer created. *layer:
// that layer. Returns NULL or what was wrong.
static inline const char *pf_agent_check(const pfnav_agent &a, size_t nflocks, int nlayers, int *layer)
{
    if (a.flock >= (int64_t)nflocks) return "agent flock index out of range";
    *layer = pf_layer_base(a.flags) + pf_layer_class(a.radius);
    if (*layer >= nlayers) return "agent needs a navigation layer that was not created (radius/flags)";
    return nullptr;
}

// pfnav_agents_upload_blocking's check of one record
static inline const char *pf_blocking_check(const pfnav_blocking &b)
{
    if (b.blocking > 1) return "blocking must be 0 or 1";
    if (b.faction_id < 0 || b.faction_id > 15) return "faction_id must lie in 0..15";
    return nullptr;
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
    // pfnav_agents_change_population: drop the entities `removed` names (sorted, unique), keep the others in order, append
    // (flock[k], layer[k]) for k < nadd, and resize the counts to a table of nflocks_new flocks, which holds every flock
    // index left (pf_pop_plan checked it)
    void compact_append(const std::vector<uint32_t> &removed, const int32_t *add_flock, const uint8_t *add_layer, size_t nadd,
                        size_t nflocks_new)
    {
        if (nflocks_new > nflocks) count.resize(nflocks_new * PFNAV_NAV_LAYER_MAX, 0);
        size_t w = 0, m = 0;
        for (size_t i = 0; i < flock.size(); i++) {
            if (m < removed.size() && removed[m] == i) {
                if (flock[i] >= 0) count[(size_t)flock[i] * PFNAV_NAV_LAYER_MAX + layer[i]]--;
                m++;
                continue;
            }
            flock[w] = flock[i]; layer[w] = layer[i]; w++;
        }
        flock.resize(w + nadd); layer.resize(w + nadd);
        for (size_t k = 0; k < nadd; k++) set(w + k, add_flock[k] < 0 ? -1 : add_flock[k], add_layer[k]);
        count.resize(nflocks_new * PFNAV_NAV_LAYER_MAX);
        nflocks = nflocks_new;
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

// ---- pfnav_agents_change_population ----
// The numbering rule is a stable compaction followed by an append: survivor u gets u - |{removed r < u}|, appended
// entity k gets n_keep + k. removed: the removed uids, sorted and unique; key[m] = removed[m] - m, the number of
// survivors before removed[m] (non-decreasing).
// New row j < n_keep: the uid it had before the call, j plus the number of removals with key <= j.
PF_HD uint32_t pf_pop_source(const uint32_t *key, uint32_t R, uint32_t j)
{
    uint32_t lo = 0, hi = R;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (key[mid] <= j) lo = mid + 1; else hi = mid; }
    return j + lo;
}
// A uid of the population before the call (n_old entities) -> its uid after the call; PFNAV_NULL_UID when it was
// removed or names no entity.
PF_HD uint32_t pf_pop_renumber(const uint32_t *removed, uint32_t R, uint32_t n_old, uint32_t u)
{
    if (u >= n_old) return PFNAV_NULL_UID;
    uint32_t lo = 0, hi = R;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (removed[mid] < u) lo = mid + 1; else hi = mid; }
    return lo < R && removed[lo] == u ? PFNAV_NULL_UID : u - lo;
}

// the optional tables a population change writes (blocking: a blocking table covers the population)
struct pf_pop_tables { bool ms, ext, formation, blocking; };

struct pf_pop_plan {
    std::vector<uint32_t> removed, key;       // sorted unique removals and their keys (pf_pop_source)
    std::vector<int32_t> add_flock;           // flock and navigation layer of every appended entity, for the mirror
    std::vector<uint8_t> add_layer;
    size_t n_old = 0, n_keep = 0, n_new = 0, nflocks = 0;
    bool add_any_fac = false;                 // an appended blocking record names a faction other than 15
};

static inline bool pf_finite(const float *p, int n)
{
    for (int i = 0; i < n; i++)
        if (!isfinite(p[i])) return false;
    return true;
}

// Validate a population change against the mirror of the population (n_old entities) and plan it, changing nothing:
// removal uids in range (repeats removed once), appended records for exactly the tables that exist (ext and formation
// optional, movestate and blocking required), the upload's checks of appended agents and blocking records against the
// flock table after the call (nflocks_new), finite floats, appended ext targets inside the new population, and no
// survivor left with a flock index the new table drops. Returns NULL or what was wrong.
// M mirrors the entities [lo, lo + M.flock.size()) of a population of n_old: the whole population for the solo call, a
// job member's own range for the job form, where only the stranded flock indices of that range are checked.
static inline const char *pf_pop_plan_range(const pf_cmd_mirror &M, size_t lo, size_t n_old, int nlayers, const pf_pop_tables &T,
                                            const uint32_t *rm, size_t nrm, const pfnav_agent *add, const pfnav_movestate *add_ms,
                                            const pfnav_movestate_ext *add_ext, const pfnav_formation_in *add_form,
                                            const pfnav_blocking *add_blk, size_t nadd, size_t nflocks_new, pf_pop_plan &P)
{
    if (!rm && nrm) return "remove_uids == NULL";
    if (!add && nadd) return "add == NULL";
    if (add_ms && !T.ms) return "movestate records for a table that was not uploaded";
    if (add_ext && !T.ext) return "movestate_ext records for a table that was not uploaded";
    if (add_form && !T.formation) return "formation records for a table that was not uploaded";
    if (add_blk && !T.blocking) return "blocking records without a blocking table for the population";
    if (nadd && T.ms && !add_ms) return "appended entities need movestate records: a movestate table was uploaded";
    if (nadd && T.blocking && !add_blk) return "appended entities need blocking records: a blocking table covers the population";
    P.removed.assign(rm, rm + nrm);
    for (uint32_t u : P.removed)
        if (u >= n_old) return "remove uid outside the population";
    std::sort(P.removed.begin(), P.removed.end());
    P.removed.erase(std::unique(P.removed.begin(), P.removed.end()), P.removed.end());
    const size_t R = P.removed.size();
    P.n_old = n_old; P.n_keep = n_old - R; P.n_new = P.n_keep + nadd; P.nflocks = nflocks_new;
    if (P.n_new >= (1u << 31)) return "population too large";
    P.key.resize(R);
    for (size_t m = 0; m < R; m++) P.key[m] = P.removed[m] - (uint32_t)m;
    P.add_flock.resize(nadd); P.add_layer.resize(nadd);
    P.add_any_fac = false;
    for (size_t k = 0; k < nadd; k++) {
        int layer;
        if (const char *e = pf_agent_check(add[k], nflocks_new, nlayers, &layer)) return e;
        if (!pf_finite(add[k].pos, 11)) return "appended agent with a float that is not finite";      // pos .. speed
        P.add_flock[k] = add[k].flock; P.add_layer[k] = (uint8_t)layer;
        if (add_ms && !pf_finite(add_ms[k].next_pos, 40)) return "appended movestate with a float that is not finite";
        if (add_ext) {
            const pfnav_movestate_ext &x = add_ext[k];
            if (x.surround_target_uid != PFNAV_NULL_UID && x.surround_target_uid >= P.n_new)
                return "appended movestate_ext target outside the population after the call";
            if (!pf_finite(&x.target_range, 3) || !pf_finite(x.target_dir, 8)) return "appended movestate_ext with a float that is not finite";
        }
        if (add_form && !pf_finite(add_form[k].cell_pos, 14)) return "appended formation record with a float that is not finite";
        if (add_blk) {
            if (const char *e = pf_blocking_check(add_blk[k])) return e;
            if (!pf_finite(&add_blk[k].stop_x, 3)) return "appended blocking record with a float that is not finite";
            P.add_any_fac |= add_blk[k].faction_id < 15;
        }
    }
    int64_t stranded = 0;
    for (size_t f = nflocks_new; f < M.nflocks; f++)
        for (int l = 0; l < PFNAV_NAV_LAYER_MAX; l++) stranded += M.count[f * PFNAV_NAV_LAYER_MAX + l];
    for (uint32_t u : P.removed)
        if (u >= lo && u - lo < M.flock.size() && M.flock[u - lo] >= (int64_t)nflocks_new) stranded--;
    if (stranded > 0) return "the new flock table is shorter than the flock index some surviving entity keeps";
    return nullptr;
}

static inline const char *pf_pop_plan_batch(const pf_cmd_mirror &M, int nlayers, const pf_pop_tables &T,
                                            const uint32_t *rm, size_t nrm, const pfnav_agent *add, const pfnav_movestate *add_ms,
                                            const pfnav_movestate_ext *add_ext, const pfnav_formation_in *add_form,
                                            const pfnav_blocking *add_blk, size_t nadd, size_t nflocks_new, pf_pop_plan &P)
{
    return pf_pop_plan_range(M, 0, M.flock.size(), nlayers, T, rm, nrm, add, add_ms, add_ext, add_form, add_blk, nadd,
                             nflocks_new, P);
}

// ---- the job form of a population change (pfnav_mgpu_change_population / pfnav_group_change_population) ----
// Every member gets the job's whole batch and derives the same plan from it. Member r owns the balanced range
// [old_lo[r], old_lo[r + 1]) before the call and [new_lo[r], new_lo[r + 1]) after it. Compaction keeps order, so the
// survivors of member s occupy the contiguous new uids [keep_lo[s], keep_lo[s + 1]); the part of that run inside r's new
// range is the one segment s sends r (s == r: the own survivors that stay). Appended entities [n_keep, n_new) are written
// by the member whose new range holds them.
struct pf_pop_job {
    pf_pop_plan P;
    int world = 1, rank = 0;
    std::vector<size_t> old_lo, new_lo, keep_lo;      // world + 1 boundaries each
    size_t seg_lo(int s, int r) const { return std::min(std::max(keep_lo[s], new_lo[r]), new_lo[r + 1]); }
    size_t seg_hi(int s, int r) const { return std::max(seg_lo(s, r), std::min(keep_lo[s + 1], new_lo[r + 1])); }
    size_t app_lo(int r) const { return std::min(std::max(P.n_keep, new_lo[r]), new_lo[r + 1]); }
    size_t app_hi(int r) const { return new_lo[r + 1]; }
};

// pfnav_mgpu_shard_range's balanced split of n entities over world members, as world + 1 boundaries
static inline void pf_balanced_bounds(size_t n, int world, std::vector<size_t> &b)
{
    b.resize((size_t)world + 1);
    const size_t base = n / world, rem = n % world;
    for (int r = 0; r <= world; r++) b[r] = (size_t)r * base + std::min<size_t>(r, rem);
}

// A member's part of a job's population change, changing nothing: the solo validation with the member's mirror M of its
// own range (removal range, appended records, tables present, stranded flock indices of its own entities), then the
// ranges and segments of every member. Returns NULL or what was wrong.
static inline const char *pf_pop_job_plan(const pf_cmd_mirror &M, size_t n_old, int world, int rank, int nlayers,
                                          const pf_pop_tables &T, const uint32_t *rm, size_t nrm, const pfnav_agent *add,
                                          const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext,
                                          const pfnav_formation_in *add_form, const pfnav_blocking *add_blk, size_t nadd,
                                          size_t nflocks_new, pf_pop_job &J)
{
    J.world = world; J.rank = rank;
    pf_balanced_bounds(n_old, world, J.old_lo);
    if (M.flock.size() != J.old_lo[rank + 1] - J.old_lo[rank]) return "the member does not hold its balanced range";
    if (const char *e = pf_pop_plan_range(M, J.old_lo[rank], n_old, nlayers, T, rm, nrm, add, add_ms, add_ext, add_form,
                                          add_blk, nadd, nflocks_new, J.P))
        return e;
    pf_balanced_bounds(J.P.n_new, world, J.new_lo);
    J.keep_lo.resize((size_t)world + 1);
    for (int r = 0; r <= world; r++) {
        const size_t u = J.old_lo[r];
        J.keep_lo[r] = u - (size_t)(std::lower_bound(J.P.removed.begin(), J.P.removed.end(), (uint32_t)u) - J.P.removed.begin());
    }
    return nullptr;
}

// The member's mirror after the call, over its new range: its own survivors that stay keep their entries, appended
// entities take pf_pop_plan::add_flock / add_layer, and the k-th received row (in uid order: the segments of the senders
// in rank order) takes flock[k] and the layer of radius[k] and state_flags[k] (the record's state << 24 | flags) by
// pf_agent_check's rule: the member's own copies of those columns after compaction, current on every member.
static inline void pf_pop_job_mirror(const pf_cmd_mirror &M, const pf_pop_job &J, const int32_t *flock, const float *radius,
                                     const uint32_t *state_flags, pf_cmd_mirror &out)
{
    const int r = J.rank;
    const size_t lo = J.new_lo[r], hi = J.new_lo[r + 1];
    const size_t s0 = J.seg_lo(r, r), s1 = J.seg_hi(r, r);
    pf_cmd_mirror N;
    N.reset(hi - lo, J.P.nflocks);
    size_t k = 0;
    for (size_t j = lo; j < hi; j++) {
        if (j >= J.P.n_keep) {
            const size_t a = j - J.P.n_keep;
            N.set(j - lo, std::max(J.P.add_flock[a], -1), J.P.add_layer[a]);
        } else if (j >= s0 && j < s1) {
            const size_t i = pf_pop_source(J.P.key.data(), (uint32_t)J.P.removed.size(), (uint32_t)j) - J.old_lo[r];
            N.set(j - lo, M.flock[i], M.layer[i]);
        } else {
            const uint32_t f = state_flags[k] & 0xFFFFFFu;
            N.set(j - lo, std::max(flock[k], -1), pf_layer_base(f) + pf_layer_class(radius[k]));
            k++;
        }
    }
    out = std::move(N);
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
