// tests/emu/population_job_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the job form of a population change in
// permafrost-engine_b200/csrc/pfnav_commands_host.h (unmodified): a member's validation and plan (pf_pop_job_plan), the
// segments and appended runs it derives, its mirror after the call (pf_pop_job_mirror), and the solo path they must agree
// with (pf_pop_plan_batch, compact_append). This is not a product path: nothing in libpfnav.so links or calls it, and it
// is built only by tests/test_agent_population_job_emu.py.
#include <string.h>
#include <algorithm>
#include "../../permafrost-engine_b200/csrc/pfnav_commands_host.h"

extern "C" {

static int fail(const char *e, char *err)
{
    strncpy(err, e, 255); err[255] = 0;
    return -1;
}

// (flock, layer) mirror of agents[0 .. n): one member's own range, or the whole population
void *emu_mirror_new(const pfnav_agent *agents, int n, int nflocks)
{
    pf_cmd_mirror *M = new pf_cmd_mirror;
    M->reset((size_t)n, (size_t)nflocks);
    for (int i = 0; i < n; i++)
        M->set((size_t)i, std::max(agents[i].flock, -1), pf_layer_base(agents[i].flags) + pf_layer_class(agents[i].radius));
    return M;
}

void emu_mirror_delete(void *h) { delete (pf_cmd_mirror *)h; }

// used: [nflocks][PFNAV_NAV_LAYER_MAX]
void emu_mirror_state(void *h, int32_t *flock, uint8_t *layer, uint8_t *used)
{
    const pf_cmd_mirror &M = *(const pf_cmd_mirror *)h;
    std::copy(M.flock.begin(), M.flock.end(), flock);
    std::copy(M.layer.begin(), M.layer.end(), layer);
    std::vector<uint8_t> u;
    M.used(u);
    std::copy(u.begin(), u.end(), used);
}

static pf_pop_tables tables_of(int t) { return {(t & 1) != 0, (t & 2) != 0, (t & 4) != 0, (t & 8) != 0}; }

// The solo call on a whole-population mirror, committed when it passes -> the population after the call, or -1
int emu_solo(void *h, int nlayers, int tables, const uint32_t *rm, int nrm, const pfnav_agent *add, const pfnav_movestate *ms,
             const pfnav_movestate_ext *ext, const pfnav_formation_in *form, const pfnav_blocking *blk, int nadd, int nflocks_new,
             char *err)
{
    pf_cmd_mirror &M = *(pf_cmd_mirror *)h;
    pf_pop_plan P;
    if (const char *e = pf_pop_plan_batch(M, nlayers, tables_of(tables), rm, (size_t)nrm, add, ms, ext, form, blk, (size_t)nadd,
                                          (size_t)nflocks_new, P))
        return fail(e, err);
    M.compact_append(P.removed, P.add_flock.data(), P.add_layer.data(), (size_t)nadd, (size_t)nflocks_new);
    return (int)P.n_new;
}

// Member `rank` of `world`, its mirror h over its old range of a population of n_old: pf_pop_job_plan -> 0, or -1 with
// the reason in err (nothing changed). bounds (3 * (world + 1)): old_lo, new_lo, keep_lo; seg (2 * world * world): the
// new-uid run [lo, hi) of segment (sender s, receiver r) at 2 * (s * world + r); app (2 * world): the appended run of
// every member. commit != 0 replaces the mirror by pf_pop_job_mirror, the received rows read from col_flock, col_radius
// and col_sf: the compacted columns of the whole new population, as the member holds them on its device.
int emu_job_member(void *h, int n_old, int world, int rank, int nlayers, int tables, const uint32_t *rm, int nrm,
                   const pfnav_agent *add, const pfnav_movestate *ms, const pfnav_movestate_ext *ext,
                   const pfnav_formation_in *form, const pfnav_blocking *blk, int nadd, int nflocks_new,
                   const int32_t *col_flock, const float *col_radius, const uint32_t *col_sf, int commit, int64_t *bounds,
                   int64_t *seg, int64_t *app, char *err)
{
    pf_cmd_mirror &M = *(pf_cmd_mirror *)h;
    pf_pop_job J;
    if (const char *e = pf_pop_job_plan(M, (size_t)n_old, world, rank, nlayers, tables_of(tables), rm, (size_t)nrm, add, ms,
                                        ext, form, blk, (size_t)nadd, (size_t)nflocks_new, J))
        return fail(e, err);
    for (int r = 0; r <= world; r++) {
        bounds[r] = (int64_t)J.old_lo[r];
        bounds[world + 1 + r] = (int64_t)J.new_lo[r];
        bounds[2 * (world + 1) + r] = (int64_t)J.keep_lo[r];
    }
    for (int s = 0; s < world; s++)
        for (int r = 0; r < world; r++) {
            seg[2 * (s * world + r)] = (int64_t)J.seg_lo(s, r);
            seg[2 * (s * world + r) + 1] = (int64_t)J.seg_hi(s, r);
        }
    for (int r = 0; r < world; r++) { app[2 * r] = (int64_t)J.app_lo(r); app[2 * r + 1] = (int64_t)J.app_hi(r); }
    if (commit) {
        std::vector<int32_t> f;
        std::vector<float> rad;
        std::vector<uint32_t> sf;
        for (int s = 0; s < world; s++) {
            if (s == rank) continue;
            for (size_t j = J.seg_lo(s, rank); j < J.seg_hi(s, rank); j++) {
                f.push_back(col_flock[j]); rad.push_back(col_radius[j]); sf.push_back(col_sf[j]);
            }
        }
        pf_pop_job_mirror(M, J, f.data(), rad.data(), sf.data(), M);
    }
    return 0;
}

}
