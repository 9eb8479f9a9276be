// tests/emu/commands_job_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the job form of the command batch in
// permafrost-engine_b200/csrc/pfnav_commands_host.h (unmodified): a member's validation, split and mirror plan
// (pf_cmd_job_plan), the foreign write rule k_apply_foreign runs (pf_foreign_apply, here on the CPU), and the solo path
// they must agree with. This is not a product path: nothing in libpfnav.so links or calls it, and it is built only by
// tests/test_mgpu_commands_emu.py.
#include <string.h>
#include <algorithm>
#include "../../permafrost-engine_b200/csrc/pfnav_commands_host.h"

extern "C" {

static int fail(const char *e, char *err)
{
    strncpy(err, e, 255); err[255] = 0;
    return -1;
}

// (flock, layer) mirror of the entities agents[0 .. n) (one member's own range, or the whole population)
void *emu_mirror_new(const pfnav_agent *agents, int n, int nflocks)
{
    pf_cmd_mirror *M = new pf_cmd_mirror;
    M->reset((size_t)n, (size_t)nflocks);
    for (int i = 0; i < n; i++)
        M->set((size_t)i, agents[i].flock, pf_layer_base(agents[i].flags) + pf_layer_class(agents[i].radius));
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

// The solo call on a whole-population mirror: merge + plan, and the commit when commit != 0 -> the number of merged
// records written to `merged` (room for n), or -1 (nothing changed) with the reason in err (256 bytes)
int emu_solo(const pfnav_agent_delta *d, int n, int n_agents, int nflocks_new, int have_ms, int have_ext, void *mirror,
             int nlayers, int commit, pfnav_agent_delta *merged, char *err)
{
    const pf_cmd_limits L = {0, (size_t)n_agents, (size_t)n_agents, (size_t)nflocks_new, have_ms != 0, have_ext != 0};
    std::vector<pfnav_agent_delta> m;
    std::vector<pf_cmd_change> ch;
    if (const char *e = pf_cmd_merge(d, (size_t)n, L, m)) return fail(e, err);
    if (const char *e = pf_cmd_plan(*(pf_cmd_mirror *)mirror, 0, m, (size_t)nflocks_new, nlayers, ch)) return fail(e, err);
    if (commit) pf_cmd_commit(*(pf_cmd_mirror *)mirror, ch, (size_t)nflocks_new);
    if (!m.empty()) memcpy(merged, m.data(), m.size() * sizeof(pfnav_agent_delta));
    return (int)m.size();
}

// The member holding [lo, hi): pf_cmd_job_plan on its mirror, and the commit when commit != 0 -> 0 with the own records
// in own[0 .. *n_own) and the foreign ones in foreign[0 .. *n_foreign) (room for n each), or -1 (nothing changed)
int emu_job_member(const pfnav_agent_delta *d, int n, int n_agents, int nflocks_new, int have_ms, int have_ext, int lo, int hi,
                   void *mirror, int nlayers, int commit, pfnav_agent_delta *own, int *n_own, pf_cmd_foreign *foreign,
                   int *n_foreign, char *err)
{
    const pf_cmd_limits L = {0, (size_t)n_agents, (size_t)n_agents, (size_t)nflocks_new, have_ms != 0, have_ext != 0};
    std::vector<pfnav_agent_delta> o;
    std::vector<pf_cmd_foreign> f;
    std::vector<pf_cmd_change> ch;
    if (const char *e = pf_cmd_job_plan(d, (size_t)n, L, (size_t)lo, (size_t)hi, *(pf_cmd_mirror *)mirror, nlayers, o, f, ch))
        return fail(e, err);
    if (commit) pf_cmd_commit(*(pf_cmd_mirror *)mirror, ch, (size_t)nflocks_new);
    if (!o.empty()) memcpy(own, o.data(), o.size() * sizeof(pfnav_agent_delta));
    if (!f.empty()) memcpy(foreign, f.data(), f.size() * sizeof(pf_cmd_foreign));
    *n_own = (int)o.size(); *n_foreign = (int)f.size();
    return 0;
}

// k_apply_deltas' entity writes (tables indexed by uid), followed by the record fields it packs
void emu_apply_own(pfnav_agent *agents, pfnav_movestate *ms, pfnav_movestate_ext *ext, const pfnav_agent_delta *d, int n,
                   int32_t *flock_of, float *radius, uint32_t *state_flags)
{
    for (int i = 0; i < n; i++) {
        const uint32_t u = d[i].uid;
        pf_delta_apply(agents + u, ms + u, ext + u, d[i]);
        flock_of[u] = agents[u].flock;
        radius[u] = agents[u].radius;
        state_flags[u] = (agents[u].state << 24) | (agents[u].flags & 0xFFFFFFu);
    }
}

// k_apply_foreign's writes on the columns of the neighbour records
void emu_apply_foreign(const pf_cmd_foreign *f, int n, int32_t *flock_of, float *radius, uint32_t *state_flags)
{
    for (int i = 0; i < n; i++) pf_foreign_apply(f[i], flock_of[f[i].uid], radius[f[i].uid], state_flags[f[i].uid]);
}

int emu_foreign_size(void) { return (int)sizeof(pf_cmd_foreign); }

}
