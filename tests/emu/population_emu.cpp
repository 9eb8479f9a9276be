// tests/emu/population_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the host side of pfnav_agents_change_population
// (permafrost-engine_b200/csrc/pfnav_commands_host.h, unmodified): validation and planning of a batch, the numbering rule
// k_pop_gather runs per row (pf_pop_source, pf_pop_renumber, here on the CPU) and the compaction + append of the
// (flock, layer) mirror. This is not a product path: nothing in libpfnav.so links or calls it, and it is built only by
// tests/test_agent_population_emu.py.
#include <string.h>
#include <algorithm>
#include "../../permafrost-engine_b200/csrc/pfnav_commands_host.h"

extern "C" {

void *emu_mirror_new(const pfnav_agent *agents, int n, int nflocks)
{
    pf_cmd_mirror *M = new pf_cmd_mirror;
    M->reset((size_t)n, (size_t)nflocks);
    for (int i = 0; i < n; i++)
        M->set((size_t)i, std::max(agents[i].flock, -1), pf_layer_base(agents[i].flags) + pf_layer_class(agents[i].radius));
    return M;
}

void emu_mirror_delete(void *h) { delete (pf_cmd_mirror *)h; }

// tables: bit 0 movestate, 1 ext, 2 formation, 3 blocking. Plans the batch; commit != 0 also applies it to the mirror.
// -> the population after the call, or -1 with the reason in err (256 bytes; the mirror unchanged). src (room for
// n_keep): the old uid of every survivor row by pf_pop_source; renum (room for n_old + 1): pf_pop_renumber of every old
// uid and of PFNAV_NULL_UID; any_fac: whether an appended blocking record names a faction other than 15.
int emu_pop_batch(void *h, int nlayers, int tables, const uint32_t *rm, int nrm, const pfnav_agent *add, const pfnav_movestate *ms,
                  const pfnav_movestate_ext *ext, const pfnav_formation_in *form, const pfnav_blocking *blk, int nadd,
                  int nflocks_new, int commit, uint32_t *src, uint32_t *renum, int *any_fac, char *err)
{
    pf_cmd_mirror &M = *(pf_cmd_mirror *)h;
    const pf_pop_tables T = {(tables & 1) != 0, (tables & 2) != 0, (tables & 4) != 0, (tables & 8) != 0};
    pf_pop_plan P;
    if (const char *e = pf_pop_plan_batch(M, nlayers, T, rm, (size_t)nrm, add, ms, ext, form, blk, (size_t)nadd,
                                          (size_t)nflocks_new, P)) {
        strncpy(err, e, 255); err[255] = 0;
        return -1;
    }
    const uint32_t R = (uint32_t)P.removed.size();
    for (size_t j = 0; j < P.n_keep; j++) src[j] = pf_pop_source(P.key.data(), R, (uint32_t)j);
    for (size_t u = 0; u <= P.n_old; u++)
        renum[u] = pf_pop_renumber(P.removed.data(), R, (uint32_t)P.n_old, u < P.n_old ? (uint32_t)u : PFNAV_NULL_UID);
    *any_fac = P.add_any_fac ? 1 : 0;
    if (commit) M.compact_append(P.removed, P.add_flock.data(), P.add_layer.data(), (size_t)nadd, (size_t)nflocks_new);
    return (int)P.n_new;
}

// used: [nflocks][PFNAV_NAV_LAYER_MAX]; count: the same shape
void emu_mirror_state(void *h, int32_t *flock, uint8_t *layer, uint8_t *used, uint32_t *count)
{
    const pf_cmd_mirror &M = *(const pf_cmd_mirror *)h;
    std::copy(M.flock.begin(), M.flock.end(), flock);
    std::copy(M.layer.begin(), M.layer.end(), layer);
    std::vector<uint8_t> u;
    M.used(u);
    std::copy(u.begin(), u.end(), used);
    std::copy(M.count.begin(), M.count.end(), count);
}

int emu_mirror_size(void *h, int *nflocks) { *nflocks = (int)((pf_cmd_mirror *)h)->nflocks; return (int)((pf_cmd_mirror *)h)->flock.size(); }

}
