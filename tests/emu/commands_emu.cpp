// tests/emu/commands_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the host side of pfnav_agents_commands
// (permafrost-engine_b200/csrc/pfnav_commands_host.h, unmodified): delta validation, per-uid merging, the write rule
// k_apply_deltas runs per entity (pf_delta_apply, here on the CPU) and the (flock, layer) mirror. This is not a product
// path: nothing in libpfnav.so links or calls it, and it is built only by tests/test_agent_commands_emu.py.
#include <string.h>
#include <algorithm>
#include "../../permafrost-engine_b200/csrc/pfnav_commands_host.h"

extern "C" {

// -> the number of merged records written to out (room for n), or -1 with the reason in err (256 bytes)
int emu_cmd_merge(const pfnav_agent_delta *d, int n, int lo, int hi, int n_agents, int nflocks, int have_ms, int have_ext,
                  pfnav_agent_delta *out, char *err)
{
    const pf_cmd_limits L = {(size_t)lo, (size_t)hi, (size_t)n_agents, (size_t)nflocks, have_ms != 0, have_ext != 0};
    std::vector<pfnav_agent_delta> m;
    if (const char *e = pf_cmd_merge(d, (size_t)n, L, m)) { strncpy(err, e, 255); err[255] = 0; return -1; }
    if (!m.empty()) memcpy(out, m.data(), m.size() * sizeof(pfnav_agent_delta));
    return (int)m.size();
}

// the records in array order, each on the entity its uid names (tables indexed by uid)
void emu_cmd_apply(pfnav_agent *agents, pfnav_movestate *ms, pfnav_movestate_ext *ext, const pfnav_agent_delta *d, int n)
{
    for (int i = 0; i < n; i++) pf_delta_apply(agents + d[i].uid, ms + d[i].uid, ext + d[i].uid, d[i]);
}

int emu_layer(uint32_t flags, float radius) { return pf_layer_base(flags) + pf_layer_class(radius); }

void *emu_mirror_new(const pfnav_agent *agents, int n, int nflocks)
{
    pf_cmd_mirror *M = new pf_cmd_mirror;
    M->reset((size_t)n, (size_t)nflocks);
    for (int i = 0; i < n; i++) M->set((size_t)i, agents[i].flock, emu_layer(agents[i].flags, agents[i].radius));
    return M;
}

void emu_mirror_delete(void *h) { delete (pf_cmd_mirror *)h; }

// plan + commit of one merged batch -> 0, or -1 (nothing changed) with the reason in err
int emu_mirror_batch(void *h, const pfnav_agent_delta *merged, int n, int nflocks_new, int nlayers, char *err)
{
    pf_cmd_mirror &M = *(pf_cmd_mirror *)h;
    std::vector<pfnav_agent_delta> m(merged, merged + n);
    std::vector<pf_cmd_change> ch;
    if (const char *e = pf_cmd_plan(M, 0, m, (size_t)nflocks_new, nlayers, ch)) { strncpy(err, e, 255); err[255] = 0; return -1; }
    pf_cmd_commit(M, ch, (size_t)nflocks_new);
    return 0;
}

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

}
