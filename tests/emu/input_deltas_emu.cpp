// tests/emu/input_deltas_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the host side of pfnav_agents_input_deltas
// (permafrost-engine_b200/csrc/pfnav_inputs_host.h, unmodified): record validation, per-uid folding, the job split and
// the write rule k_apply_input_deltas runs per entity (pf_input_apply, here on the CPU). This is not a product path:
// nothing in libpfnav.so links or calls it, and it is built only by tests/test_input_deltas_emu.py.
#include <string.h>
#include "../../permafrost-engine_b200/csrc/pfnav_inputs_host.h"

extern "C" {

static int fail(const char *e, char *err) { strncpy(err, e, 255); err[255] = 0; return -1; }

// -> the number of folded records written to out (room for n), or -1 with the reason in err (256 bytes)
int emu_input_merge(const pfnav_input_delta *d, int n, int lo, int hi, int have_ext, pfnav_input_delta *out, char *err)
{
    const pf_input_limits L = {(size_t)lo, (size_t)hi, have_ext != 0};
    std::vector<pfnav_input_delta> m;
    if (const char *e = pf_input_merge(d, (size_t)n, L, m)) return fail(e, err);
    if (!m.empty()) memcpy(out, m.data(), m.size() * sizeof(pfnav_input_delta));
    return (int)m.size();
}

// a job member owning [lo, hi) of n_total: -> the number of own folded records, *any_form, or -1 with the reason
int emu_input_job(const pfnav_input_delta *d, int n, int n_total, int lo, int hi, int have_ext, pfnav_input_delta *out,
                  int *any_form, char *err)
{
    const pf_input_limits L = {0, (size_t)n_total, have_ext != 0};
    std::vector<pfnav_input_delta> own;
    bool af = false;
    if (const char *e = pf_input_job_plan(d, (size_t)n, L, (size_t)lo, (size_t)hi, own, af)) return fail(e, err);
    if (!own.empty()) memcpy(out, own.data(), own.size() * sizeof(pfnav_input_delta));
    *any_form = af ? 1 : 0;
    return (int)own.size();
}

// the records in array order, each on the entity its uid names (tables indexed by uid - base)
void emu_input_apply(pfnav_movestate_ext *ext, pfnav_formation_in *form, const pfnav_input_delta *d, int n, int base)
{
    for (int i = 0; i < n; i++) pf_input_apply(ext + (d[i].uid - base), form + (d[i].uid - base), d[i]);
}

}
