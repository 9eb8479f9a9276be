// tests/emu/digest_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the state digests of
// permafrost-engine_b200/csrc/pfnav_digest_host.h (unmodified): the digests of checkpoint and pool segments that the
// device's pfnav_state_digest must equal, and the per-item terms, so that tests/test_digest_emu.py can check them against
// a numpy restatement. This is not a product path: nothing in libpfnav.so links or calls it, and it is built only by
// the tests.
#include <stdio.h>
#include "../../permafrost-engine_b200/csrc/pfnav_digest_host.h"

void pfnav_set_error(const char *, ...) {}

extern "C" {

size_t emu_dg_nblocks(size_t n_total, int k) { return pf_digest_nblocks(n_total, k); }

// pf_digest_agents_segment: out = {population, flocks, records}; blocks (may be NULL) is added to. 0, or 1 with the
// reason in err (256 bytes).
int emu_dg_agents(const uint8_t *seg, size_t size, int k, uint64_t *blocks, uint64_t *out, char *err)
{
    pf_digest_agents d;
    if (const char *e = pf_digest_agents_segment(seg, size, k, blocks, &d)) {
        snprintf(err, 256, "%s", e);
        return 1;
    }
    out[0] = d.population; out[1] = d.flocks; out[2] = d.records;
    return 0;
}

int emu_dg_pool(const uint8_t *seg, size_t size, uint64_t *out, char *err)
{
    if (const char *e = pf_digest_pool_segment(seg, size, out)) {
        snprintf(err, 256, "%s", e);
        return 1;
    }
    return 0;
}

uint64_t emu_dg_splitmix64(uint64_t x) { return pf_splitmix64(x); }

}
