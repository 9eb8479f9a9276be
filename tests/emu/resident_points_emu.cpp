// tests/emu/resident_points_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the host rule of the calls whose positions may
// name resident entities (pf_resident_points_check in permafrost-engine_b200/csrc/pfnav_resident_host.h, unmodified), so
// that tests/test_resident_requests_emu.py can run it on synthetic record arrays. The device's part (k_resident_xz: the
// x, z of each named record written over the given positions at a float stride and offset) is restated here on the host
// record array. This is not a product path: nothing in libpfnav.so links or calls it, and it is built only by
// tests/test_resident_requests_emu.py.
#include <string.h>
#include "../../permafrost-engine_b200/csrc/pfnav_resident_host.h"

static const char *g_err = "";

extern "C" {

const char *emu_last_error() { return g_err; }

// The check on n entries with uid arrays a and b (either may be NULL; given_a / given_b: the given positions exist),
// then the pairs' records (rec: 6 floats per entity {x, z, vx, vz, radius, state_flags}) written into buf at
// entry * stride + off_a (array a's pairs) or + off_b (array b's). Outputs are written only on success: out_entry and
// out_uid (the pairs, array a's first), *out_np, *out_n0 and buf.
int emu_points(size_t n, const uint32_t *uids_a, int given_a, const uint32_t *uids_b, int given_b, size_t population,
               const float *rec, int stride, int off_a, int off_b, float *buf, uint32_t *out_entry, uint32_t *out_uid,
               size_t *out_np, size_t *out_n0)
{
    pf_resident_points P;
    g_err = "";
    if (int rc = pf_resident_points_check(n, uids_a, given_a != 0, uids_b, given_b != 0, population, P, &g_err)) return rc;
    const size_t np = P.entry.size();
    std::vector<uint8_t> packed(P.bytes());
    P.pack(packed.data());
    const uint32_t *entry = (const uint32_t *)packed.data(), *uid = entry + np;
    for (size_t i = 0; i < np; i++) {
        float *p = buf + (size_t)entry[i] * stride + (i < P.n0 ? off_a : off_b);
        p[0] = rec[6 * (size_t)uid[i]];
        p[1] = rec[6 * (size_t)uid[i] + 1];
    }
    if (np) {
        memcpy(out_entry, entry, np * 4);
        memcpy(out_uid, uid, np * 4);
    }
    *out_np = np;
    *out_n0 = P.n0;
    return 0;
}

}
