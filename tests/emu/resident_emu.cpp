// tests/emu/resident_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the host rule of the entity-field batches named by uid
// (permafrost-engine_b200/csrc/pfnav_resident_host.h, unmodified), so that tests/test_entity_fields_resident_emu.py can
// run it on synthetic record arrays. The device's part (k_resident_footprints: {x, z, radius} of a record, the chunk
// under its position) is restated here on the host record array. This is not a product path: nothing in libpfnav.so
// links or calls it, and it is built only by tests/test_entity_fields_resident_emu.py.
#include <string.h>
#include "../../permafrost-engine_b200/csrc/pfnav_resident_host.h"

static const char *g_err = "";

extern "C" {

const char *emu_last_error() { return g_err; }

// rec: 6 floats per entity {x, z, vx, vz, radius, state_flags}; seek_chunk_of[uid]: the chunk under the entity or -1.
// Outputs are written only on success: out_reqs (m), out_ents (nents), out_chunks (cap_chunks pairs) and *out_nchunks.
// *out_kept: the batch the rule writes into still holds what it held before the call (the error case's promise).
int emu_resolve(const pfnav_entity_field_req *reqs, size_t m, const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents,
                const uint32_t *seeker_uids, size_t nseekers, const float *rec, const int32_t *chunk_of, size_t population,
                int chunk_w, int chunk_h, pfnav_entity_field_req *out_reqs, pfnav_footprint *out_ents, int32_t *out_chunks,
                size_t cap_chunks, size_t *out_nchunks, int *out_kept)
{
    pf_resident_names N;
    g_err = "";
    int rc = pf_resident_check(reqs, m, ents, ent_uids, nents, seeker_uids, nseekers, population, N, &g_err);
    if (rc) return rc;
    if (m == 0) { *out_nchunks = 0; return 0; }
    const size_t nfp = N.fp_index.size();
    std::vector<float> xzr(3 * nfp);
    std::vector<int32_t> ch(nseekers);
    for (size_t k = 0; k < N.uids.size(); k++) {
        const float *r = rec + 6 * (size_t)N.uids[k];
        if (k < nfp) { xzr[3 * k] = r[0]; xzr[3 * k + 1] = r[1]; xzr[3 * k + 2] = r[4]; }
        else ch[k - nfp] = chunk_of[N.uids[k]];
    }
    pf_resident_batch B;
    B.reqs.assign(1, pfnav_entity_field_req{7, 7, 7, 7, 7, 7, 7, 7});
    B.ents.assign(1, pfnav_footprint{});
    B.chunks_rc.assign(2, 7);
    rc = pf_resident_merge(reqs, m, ents, nents, N, xzr.data(), ch.data(), nseekers, chunk_w, chunk_h, B, &g_err);
    *out_kept = B.reqs.size() == 1 && B.reqs[0].dest == 7 && B.ents.size() == 1 && B.chunks_rc.size() == 2;
    if (rc) return rc;
    if (B.chunks_rc.size() / 2 > cap_chunks) return -100;
    memcpy(out_reqs, B.reqs.data(), m * sizeof(pfnav_entity_field_req));
    if (nents) memcpy(out_ents, B.ents.data(), nents * sizeof(pfnav_footprint));
    if (!B.chunks_rc.empty()) memcpy(out_chunks, B.chunks_rc.data(), B.chunks_rc.size() * 4);
    *out_nchunks = B.chunks_rc.size() / 2;
    return 0;
}

}
