// pfnav_resident_host.h -- the host rules of the calls that name resident entities by uid, CUDA-free:
// - pfnav_pool_request_entity_fields_resident and its job forms: the checks of the uid arguments, and the turn of what
//   k_resident_footprints resolves from the records into the inputs of pfnav_pool_request_entity_fields_batch
//   (footprints merged with the given ones, each request's seekers as the chunks under them, first seen first, each
//   once). tests/emu/resident_emu.cpp builds this part with g++.
// - pfnav_pool_request_paths_resident, pfnav_map_query_resident and pfnav_group_arrival_velocity_resident: the checks
//   of their uid arrays and the (entry, uid) pairs whose positions k_resident_xz writes over the given ones.
//   tests/emu/resident_points_emu.cpp builds this part with g++.
#pragma once
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../include/pfnav.h"

#define PF_RES_ARG(cond, msg) do { if (!(cond)) { *err = msg; return PFNAV_ERR_ARG; } } while (0)

// The uids the device resolves: the footprint entries that name one (their indices into ents, ascending) and then
// every seeker, in the argument order.
struct pf_resident_names {
    std::vector<uint32_t> fp_index;
    std::vector<uint32_t> uids;          // fp_index.size() footprint uids, then the seekers
};
// The inputs of pfnav_pool_request_entity_fields_batch: m requests, nents footprints, chunks_rc.size() / 2 chunks.
struct pf_resident_batch {
    std::vector<pfnav_entity_field_req> reqs;
    std::vector<pfnav_footprint> ents;
    std::vector<int32_t> chunks_rc;
};

// Entries 0 .. n-1 of one argument array whose values may name resident entities: entry k names uids[k] unless uids is
// NULL or uids[k] == PFNAV_NULL_UID, and then the caller's given value stands, which needs `given` (the array of given
// values is not NULL). Appends each naming entry's index to `entry` and its uid to `uid`, in order. PFNAV_ERR_ARG with
// *err = no_given or outside: an entry that names nothing without a given value, or a uid not below `population`.
static inline int pf_resident_named(const uint32_t *uids, size_t n, bool given, size_t population, std::vector<uint32_t> &entry,
                                    std::vector<uint32_t> &uid, const char *no_given, const char *outside, const char **err)
{
    for (size_t k = 0; k < n; k++) {
        const uint32_t u = uids ? uids[k] : PFNAV_NULL_UID;
        if (u == PFNAV_NULL_UID) {
            PF_RES_ARG(given, no_given);
            continue;
        }
        PF_RES_ARG(u < population, outside);
        entry.push_back((uint32_t)k);
        uid.push_back(u);
    }
    return PFNAV_OK;
}

// Checks what the uid arguments add to the batch's own validation: the non-NULL rules (ents may be NULL only when every
// entry names a uid), nents and nseekers below 2^24, every uid below `population`, and every request's footprint and
// seeker range inside its array. Fills N. PFNAV_ERR_ARG with *err naming the check; N is then unspecified.
static inline int pf_resident_check(const pfnav_entity_field_req *reqs, size_t m, const pfnav_footprint *ents,
                                    const uint32_t *ent_uids, size_t nents, const uint32_t *seeker_uids, size_t nseekers,
                                    size_t population, pf_resident_names &N, const char **err)
{
    PF_RES_ARG(m < (1u << 24) && nents < (1u << 24) && nseekers < (1u << 24), "m / nents / nseekers");
    PF_RES_ARG(m == 0 || reqs, "reqs");
    PF_RES_ARG(nents == 0 || ents || ent_uids, "ents and ent_uids are both NULL");
    PF_RES_ARG(nseekers == 0 || seeker_uids, "seeker_uids");
    N.fp_index.clear();
    N.uids.clear();
    if (int rc = pf_resident_named(ent_uids, nents, ents != nullptr, population, N.fp_index, N.uids,
                                   "ents == NULL, but an entry of ent_uids names no uid", "footprint uid outside the population", err))
        return rc;
    for (size_t k = 0; k < nseekers; k++) {
        PF_RES_ARG(seeker_uids[k] < population, "seeker uid outside the population");
        N.uids.push_back(seeker_uids[k]);
    }
    for (size_t i = 0; i < m; i++) {
        PF_RES_ARG((uint64_t)reqs[i].ent_off + reqs[i].ent_n <= nents, "footprint range");
        PF_RES_ARG((uint64_t)reqs[i].chunk_off + reqs[i].chunk_n <= nseekers, "seeker range");
    }
    return PFNAV_OK;
}

// The batch's inputs from the resolved values: fp_xzr[3k ..] = {x, z, radius} of the record of N.uids[k] (footprint
// N.fp_index[k]), seek_chunk[s] = the chunk index (r * chunk_w + c) under seeker s, or -1 when no tile lies under it.
// Footprint k is ents[k] unless it names a uid; then it is that record's circle (is_building 0, corners 0). Request i
// keeps everything but its chunk range, which now lists the chunks of its seekers in the order of their first seeker,
// each once. A seeker off the map: PFNAV_ERR_ARG, and B is untouched.
static inline int pf_resident_merge(const pfnav_entity_field_req *reqs, size_t m, const pfnav_footprint *ents, size_t nents,
                                    const pf_resident_names &N, const float *fp_xzr, const int32_t *seek_chunk,
                                    size_t nseekers, int chunk_w, int chunk_h, pf_resident_batch &B, const char **err)
{
    for (size_t s = 0; s < nseekers; s++)
        if (seek_chunk[s] < 0 || seek_chunk[s] >= chunk_w * chunk_h) {
            *err = "a seeker stands where no tile lies under it";
            return PFNAV_ERR_ARG;
        }
    B.ents.assign(nents, pfnav_footprint());
    if (ents) memcpy(B.ents.data(), ents, nents * sizeof(pfnav_footprint));
    for (size_t k = 0; k < N.fp_index.size(); k++) {
        pfnav_footprint &f = B.ents[N.fp_index[k]];
        memset(&f, 0, sizeof(f));
        f.x = fp_xzr[3 * k]; f.z = fp_xzr[3 * k + 1]; f.sel_radius = fp_xzr[3 * k + 2];
    }
    B.reqs.assign(reqs, reqs + m);
    B.chunks_rc.clear();
    std::vector<uint32_t> seen((size_t)chunk_w * chunk_h, 0);       // request i + 1 once request i has listed the chunk
    for (size_t i = 0; i < m; i++) {
        pfnav_entity_field_req &q = B.reqs[i];
        const uint32_t off = (uint32_t)(B.chunks_rc.size() / 2);
        for (uint32_t k = 0; k < reqs[i].chunk_n; k++) {
            const int32_t c = seek_chunk[reqs[i].chunk_off + k];
            if (seen[c] == i + 1) continue;
            seen[c] = (uint32_t)(i + 1);
            B.chunks_rc.push_back(c / chunk_w);
            B.chunks_rc.push_back(c % chunk_w);
        }
        q.chunk_off = off;
        q.chunk_n = (uint32_t)(B.chunks_rc.size() / 2) - off;
    }
    return PFNAV_OK;
}

// The positions a call names by uid (pfnav_pool_request_paths_resident: sources, destinations; pfnav_map_query_resident:
// (x, z), (dst_x, dst_z); pfnav_group_arrival_velocity_resident: the positions): the (entry, uid) pairs of the first
// array, then those of the second. The device reads them as entry[np] then uid[np] (np = entry.size()).
struct pf_resident_points {
    std::vector<uint32_t> entry, uid;
    size_t n0 = 0;                       // how many pairs the first array names
    size_t bytes() const { return entry.size() * 8; }
    void pack(uint8_t *dst) const
    {
        if (entry.empty()) return;
        memcpy(dst, entry.data(), entry.size() * 4);
        memcpy(dst + entry.size() * 4, uid.data(), uid.size() * 4);
    }
};

// Checks the uid arrays of n entries with up to two named positions each: n below 2^24; array a's entry k names uids_a[k]
// unless uids_a is NULL or the entry is PFNAV_NULL_UID, and then it needs the given positions (given_a); every named uid
// below `population`. uids_b / given_b the same for the second position (NULL and true when there is none). Fills P.
// PFNAV_ERR_ARG with *err naming the check; P is then unspecified.
static inline int pf_resident_points_check(size_t n, const uint32_t *uids_a, bool given_a, const uint32_t *uids_b, bool given_b,
                                           size_t population, pf_resident_points &P, const char **err)
{
    PF_RES_ARG(n < (1u << 24), "n");
    P.entry.clear();
    P.uid.clear();
    const char *no_given = "an entry names no uid, and its positions are NULL", *outside = "uid outside the population";
    if (int rc = pf_resident_named(uids_a, n, given_a, population, P.entry, P.uid, no_given, outside, err)) return rc;
    P.n0 = P.entry.size();
    return pf_resident_named(uids_b, n, given_b, population, P.entry, P.uid, no_given, outside, err);
}

#undef PF_RES_ARG
