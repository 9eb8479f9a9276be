// pfnav_inputs_host.h -- the host side of pfnav_agents_input_deltas and the write rule its kernel applies, CUDA-free:
// record validation, per-uid folding in array order, the field write of one record, and the split of a multi-GPU job's
// batch into the records a member owns. tests/emu/input_deltas_emu.cpp builds this header with g++.
#pragma once
#include <math.h>
#include <stdint.h>
#include <unordered_map>
#include <vector>
#include "../../include/pfnav.h"

#ifndef PF_HD
#ifdef __CUDACC__
#define PF_HD __host__ __device__ __forceinline__
#else
#define PF_HD inline
#endif
#endif

#define PF_INPUT_EXT (PFNAV_INPUT_TARGET_PREV | PFNAV_INPUT_TARGET_DIR | PFNAV_INPUT_ROT | PFNAV_INPUT_SURROUND_FIELD)
#define PF_INPUT_PUBLIC (PF_INPUT_EXT | PFNAV_INPUT_FORMATION)
#define PF_FORM_FLAGS 0x1Fu          // the five PFNAV_FORM_* bits

// One record on one entity. ex / f may be NULL when the record carries no bit that writes them.
PF_HD void pf_input_apply(pfnav_movestate_ext *ex, pfnav_formation_in *f, const pfnav_input_delta &d)
{
    if (d.mask & PFNAV_INPUT_TARGET_PREV) { ex->target_prev_pos[0] = d.target_prev_pos[0]; ex->target_prev_pos[1] = d.target_prev_pos[1]; }
    if (d.mask & PFNAV_INPUT_TARGET_DIR)
        for (int k = 0; k < 4; k++) ex->target_dir[k] = d.target_dir[k];
    if (d.mask & PFNAV_INPUT_ROT)
        for (int k = 0; k < 4; k++) ex->rot[k] = d.rot[k];
    if (d.mask & PFNAV_INPUT_SURROUND_FIELD) ex->using_surround_field = d.using_surround_field;
    if (d.mask & PFNAV_INPUT_FORMATION) *f = d.formation;
}

struct pf_input_limits {
    size_t lo, hi;                // uids accepted: the own range (solo), the population (job)
    bool have_ext;                // movestate_ext table uploaded
};

static inline bool pf_input_finite(const float *p, int n)
{
    for (int i = 0; i < n; i++)
        if (!isfinite(p[i])) return false;
    return true;
}

// the checks of one record; NULL when it passes
static inline const char *pf_input_check(const pfnav_input_delta &d, const pf_input_limits &L)
{
    if (d.uid < L.lo || d.uid >= L.hi) return "input delta uid outside this context's own entity range";
    if (d.mask & ~PF_INPUT_PUBLIC) return "unknown input delta mask bit";
    if ((d.mask & PF_INPUT_EXT) && !L.have_ext)
        return "PFNAV_INPUT_TARGET_PREV / _TARGET_DIR / _ROT / _SURROUND_FIELD need pfnav_agents_upload_movestate_ext";
    if ((d.mask & PFNAV_INPUT_TARGET_PREV) && !pf_input_finite(d.target_prev_pos, 2)) return "input delta target_prev_pos not finite";
    if ((d.mask & PFNAV_INPUT_TARGET_DIR) && !pf_input_finite(d.target_dir, 4)) return "input delta target_dir not finite";
    if ((d.mask & PFNAV_INPUT_ROT) && !pf_input_finite(d.rot, 4)) return "input delta rot not finite";
    if ((d.mask & PFNAV_INPUT_SURROUND_FIELD) && d.using_surround_field > 1) return "input delta using_surround_field must be 0 or 1";
    if (d.mask & PFNAV_INPUT_FORMATION) {
        if (!pf_input_finite(d.formation.cell_pos, 14)) return "input delta formation record with a float that is not finite";
        if (d.formation.flags & ~PF_FORM_FLAGS) return "input delta formation flags outside the PFNAV_FORM_* bits";
    }
    return nullptr;
}

// Validate every record and fold the records of one uid, in array order, into one record (first-occurrence order), so
// that one thread owns each entity: per field the last writer wins, and the folded mask is the union of the masks.
// Applying `out` equals applying `d` one by one. Returns NULL, or what was wrong (out is then meaningless).
static inline const char *pf_input_merge(const pfnav_input_delta *d, size_t n, const pf_input_limits &L,
                                         std::vector<pfnav_input_delta> &out)
{
    out.clear();
    std::unordered_map<uint32_t, uint32_t> at;
    at.reserve(n * 2);
    for (size_t i = 0; i < n; i++) {
        const pfnav_input_delta &s = d[i];
        if (const char *e = pf_input_check(s, L)) return e;
        auto it = at.find(s.uid);
        if (it == at.end()) {
            it = at.emplace(s.uid, (uint32_t)out.size()).first;
            pfnav_input_delta z = {};
            z.uid = s.uid;
            out.push_back(z);
        }
        pfnav_input_delta &m = out[it->second];
        if (s.mask & PFNAV_INPUT_TARGET_PREV) { m.target_prev_pos[0] = s.target_prev_pos[0]; m.target_prev_pos[1] = s.target_prev_pos[1]; }
        if (s.mask & PFNAV_INPUT_TARGET_DIR)
            for (int k = 0; k < 4; k++) m.target_dir[k] = s.target_dir[k];
        if (s.mask & PFNAV_INPUT_ROT)
            for (int k = 0; k < 4; k++) m.rot[k] = s.rot[k];
        if (s.mask & PFNAV_INPUT_SURROUND_FIELD) m.using_surround_field = s.using_surround_field;
        if (s.mask & PFNAV_INPUT_FORMATION) m.formation = s.formation;
        m.mask |= s.mask;
    }
    return nullptr;
}

// A member's part of a job batch, changing nothing: validation of every record against the population (L.lo = 0,
// L.hi = n_total), folding, and the folded records of the own range [lo, hi). any_form: some record of the batch carries
// PFNAV_INPUT_FORMATION (every member then holds a formation table afterwards). Returns NULL or what was wrong.
static inline const char *pf_input_job_plan(const pfnav_input_delta *d, size_t n, const pf_input_limits &L, size_t lo, size_t hi,
                                            std::vector<pfnav_input_delta> &own, bool &any_form)
{
    std::vector<pfnav_input_delta> merged;
    own.clear();
    any_form = false;
    if (const char *e = pf_input_merge(d, n, L, merged)) return e;
    for (const pfnav_input_delta &m : merged) {
        any_form |= (m.mask & PFNAV_INPUT_FORMATION) != 0;
        if (m.uid >= lo && m.uid < hi) own.push_back(m);
    }
    return nullptr;
}
