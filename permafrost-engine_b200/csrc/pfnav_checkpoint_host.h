// pfnav_checkpoint_host.h -- the checkpoint segment of pfnav_agents_save / pfnav_agents_restore, CUDA-free: its layout,
// the validation of segments that arrive from outside the program, the choice of the records a restore takes for an
// entity range, and the two per-item rules the device runs (the pack of a record row, the incref a restored blocking row
// queues). tests/emu/checkpoint_emu.cpp builds this header with g++.
//
// A segment is
//   pf_ckpt_header (64 bytes)
//   the whole flock table: nflocks pfnav_flock records
//   for each uid in [lo, hi), in uid order, one row: pfnav_agent, then pfnav_movestate, pfnav_movestate_ext,
//   pfnav_formation_in and pfnav_blocking, each only when its bit is in `tables`.
// Every record size is a multiple of 16 bytes, so every row and record starts 16-byte aligned relative to the segment.
#pragma once
#include <stddef.h>
#include <string.h>
#include "pfnav_commands_host.h"

#define PF_CKPT_MAGIC   0x4B434650u           // "PFCK" little-endian
#define PF_CKPT_VERSION 1u
#define PF_CKPT_MS      (1u << 0)             // pfnav_movestate per entity
#define PF_CKPT_EXT     (1u << 1)             // pfnav_movestate_ext
#define PF_CKPT_FORM    (1u << 2)             // pfnav_formation_in
#define PF_CKPT_BLK     (1u << 3)             // pfnav_blocking
#define PF_CKPT_TABLES  0xFu

struct pf_ckpt_header {
    uint32_t magic, version;
    uint32_t rec_size[5];                     // pfnav_agent, _movestate, _movestate_ext, _formation_in, _blocking
    uint32_t tables;                          // PF_CKPT_* bits
    uint64_t n_total, lo, hi;                 // the population and the uid range of this segment's rows
    int32_t  hz;
    uint32_t nflocks;
};
static_assert(sizeof(pf_ckpt_header) == 64, "pf_ckpt_header is 64 bytes");

static const uint32_t pf_ckpt_sizes[5] = {sizeof(pfnav_agent), sizeof(pfnav_movestate), sizeof(pfnav_movestate_ext),
                                          sizeof(pfnav_formation_in), sizeof(pfnav_blocking)};

// 16-byte words of one row; w_ms / w_ext / w_form / w_blk: where each record starts in it (valid when present)
struct pf_ckpt_row {
    uint32_t words, w_ms, w_ext, w_form, w_blk;
};
PF_HD pf_ckpt_row pf_ckpt_row_of(uint32_t tables)
{
    pf_ckpt_row r;
    uint32_t w = sizeof(pfnav_agent) / 16;
    r.w_ms = w;   if (tables & PF_CKPT_MS) w += sizeof(pfnav_movestate) / 16;
    r.w_ext = w;  if (tables & PF_CKPT_EXT) w += sizeof(pfnav_movestate_ext) / 16;
    r.w_form = w; if (tables & PF_CKPT_FORM) w += sizeof(pfnav_formation_in) / 16;
    r.w_blk = w;  if (tables & PF_CKPT_BLK) w += sizeof(pfnav_blocking) / 16;
    r.words = w;
    return r;
}

// The device pack of a segment's rows: word q of the row of uid (0 <= q < row.words) comes from word *k of table *t
// (0 agent, 1 movestate, 2 movestate_ext, 3 formation, 4 blocking) of that uid.
PF_HD void pf_ckpt_word_source(const pf_ckpt_row &row, uint32_t tables, uint32_t q, int *t, uint32_t *k)
{
    if (q < row.w_ms) { *t = 0; *k = q; }
    else if ((tables & PF_CKPT_MS) && q < row.w_ext) { *t = 1; *k = q - row.w_ms; }
    else if ((tables & PF_CKPT_EXT) && q < row.w_form) { *t = 2; *k = q - row.w_ext; }
    else if ((tables & PF_CKPT_FORM) && q < row.w_blk) { *t = 3; *k = q - row.w_form; }
    else { *t = 4; *k = q - row.w_blk; }
}

// The one op a restore queues for a restored row: the incref of the circle its blocking record describes, on the entity's
// layers (its flags), when it holds a block. Returns whether there is one.
PF_HD bool pf_ckpt_restore_op(const pfnav_agent &a, const pfnav_blocking &b, pfnav_blocker_op *op)
{
    if (!b.blocking) return false;
    *op = {b.stop_x, b.stop_z, b.stop_radius, b.faction_id, a.flags, +1};
    return true;
}

static inline size_t pf_ckpt_bytes(uint32_t tables, size_t nflocks, size_t nrows)
{
    return sizeof(pf_ckpt_header) + nflocks * sizeof(pfnav_flock) + nrows * (size_t)pf_ckpt_row_of(tables).words * 16;
}

static inline pf_ckpt_header pf_ckpt_header_make(uint32_t tables, size_t n_total, size_t lo, size_t hi, int hz, size_t nflocks)
{
    pf_ckpt_header h;
    memset(&h, 0, sizeof(h));
    h.magic = PF_CKPT_MAGIC; h.version = PF_CKPT_VERSION;
    memcpy(h.rec_size, pf_ckpt_sizes, sizeof(h.rec_size));
    h.tables = tables; h.n_total = n_total; h.lo = lo; h.hi = hi; h.hz = hz; h.nflocks = (uint32_t)nflocks;
    return h;
}

// A validated set of segments. segs: the non-empty segments in uid order, each with its header.
struct pf_ckpt_seg { const uint8_t *base; pf_ckpt_header h; };
struct pf_ckpt_set {
    pf_ckpt_header h;                         // what every segment agrees on (n_total, hz, nflocks, tables); lo = 0, hi = n_total
    std::vector<pf_ckpt_seg> segs;
    const pfnav_flock *flocks = nullptr;      // the flock table of the first segment (every segment holds the same bytes)
    std::vector<uint8_t> layers_used;         // [layer]: some entity of some flock stands on it (pfnav_route_build needed)
};

// The checks of one row: those of pfnav_agents_upload (flock index, layer created), pfnav_agents_change_population
// (finite floats, ext targets inside the population) and pfnav_agents_upload_blocking (blocking 0 / 1, faction 0..15),
// and no other: whatever those calls accept, and so whatever pfnav_agents_save writes, restores. *layer: the entity's
// navigation layer.
static inline const char *pf_ckpt_row_check(const uint8_t *row, const pf_ckpt_row &R, uint32_t tables, size_t n_total,
                                            size_t nflocks, int nlayers, int *layer)
{
    pfnav_agent a;
    memcpy(&a, row, sizeof(a));
    if (const char *e = pf_agent_check(a, nflocks, nlayers, layer)) return e;
    if (!pf_finite(a.pos, 11)) return "agent with a float that is not finite";
    if (tables & PF_CKPT_MS) {
        pfnav_movestate m;
        memcpy(&m, row + R.w_ms * 16, sizeof(m));
        if (!pf_finite(m.next_pos, 40)) return "movestate with a float that is not finite";
    }
    if (tables & PF_CKPT_EXT) {
        pfnav_movestate_ext x;
        memcpy(&x, row + R.w_ext * 16, sizeof(x));
        if (x.surround_target_uid != PFNAV_NULL_UID && x.surround_target_uid >= n_total) return "movestate_ext target outside the population";
        if (!pf_finite(&x.target_range, 3) || !pf_finite(x.target_dir, 8)) return "movestate_ext with a float that is not finite";
    }
    if (tables & PF_CKPT_FORM) {
        pfnav_formation_in f;
        memcpy(&f, row + R.w_form * 16, sizeof(f));
        if (!pf_finite(f.cell_pos, 14)) return "formation record with a float that is not finite";
    }
    if (tables & PF_CKPT_BLK) {
        pfnav_blocking b;
        memcpy(&b, row + R.w_blk * 16, sizeof(b));
        if (const char *e = pf_blocking_check(b)) return e;
        if (!pf_finite(&b.stop_x, 3)) return "blocking record with a float that is not finite";
    }
    return nullptr;
}

// Validate nseg segments completely, changing nothing: each segment's header (magic, version, record sizes, table bits, hz,
// lo <= hi <= n_total) and its exact size; the segments agree on n_total, hz, nflocks, tables and the flock table bytes;
// their ranges tile [0, n_total) without overlap or gap (empty segments are allowed anywhere); every flock target is
// finite; every row passes pf_ckpt_row_check against nlayers created layers. Fills S. Returns NULL or what was wrong.
// The verdict depends on the segments and nlayers only, so every member of a job reaches the same one.
static inline const char *pf_ckpt_check(const void *const *segs, const size_t *sizes, size_t nseg, int nlayers, pf_ckpt_set &S)
{
    if (nseg == 0) return "no segment";
    if (!segs || !sizes) return "segs / sizes == NULL";
    S.segs.clear();
    for (size_t i = 0; i < nseg; i++) {
        if (!segs[i]) return "a segment pointer is NULL";
        if (sizes[i] < sizeof(pf_ckpt_header)) return "a segment is shorter than its header";
        pf_ckpt_seg s;
        s.base = (const uint8_t *)segs[i];
        memcpy(&s.h, s.base, sizeof(s.h));
        const pf_ckpt_header &h = s.h;
        if (h.magic != PF_CKPT_MAGIC) return "not a checkpoint segment (magic)";
        if (h.version != PF_CKPT_VERSION) return "checkpoint format version not supported";
        if (memcmp(h.rec_size, pf_ckpt_sizes, sizeof(h.rec_size))) return "checkpoint record sizes differ from this library's";
        if (h.tables & ~PF_CKPT_TABLES) return "unknown table bit";
        if (!(h.hz == 20 || h.hz == 10 || h.hz == 5 || h.hz == 1)) return "hz must be 20, 10, 5 or 1";
        if (h.n_total >= (1u << 31) || h.nflocks >= (1u << 24)) return "population or flock table too large";
        if (h.lo > h.hi || h.hi > h.n_total) return "segment range outside the population";
        if (sizes[i] != pf_ckpt_bytes(h.tables, h.nflocks, h.hi - h.lo)) return "segment size does not match its header (truncated or padded)";
        if (i == 0) S.h = h;
        const pf_ckpt_header &h0 = S.h;
        if (h.n_total != h0.n_total) return "segments disagree on the population size";
        if (h.hz != h0.hz) return "segments disagree on hz";
        if (h.nflocks != h0.nflocks) return "segments disagree on the flock table";
        if (h.tables != h0.tables) return "segments disagree on the tables they hold";
        if (i == 0) S.flocks = (const pfnav_flock *)(s.base + sizeof(pf_ckpt_header));
        else if (memcmp(s.base + sizeof(pf_ckpt_header), S.flocks, h.nflocks * sizeof(pfnav_flock)))
            return "segments disagree on the flock table";
        if (h.hi > h.lo) S.segs.push_back(s);
    }
    S.h.lo = 0; S.h.hi = S.h.n_total;
    std::sort(S.segs.begin(), S.segs.end(), [](const pf_ckpt_seg &a, const pf_ckpt_seg &b) { return a.h.lo < b.h.lo; });
    uint64_t at = 0;
    for (const pf_ckpt_seg &s : S.segs) {
        if (s.h.lo < at) return "segments overlap";
        if (s.h.lo > at) return "segments leave a gap in the population";
        at = s.h.hi;
    }
    if (at != S.h.n_total) return "segments leave a gap in the population";
    for (uint32_t f = 0; f < S.h.nflocks; f++) {
        pfnav_flock fl;
        memcpy(&fl, (const uint8_t *)S.flocks + (size_t)f * sizeof(pfnav_flock), sizeof(fl));
        if (!pf_finite(fl.target, 2)) return "flock target not finite";
    }
    const pf_ckpt_row R = pf_ckpt_row_of(S.h.tables);
    S.layers_used.assign(PFNAV_NAV_LAYER_MAX, 0);
    for (const pf_ckpt_seg &s : S.segs) {
        const uint8_t *rows = s.base + sizeof(pf_ckpt_header) + (size_t)S.h.nflocks * sizeof(pfnav_flock);
        for (uint64_t u = 0; u < s.h.hi - s.h.lo; u++) {
            int layer;
            const uint8_t *row = rows + u * R.words * 16;
            if (const char *e = pf_ckpt_row_check(row, R, S.h.tables, S.h.n_total, S.h.nflocks, nlayers, &layer)) return e;
            int32_t flock;
            memcpy(&flock, row + offsetof(pfnav_agent, flock), 4);
            if (flock >= 0) S.layers_used[layer] = 1;
        }
    }
    return nullptr;
}

// The runs of rows that make up [lo, hi): (segment index into S.segs, first row in it, count), in uid order
struct pf_ckpt_run { uint32_t seg; uint64_t first, n; };
static inline void pf_ckpt_runs(const pf_ckpt_set &S, size_t lo, size_t hi, std::vector<pf_ckpt_run> &out)
{
    out.clear();
    for (uint32_t i = 0; i < S.segs.size(); i++) {
        const uint64_t a = std::max<uint64_t>(lo, S.segs[i].h.lo), b = std::min<uint64_t>(hi, S.segs[i].h.hi);
        if (a < b) out.push_back({i, a - S.segs[i].h.lo, b - a});
    }
}

// The records of [lo, hi) of a validated set, one array per table (an array may be NULL to skip its table; a table the
// set does not hold is not written)
static inline void pf_ckpt_gather(const pf_ckpt_set &S, size_t lo, size_t hi, pfnav_agent *agents, pfnav_movestate *ms,
                                  pfnav_movestate_ext *ext, pfnav_formation_in *form, pfnav_blocking *blk)
{
    const pf_ckpt_row R = pf_ckpt_row_of(S.h.tables);
    std::vector<pf_ckpt_run> runs;
    pf_ckpt_runs(S, lo, hi, runs);
    size_t j = 0;
    for (const pf_ckpt_run &r : runs) {
        const uint8_t *rows = S.segs[r.seg].base + sizeof(pf_ckpt_header) + (size_t)S.h.nflocks * sizeof(pfnav_flock);
        for (uint64_t k = 0; k < r.n; k++, j++) {
            const uint8_t *row = rows + (r.first + k) * R.words * 16;
            if (agents) memcpy(agents + j, row, sizeof(pfnav_agent));
            if (ms && (S.h.tables & PF_CKPT_MS)) memcpy(ms + j, row + R.w_ms * 16, sizeof(pfnav_movestate));
            if (ext && (S.h.tables & PF_CKPT_EXT)) memcpy(ext + j, row + R.w_ext * 16, sizeof(pfnav_movestate_ext));
            if (form && (S.h.tables & PF_CKPT_FORM)) memcpy(form + j, row + R.w_form * 16, sizeof(pfnav_formation_in));
            if (blk && (S.h.tables & PF_CKPT_BLK)) memcpy(blk + j, row + R.w_blk * 16, sizeof(pfnav_blocking));
        }
    }
}
