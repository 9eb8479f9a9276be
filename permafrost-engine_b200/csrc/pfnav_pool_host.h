// pfnav_pool_host.h -- the field pool's host bookkeeping and its two slot policies. No CUDA: the device side is
// pfnav_pool.cu, and tests/test_pool_emu.py compiles this header with g++ to run the real policies.
//
// One slot holds the flow AND the LOS field of a (dest, chunk) key, key = dest * chunks + chunk. Every slot below `used`
// is in exactly one of three states: on the free list, owned by the key pf_pool_reserve gave it to (evictable), or taken
// by the zone rule (pf_pool_zone_take: no owner, never evicted, held until the pool is cleared). Only the functions here
// and in pfnav_pool.cu write the slot table, the owners, the free list and `used`.
//
// The pool segment of pfnav_pool_save / pfnav_pool_restore (its layout, validation and load) is at the end of this file;
// tests/emu/pool_checkpoint_emu.cpp builds it with g++. The map digest that ties a segment to the map its fields were
// built on is defined with the other state digests in pfnav_digest_host.h, which this header includes at its end.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include "../../include/pfnav.h"
#include "pfnav_commands_host.h"

void pfnav_set_error(const char *fmt, ...);

// a TARGET_ENEMIES / TARGET_ENTITY destination (pfnav_pool_request_entity_fields): the footprints its in-place repairs
// start from (kind -1: no entity field was requested for the destination)
struct pf_aux_target { int kind = -1, layer = 0, ref_layer = 0; std::vector<pfnav_footprint> ents; };

struct pf_pool {
    int ndests = 0, max = 0, used = 0;
    int nzone = 0;                           // slots taken by the zone rule
    std::vector<int32_t> slot;               // [ndests][chunks] -> slot or -1
    std::vector<uint64_t> ffid;              // [ndests][chunks]: ff_id currently mapped (dest, chunk) -> field, 0 = none
    std::vector<uint8_t> has;                // [max]: bit 0 flow field built, bit 1 LOS field built
    std::vector<pfnav_field_req> req;        // [max]: the last request applied to the slot (== flow_field::target, field.c:2076)
    std::vector<uint32_t> touch;             // [max]: last tick number a request named the slot
    std::vector<int64_t> owner;              // [max]: the owning key, or -1 (free or zone-held)
    std::vector<int32_t> free_list;          // evicted slots, reused last in first out before `used` grows
    // device copies (pfnav_pool.cu). The `has` bytes sit behind the LOS fields in one allocation: d_has = d_los + max * 4096
    int32_t *d_slot = nullptr;
    uint8_t *d_flow = nullptr, *d_los = nullptr, *d_has = nullptr;
    uint32_t *d_touch = nullptr;             // [max]: last tick number a work item read the slot (desired-velocity kernels)
    bool dev_stale = false;                  // cleared on the host only: the device copies wait for pf_pool_refresh

    int32_t slot_of(size_t key) const { return slot[key]; }
    uint8_t has_of(size_t key) const { const int32_t s = slot[key]; return s < 0 ? 0 : has[s]; }
    size_t avail() const { return free_list.size() + (size_t)(max - used); }       // slots a reservation takes without evicting
    size_t table_bytes() const { return slot.size() * 4 + (size_t)max; }          // the slot table, then the `has` bytes
    void built(int32_t s, uint8_t bits) { has[s] |= bits; }
    void built_flow(int32_t s, const pfnav_field_req &q) { has[s] |= 1; req[s] = q; }
};

// host mirrors as pfnav_pool_clear leaves them (the last requests stay: a slot is read only while its `has` bit is set)
inline void pf_pool_reset(pf_pool &P)
{
    std::fill(P.slot.begin(), P.slot.end(), -1);
    std::fill(P.has.begin(), P.has.end(), 0);
    std::fill(P.ffid.begin(), P.ffid.end(), 0);
    std::fill(P.touch.begin(), P.touch.end(), 0);
    std::fill(P.owner.begin(), P.owner.end(), -1);
    P.free_list.clear();
    P.used = 0; P.nzone = 0;
}

// the distinct keys of keys[0, n) without a slot, ascending (a key is marked -2 while it is collected, so repeats are skipped)
inline void pf_pool_fresh(pf_pool &P, const size_t *keys, size_t n, std::vector<size_t> &fresh)
{
    fresh.clear();
    for (size_t i = 0; i < n; i++)
        if (P.slot[keys[i]] == -1) { P.slot[keys[i]] = -2; fresh.push_back(keys[i]); }
    for (size_t key : fresh) P.slot[key] = -1;
    std::sort(fresh.begin(), fresh.end());
}

// ------------------------------------------------------------------------------------------
// Pool slots with LRU eviction. The reference keeps its fields in LRU caches of fixed capacity
// (fieldcache.c:59-71; CONFIG_FLOW_CACHE_SZ / CONFIG_LOS_CACHE_SZ, config.h:64-65): a request that finds the
// cache full evicts the least recently used entry, and an agent that later misses it re-requests its path
// (nav.c:3484-3506 == pfnav_pool_repair). "Recently used" = the last tick whose desired-velocity pass read the slot
// (device side) or whose request named it (host side); ties go to the lower slot index.
// pf_pool_reserve: slots for the keys a request batch is about to write -- all or nothing: on PFNAV_ERR_NOMEM nothing
// was changed. keys may repeat; `tick` stamps every slot named. *out_evicted: slot-table entries of OTHER keys changed
// (the caller re-uploads the whole table and the `has` bytes). device_stamps(std::vector<uint32_t> &stamp) raises
// stamp[s] to the device's stamp of slot s and returns a pfnav status; it is called only when a slot must be evicted.
// ------------------------------------------------------------------------------------------
template <class DeviceStamps>
int pf_pool_reserve(pf_pool &P, const size_t *keys, size_t n, uint32_t tick, int32_t *slots_out, bool *out_evicted,
                    DeviceStamps &&device_stamps)
{
    if (out_evicted) *out_evicted = false;
    std::vector<size_t> fresh;
    pf_pool_fresh(P, keys, n, fresh);
    const size_t avail = P.avail();
    if (fresh.size() > avail) {
        const size_t k = fresh.size() - avail;
        std::vector<uint32_t> stamp(P.touch);
        if (int rc = device_stamps(stamp)) return rc;
        std::vector<uint8_t> pinned(P.max, 0);
        for (size_t i = 0; i < n; i++) { const int s = P.slot[keys[i]]; if (s >= 0) pinned[s] = 1; }
        std::vector<int32_t> cand;
        for (int s = 0; s < P.used; s++)
            if (P.owner[s] >= 0 && !pinned[s]) cand.push_back(s);
        if (cand.size() < k) {
            pfnav_set_error("field pool full: %zu new (dest, chunk) fields requested, %zu slots free, %zu evictable of %d",
                            fresh.size(), avail, cand.size(), P.max);
            return PFNAV_ERR_NOMEM;
        }
        std::sort(cand.begin(), cand.end(), [&](int32_t a, int32_t b) { return stamp[a] != stamp[b] ? stamp[a] < stamp[b] : a < b; });
        for (size_t i = 0; i < k; i++) {
            const int32_t s = cand[i];
            const size_t owner = (size_t)P.owner[s];
            P.slot[owner] = -1; P.ffid[owner] = 0;
            P.has[s] = 0; P.owner[s] = -1;
            P.free_list.push_back(s);
        }
        if (out_evicted) *out_evicted = true;
    }
    for (size_t key : fresh) {
        int32_t s;
        if (!P.free_list.empty()) { s = P.free_list.back(); P.free_list.pop_back(); }
        else s = P.used++;
        P.slot[key] = s; P.owner[s] = (int64_t)key; P.has[s] = 0;
    }
    for (size_t i = 0; i < n; i++) {
        const int32_t s = P.slot[keys[i]];
        P.touch[s] = tick;
        if (slots_out) slots_out[i] = s;
    }
    return PFNAV_OK;
}

// pf_pool_reserve's verdict on keys, without its changes and without the device stamps. Closed form: the slots a batch
// can hold are the max - nzone that are not zone-held, and the keys that need one are the distinct keys not held by a
// zone-held slot. pf_pool_reserve never changes the zone-held set, so the verdicts of several batches reserved in turn
// are each this one, taken on the pool as it is now.
inline bool pf_pool_fits(const pf_pool &P, const size_t *keys, size_t n)
{
    std::vector<size_t> need;
    for (size_t i = 0; i < n; i++) {
        const int32_t s = P.slot[keys[i]];
        if (s < 0 || P.owner[s] >= 0) need.push_back(keys[i]);        // a mapped slot without an owner is zone-held
    }
    std::sort(need.begin(), need.end());
    return (size_t)(std::unique(need.begin(), need.end()) - need.begin()) <= (size_t)(P.max - P.nzone);
}

// The zone rule (pfnav_pool_request_zones, the single call's rule): the key's slot if it has one, else a fresh slot from
// `used` -- never a free-listed one, and no owner, so it is never evicted. -1: every slot below max is used.
inline int32_t pf_pool_zone_take(pf_pool &P, size_t key)
{
    if (P.slot[key] >= 0) return P.slot[key];
    if (P.used >= P.max) return -1;
    P.nzone++;
    return P.slot[key] = P.used++;
}

// the zone rule's verdict on keys: the distinct keys without a slot fit in the slots above `used`
inline bool pf_pool_zone_fits(const pf_pool &P, const size_t *keys, size_t n)
{
    std::vector<size_t> fresh;
    for (size_t i = 0; i < n; i++) if (P.slot[keys[i]] < 0) fresh.push_back(keys[i]);
    std::sort(fresh.begin(), fresh.end());
    return (size_t)(std::unique(fresh.begin(), fresh.end()) - fresh.begin()) <= (size_t)(P.max - P.used);
}

// the map changed under a key's fields: its `has` bits and its ff_id go, its slot stays mapped
inline void pf_pool_drop(pf_pool &P, size_t key)
{
    const int32_t s = P.slot[key];
    if (s >= 0) P.has[s] = 0;
    P.ffid[key] = 0;
}

// ------------------------------------------------------------------------------------------
// The pool segment (pfnav_pool_save / pfnav_pool_restore). Every section starts 16-byte aligned:
//   pf_pool_header (64 bytes)
//   slot table int32 [ndests * chunks], ff_ids uint64 [ndests * chunks], `has` bytes [max], last requests
//   pfnav_field_req [max], host touch stamps uint32 [max], owners int64 [max], free list int32 [nfree] (in order)
//   aux targets pf_pool_aux_rec [naux] (destination d = record d), then their footprints pfnav_footprint [nfp] in order
//   device touch stamps uint32 [max]
//   for each slot with `has` != 0, ascending: its flow field (4096 bytes) and its LOS field (4096 bytes)
// The device touch column sits right before the fields, so that it and the packed fields travel in one copy.
// ------------------------------------------------------------------------------------------
#define PF_POOL_MAGIC   0x4C504650u           // "PFPL" little-endian
#define PF_POOL_VERSION 1u

struct pf_pool_header {
    uint32_t magic, version;
    uint16_t req_size, fp_size;               // sizeof(pfnav_field_req), sizeof(pfnav_footprint)
    uint8_t  chunk_w, chunk_h, nlayers, _pad0;
    int32_t  ndests, max, used, nzone;
    uint32_t tick_no;
    uint32_t nfree, naux, nfp, nstored;       // free-list entries, aux targets, their footprints, stored fields
    uint32_t _pad1;
    uint64_t digest;                          // pf_map_digest of the map the fields were built on
};
static_assert(sizeof(pf_pool_header) == 64, "pf_pool_header is 64 bytes");
struct pf_pool_aux_rec { int32_t kind, layer, ref_layer; uint32_t nents; };

struct pf_pool_layout { size_t slot, ffid, has, req, touch, owner, free, aux, fp, dtouch, fields, size; };
static inline pf_pool_layout pf_pool_layout_of(size_t nkeys, size_t max, size_t nfree, size_t naux, size_t nfp, size_t nstored)
{
    pf_pool_layout L;
    size_t o = sizeof(pf_pool_header);
    auto sec = [&](size_t bytes) { const size_t at = o; o = (o + bytes + 15) & ~(size_t)15; return at; };
    L.slot = sec(nkeys * 4); L.ffid = sec(nkeys * 8); L.has = sec(max); L.req = sec(max * sizeof(pfnav_field_req));
    L.touch = sec(max * 4); L.owner = sec(max * 8); L.free = sec(nfree * 4); L.aux = sec(naux * sizeof(pf_pool_aux_rec));
    L.fp = sec(nfp * sizeof(pfnav_footprint)); L.dtouch = sec(max * 4); L.fields = sec(nstored * 8192);
    L.size = o;
    return L;
}

// what a segment must match on the restoring context: map and pool geometry, and the digest of its committed map
struct pf_pool_target { int chunk_w, chunk_h, nlayers, ndests, max; uint64_t digest; };

// The slots whose fields a save stores (`has` != 0, ascending) and the segment's layout
static inline pf_pool_layout pf_pool_seg_plan(const pf_pool &P, const std::vector<pf_aux_target> &aux, std::vector<int32_t> &stored)
{
    stored.clear();
    for (int s = 0; s < P.max; s++) if (P.has[s]) stored.push_back(s);
    size_t nfp = 0;
    for (const pf_aux_target &A : aux) nfp += A.ents.size();
    return pf_pool_layout_of(P.slot.size(), P.max, P.free_list.size(), aux.size(), nfp, stored.size());
}

// The host part of a segment into out (L.size bytes, planned by pf_pool_seg_plan): the header and every section but the
// device touch stamps and the fields, which the caller writes at L.dtouch and L.fields. Padding is zero.
static inline void pf_pool_seg_write(const pf_pool &P, const std::vector<pf_aux_target> &aux, const pf_pool_target &G,
                                     uint32_t tick_no, const std::vector<int32_t> &stored, const pf_pool_layout &L, uint8_t *out)
{
    memset(out, 0, L.dtouch);
    pf_pool_header h;
    memset(&h, 0, sizeof(h));
    h.magic = PF_POOL_MAGIC; h.version = PF_POOL_VERSION;
    h.req_size = sizeof(pfnav_field_req); h.fp_size = sizeof(pfnav_footprint);
    h.chunk_w = (uint8_t)G.chunk_w; h.chunk_h = (uint8_t)G.chunk_h; h.nlayers = (uint8_t)G.nlayers;
    h.ndests = P.ndests; h.max = P.max; h.used = P.used; h.nzone = P.nzone; h.tick_no = tick_no;
    h.nfree = (uint32_t)P.free_list.size(); h.naux = (uint32_t)aux.size(); h.nstored = (uint32_t)stored.size();
    h.digest = G.digest;
    uint32_t nfp = 0;
    for (const pf_aux_target &A : aux) nfp += (uint32_t)A.ents.size();
    h.nfp = nfp;
    memcpy(out, &h, sizeof(h));
    memcpy(out + L.slot, P.slot.data(), P.slot.size() * 4);
    memcpy(out + L.ffid, P.ffid.data(), P.ffid.size() * 8);
    memcpy(out + L.has, P.has.data(), P.max);
    memcpy(out + L.req, P.req.data(), (size_t)P.max * sizeof(pfnav_field_req));
    memcpy(out + L.touch, P.touch.data(), (size_t)P.max * 4);
    memcpy(out + L.owner, P.owner.data(), (size_t)P.max * 8);
    if (!P.free_list.empty()) memcpy(out + L.free, P.free_list.data(), P.free_list.size() * 4);
    size_t f = 0;
    for (size_t d = 0; d < aux.size(); d++) {
        const pf_aux_target &A = aux[d];
        const pf_pool_aux_rec r = {A.kind, A.layer, A.ref_layer, (uint32_t)A.ents.size()};
        memcpy(out + L.aux + d * sizeof(r), &r, sizeof(r));
        if (!A.ents.empty()) memcpy(out + L.fp + f * sizeof(pfnav_footprint), A.ents.data(), A.ents.size() * sizeof(pfnav_footprint));
        f += A.ents.size();
    }
}

// A validated segment, read out of its bytes: the pool bookkeeping pf_pool_load installs, and where the device part is
// (base + L.dtouch: the device touch stamps, then the stored fields of the slots in `stored`, in that order).
struct pf_pool_image {
    pf_pool_header h;
    pf_pool_layout L;
    const uint8_t *base = nullptr;
    std::vector<int32_t> slot, free_list, stored;
    std::vector<uint64_t> ffid;
    std::vector<uint8_t> has;
    std::vector<pfnav_field_req> req;
    std::vector<uint32_t> touch, dtouch;
    std::vector<int64_t> owner;
    std::vector<pf_aux_target> aux;
};

template <typename T>
static inline void pf_pool_read(std::vector<T> &v, const uint8_t *p, size_t n)
{
    v.resize(n);
    if (n) memcpy(v.data(), p, n * sizeof(T));
}

// Validate a segment completely against the restoring context T, changing nothing: header (magic, version, record sizes,
// padding), map and pool geometry, counts, exact size, map digest, then the bookkeeping invariants written at the top of
// this file, the stamps, the requests of built flow fields and the aux targets. Fills I. Returns NULL or what was wrong.
static inline const char *pf_pool_check(const void *seg, size_t size, const pf_pool_target &T, pf_pool_image &I)
{
    if (!seg) return "segment == NULL";
    if (size < sizeof(pf_pool_header)) return "segment shorter than its header";
    const uint8_t *b = (const uint8_t *)seg;
    pf_pool_header &h = I.h;
    memcpy(&h, b, sizeof(h));
    if (h.magic != PF_POOL_MAGIC) return "not a pool segment (magic)";
    if (h.version != PF_POOL_VERSION) return "pool segment format version not supported";
    if (h.req_size != sizeof(pfnav_field_req) || h.fp_size != sizeof(pfnav_footprint)) return "pool segment record sizes differ from this library's";
    if (h._pad0 || h._pad1) return "pool segment header padding is not zero";
    if (h.chunk_w != T.chunk_w || h.chunk_h != T.chunk_h || h.nlayers != T.nlayers)
        return "pool segment map geometry (chunk_w, chunk_h, nlayers) differs from the context's";
    if (h.ndests != T.ndests || h.max != T.max) return "pool segment geometry (ndests, max_fields) differs from the context's pool";
    const size_t chunks = (size_t)T.chunk_w * T.chunk_h, nkeys = (size_t)T.ndests * chunks, mx = (size_t)T.max;
    if (h.used < 0 || h.used > h.max || h.nzone < 0 || h.nzone > h.used || h.nfree > (uint32_t)h.used ||
        h.naux > (uint32_t)h.ndests || h.nstored > (uint32_t)h.used || h.nfp >= (1u << 24))
        return "pool segment counts outside the pool";
    I.L = pf_pool_layout_of(nkeys, mx, h.nfree, h.naux, h.nfp, h.nstored);
    const pf_pool_layout &L = I.L;
    if (size != L.size) return "pool segment size does not match its header (truncated or padded)";
    if (h.digest != T.digest) return "pool segment was saved on another map (map digest differs)";
    I.base = b;
    pf_pool_read(I.slot, b + L.slot, nkeys);
    pf_pool_read(I.ffid, b + L.ffid, nkeys);
    pf_pool_read(I.has, b + L.has, mx);
    pf_pool_read(I.req, b + L.req, mx);
    pf_pool_read(I.touch, b + L.touch, mx);
    pf_pool_read(I.owner, b + L.owner, mx);
    pf_pool_read(I.free_list, b + L.free, h.nfree);
    pf_pool_read(I.dtouch, b + L.dtouch, mx);
    const int used = h.used;
    // the slot table: entries in [-1, used), each slot mapped by at most one key
    std::vector<int64_t> key_of(mx, -1);
    for (size_t k = 0; k < nkeys; k++) {
        const int32_t s = I.slot[k];
        if (s < -1 || s >= h.max) return "slot-table entry outside the pool";
        if (s < 0) {
            if (I.ffid[k]) return "an ff_id on an unmapped key";
            continue;
        }
        if (s >= used) return "a key is mapped to a slot at or above used";
        if (key_of[s] >= 0) return "a slot is mapped by more than one key";
        key_of[s] = (int64_t)k;
    }
    // the free list: distinct entries below used, unmapped, no owner, no fields
    std::vector<uint8_t> freed(mx, 0);
    for (int32_t s : I.free_list) {
        if (s < 0 || s >= used) return "free-list entry outside [0, used)";
        if (freed[s]) return "free-list entry repeated";
        freed[s] = 1;
        if (key_of[s] >= 0 || I.owner[s] != -1 || I.has[s]) return "free-list entry is mapped, owned or has fields";
    }
    // every slot below used: free, owned by the key that maps it, or zone-held (mapped, no owner); nothing above
    int nzone = 0;
    uint32_t nstored = 0;
    for (int s = 0; s < h.max; s++) {
        const int64_t o = I.owner[s];
        if (s >= used) {
            if (o != -1 || I.has[s]) return "a slot at or above used is owned or has fields";
        } else if (!freed[s]) {
            if (key_of[s] < 0) return "a used slot is neither free, owned nor zone-held";
            if (o == -1) nzone++;
            else if (o != key_of[s]) return "an owned slot is not mapped by its owner";
        }
        if (I.has[s] & ~3u) return "a has byte with bits outside flow | LOS";
        if (I.has[s]) { nstored++; I.stored.push_back(s); }
        if (I.touch[s] > h.tick_no || I.dtouch[s] > h.tick_no) return "a touch stamp is above tick_no";
        if ((I.has[s] & 1) && (I.req[s].layer < 0 || I.req[s].layer >= T.nlayers))
            return "the request of a built flow field names a layer that is not created";
    }
    if (nzone != h.nzone) return "nzone does not count the zone-held slots";
    if (nstored != h.nstored) return "stored field count does not match the has bytes";
    // aux targets and their footprints
    I.aux.assign(h.naux, pf_aux_target());
    size_t f = 0;
    for (uint32_t d = 0; d < h.naux; d++) {
        pf_pool_aux_rec r;
        memcpy(&r, b + L.aux + (size_t)d * sizeof(r), sizeof(r));
        if (r.kind != -1 && r.kind != PFNAV_TARGET_ENTITY && r.kind != PFNAV_TARGET_ENEMIES) return "aux target with a bad kind";
        if (r.kind == -1 && (r.layer || r.ref_layer || r.nents)) return "aux target with a bad kind";
        if (r.kind == PFNAV_TARGET_ENTITY && r.nents != 1) return "aux target with a bad kind";
        if (r.layer < 0 || r.layer >= T.nlayers || r.ref_layer < 0 || r.ref_layer >= PFNAV_NAV_LAYER_MAX)
            return "aux target with a bad layer";
        if (r.nents > h.nfp - f) return "aux footprint counts do not add up";
        pf_aux_target &A = I.aux[d];
        A.kind = r.kind; A.layer = r.layer; A.ref_layer = r.ref_layer;
        pf_pool_read(A.ents, b + L.fp + f * sizeof(pfnav_footprint), r.nents);
        for (const pfnav_footprint &e : A.ents)
            if (!pf_finite(&e.x, 3) || !pf_finite(e.corners_xz, 8)) return "aux footprint not finite";
        f += r.nents;
    }
    if (f != h.nfp) return "aux footprint counts do not add up";
    return nullptr;
}

// Install a validated segment's bookkeeping in P (whose geometry it matches) and the aux targets; *tick_no: the saved tick
static inline void pf_pool_load(const pf_pool_image &I, pf_pool &P, std::vector<pf_aux_target> &aux, uint32_t *tick_no)
{
    P.used = I.h.used; P.nzone = I.h.nzone;
    P.slot = I.slot; P.ffid = I.ffid; P.has = I.has; P.req = I.req; P.touch = I.touch; P.owner = I.owner;
    P.free_list = I.free_list;
    aux = I.aux;
    *tick_no = I.h.tick_no;
}

// the hash primitives and the map digest (pfnav_digest_host.h builds on the layout above, so it comes last)
#include "pfnav_digest_host.h"
