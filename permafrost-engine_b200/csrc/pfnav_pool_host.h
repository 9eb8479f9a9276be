// pfnav_pool_host.h -- the field pool's host bookkeeping and its two slot policies. No CUDA: the device side is
// pfnav_pool.cu, and tests/test_pool_emu.py compiles this header with g++ to run the real policies.
//
// One slot holds the flow AND the LOS field of a (dest, chunk) key, key = dest * chunks + chunk. Every slot below `used`
// is in exactly one of three states: on the free list, owned by the key pf_pool_reserve gave it to (evictable), or taken
// by the zone rule (pf_pool_zone_take: no owner, never evicted, held until the pool is cleared). Only the functions here
// and in pfnav_pool.cu write the slot table, the owners, the free list and `used`.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <algorithm>
#include <vector>
#include "../../include/pfnav.h"

void pfnav_set_error(const char *fmt, ...);

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
