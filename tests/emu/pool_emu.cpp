// tests/emu/pool_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the field pool's host bookkeeping and slot policies
// (permafrost-engine_b200/csrc/pfnav_pool_host.h, unmodified), so that tests/test_pool_emu.py can run the real LRU
// reservation and zone rule on random sequences and check them against a Python restatement. This is not a product path:
// nothing in libpfnav.so links or calls it, and it is built only by tests/test_pool_emu.py.
#include <stdarg.h>
#include <stdio.h>
#include "../../permafrost-engine_b200/csrc/pfnav_pool_host.h"

void pfnav_set_error(const char *, ...) {}

extern "C" {

void *emu_pool_new(int ndests, int chunks, int max)
{
    pf_pool *P = new pf_pool;
    P->ndests = ndests; P->max = max;
    P->slot.assign((size_t)ndests * chunks, -1); P->ffid.assign((size_t)ndests * chunks, 0);
    P->has.assign(max, 0); P->req.assign(max, pfnav_field_req{}); P->touch.assign(max, 0); P->owner.assign(max, -1);
    return P;
}

void emu_pool_delete(void *h) { delete (pf_pool *)h; }

// dev: the device's touch stamps, merged when the reservation must evict; *out_called: whether it asked for them
int emu_pool_reserve(void *h, const uint64_t *keys, int n, uint32_t tick, const uint32_t *dev, int32_t *slots_out,
                     int *out_evicted, int *out_called)
{
    pf_pool &P = *(pf_pool *)h;
    std::vector<size_t> k(keys, keys + n);
    bool evicted = false;
    *out_called = 0;
    const int rc = pf_pool_reserve(P, k.data(), k.size(), tick, slots_out, &evicted, [&](std::vector<uint32_t> &stamp) {
        *out_called = 1;
        for (int s = 0; s < P.max; s++) stamp[s] = std::max(stamp[s], dev[s]);
        return (int)PFNAV_OK;
    });
    *out_evicted = evicted;
    return rc;
}

int emu_pool_fits(void *h, const uint64_t *keys, int n)
{
    std::vector<size_t> k(keys, keys + n);
    return pf_pool_fits(*(pf_pool *)h, k.data(), k.size());
}

int emu_pool_zone_fits(void *h, const uint64_t *keys, int n)
{
    std::vector<size_t> k(keys, keys + n);
    return pf_pool_zone_fits(*(pf_pool *)h, k.data(), k.size());
}

int emu_pool_zone_take(void *h, uint64_t key) { return pf_pool_zone_take(*(pf_pool *)h, key); }

void emu_pool_built(void *h, uint64_t key, int bits)
{
    pf_pool &P = *(pf_pool *)h;
    if (P.slot_of(key) >= 0) P.built(P.slot_of(key), (uint8_t)bits);
}

void emu_pool_drop(void *h, uint64_t key) { pf_pool_drop(*(pf_pool *)h, key); }

void emu_pool_reset(void *h) { pf_pool_reset(*(pf_pool *)h); }

// slot table, owners, `has` bytes, touch stamps, free list (returns its length); counters: used, nzone
int emu_pool_state(void *h, int32_t *slot, int64_t *owner, uint8_t *has, uint32_t *touch, int32_t *free_list, int64_t *counters)
{
    const pf_pool &P = *(const pf_pool *)h;
    std::copy(P.slot.begin(), P.slot.end(), slot);
    std::copy(P.owner.begin(), P.owner.end(), owner);
    std::copy(P.has.begin(), P.has.end(), has);
    std::copy(P.touch.begin(), P.touch.end(), touch);
    std::copy(P.free_list.begin(), P.free_list.end(), free_list);
    counters[0] = P.used; counters[1] = P.nzone;
    return (int)P.free_list.size();
}

}
