// tests/emu/pool_checkpoint_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the pool segment of pfnav_pool_save /
// pfnav_pool_restore and the map digest (permafrost-engine_b200/csrc/pfnav_pool_host.h, unmodified), so that
// tests/test_pool_checkpoint_emu.py can build pools with the real slot policies, save, validate and load them, and check
// the digest against a numpy restatement. The device part of a context is played by two host arrays: the device touch
// stamps and every slot's flow and LOS bytes, which the save packs and the load scatters as k_pool_pack / k_pool_unpack
// do. This is not a product path: nothing in libpfnav.so links or calls it, and it is built only by the test.
#include <stdarg.h>
#include <stdio.h>
#include "../../permafrost-engine_b200/csrc/pfnav_pool_host.h"

void pfnav_set_error(const char *, ...) {}

struct emu_ctx {
    pf_pool P;
    std::vector<pf_aux_target> aux;
    uint32_t tick_no = 1;
    std::vector<uint32_t> dtouch;             // the device touch stamps
    std::vector<uint8_t> fields;              // [max][8192]: flow then LOS bytes of every slot
};

extern "C" {

void *emu_pc_new(int ndests, int chunks, int max)
{
    emu_ctx *E = new emu_ctx;
    pf_pool &P = E->P;
    P.ndests = ndests; P.max = max;
    P.slot.assign((size_t)ndests * chunks, -1); P.ffid.assign((size_t)ndests * chunks, 0);
    P.has.assign(max, 0); P.req.assign(max, pfnav_field_req{}); P.touch.assign(max, 0); P.owner.assign(max, -1);
    E->dtouch.assign(max, 0);
    E->fields.assign((size_t)max * 8192, 0);
    return E;
}

void *emu_pc_clone(void *h) { return new emu_ctx(*(emu_ctx *)h); }
void emu_pc_delete(void *h) { delete (emu_ctx *)h; }

void emu_pc_set_tick(void *h, uint32_t tick) { ((emu_ctx *)h)->tick_no = tick; }

// pf_pool_reserve at the context's tick with the given device stamps (raised into the context's first)
int emu_pc_reserve(void *h, const uint64_t *keys, int n, const uint32_t *dev)
{
    emu_ctx &E = *(emu_ctx *)h;
    for (int s = 0; s < E.P.max; s++) E.dtouch[s] = std::max(E.dtouch[s], std::min(dev[s], E.tick_no));
    std::vector<size_t> k(keys, keys + n);
    bool evicted = false;
    return pf_pool_reserve(E.P, k.data(), k.size(), E.tick_no, nullptr, &evicted, [&](std::vector<uint32_t> &stamp) {
        for (int s = 0; s < E.P.max; s++) stamp[s] = std::max(stamp[s], E.dtouch[s]);
        return (int)PFNAV_OK;
    });
}

int emu_pc_zone_take(void *h, uint64_t key) { return pf_pool_zone_take(((emu_ctx *)h)->P, key); }

// fields built into the key's slot: bits 1 (flow, with a request on `layer`) and 2 (LOS); the bytes come from `bytes`
// (8192: flow then LOS); a mapped key gets ff_id `ffid`
void emu_pc_built(void *h, uint64_t key, int bits, int layer, uint64_t ffid, const uint8_t *bytes)
{
    emu_ctx &E = *(emu_ctx *)h;
    const int32_t s = E.P.slot_of(key);
    if (s < 0) return;
    if (bits & 1) {
        pfnav_field_req q;
        memset(&q, 0, sizeof(q));
        q.layer = layer; q.chunk_r = (int32_t)(key % 7); q.target_type = 1; q._pad = (int32_t)key;
        E.P.built_flow(s, q);
        memcpy(E.fields.data() + (size_t)s * 8192, bytes, 4096);
    }
    if (bits & 2) {
        E.P.built(s, 2);
        memcpy(E.fields.data() + (size_t)s * 8192 + 4096, bytes + 4096, 4096);
    }
    E.P.ffid[key] = ffid;
}

void emu_pc_drop(void *h, uint64_t key) { pf_pool_drop(((emu_ctx *)h)->P, key); }
void emu_pc_reset(void *h) { pf_pool_reset(((emu_ctx *)h)->P); std::fill(((emu_ctx *)h)->dtouch.begin(), ((emu_ctx *)h)->dtouch.end(), 0); }

void emu_pc_set_aux(void *h, int dest, int kind, int layer, int ref_layer, const pfnav_footprint *ents, int n)
{
    emu_ctx &E = *(emu_ctx *)h;
    if (E.aux.size() < (size_t)E.P.ndests) E.aux.resize(E.P.ndests);
    pf_aux_target &A = E.aux[dest];
    A.kind = kind; A.layer = layer; A.ref_layer = ref_layer; A.ents.assign(ents, ents + n);
}

static pf_pool_target target(const emu_ctx &E, int chunk_w, int chunk_h, int nlayers, uint64_t digest)
{
    return {chunk_w, chunk_h, nlayers, E.P.ndests, E.P.max, digest};
}

// the segment's size; then the save itself into out (the host part, the device stamps and the stored slots' bytes)
size_t emu_pc_size(void *h)
{
    emu_ctx &E = *(emu_ctx *)h;
    std::vector<int32_t> stored;
    return pf_pool_seg_plan(E.P, E.aux, stored).size;
}

size_t emu_pc_save(void *h, int chunk_w, int chunk_h, int nlayers, uint64_t digest, uint8_t *out)
{
    emu_ctx &E = *(emu_ctx *)h;
    std::vector<int32_t> stored;
    const pf_pool_layout L = pf_pool_seg_plan(E.P, E.aux, stored);
    pf_pool_seg_write(E.P, E.aux, target(E, chunk_w, chunk_h, nlayers, digest), E.tick_no, stored, L, out);
    memset(out + L.dtouch, 0, L.size - L.dtouch);
    memcpy(out + L.dtouch, E.dtouch.data(), (size_t)E.P.max * 4);
    for (size_t b = 0; b < stored.size(); b++) memcpy(out + L.fields + b * 8192, E.fields.data() + (size_t)stored[b] * 8192, 8192);
    return L.size;
}

// validate and load; 0 on success, 1 with the message in err (256 bytes) on a refusal, which must change nothing
int emu_pc_load(void *h, const uint8_t *seg, size_t size, int chunk_w, int chunk_h, int nlayers, uint64_t digest, char *err)
{
    emu_ctx &E = *(emu_ctx *)h;
    pf_pool_image I;
    const char *e = pf_pool_check(seg, size, target(E, chunk_w, chunk_h, nlayers, digest), I);
    if (e) {
        snprintf(err, 256, "%s", e);
        return 1;
    }
    memcpy(E.dtouch.data(), I.base + I.L.dtouch, (size_t)E.P.max * 4);
    for (size_t b = 0; b < I.stored.size(); b++)
        memcpy(E.fields.data() + (size_t)I.stored[b] * 8192, I.base + I.L.fields + b * 8192, 8192);
    pf_pool_load(I, E.P, E.aux, &E.tick_no);
    return 0;
}

// every member of the pool, the aux targets and the tick; with fields != 0 also the device stamps and the bytes of every
// slot with a `has` bit
int emu_pc_equal(void *a, void *b, int fields)
{
    const emu_ctx &A = *(const emu_ctx *)a, &B = *(const emu_ctx *)b;
    const pf_pool &P = A.P, &Q = B.P;
    if (P.ndests != Q.ndests || P.max != Q.max || P.used != Q.used || P.nzone != Q.nzone) return 0;
    if (P.slot != Q.slot || P.ffid != Q.ffid || P.has != Q.has || P.touch != Q.touch || P.owner != Q.owner ||
        P.free_list != Q.free_list)
        return 0;
    if (memcmp(P.req.data(), Q.req.data(), P.req.size() * sizeof(pfnav_field_req))) return 0;
    if (A.tick_no != B.tick_no || A.aux.size() != B.aux.size()) return 0;
    for (size_t d = 0; d < A.aux.size(); d++) {
        const pf_aux_target &x = A.aux[d], &y = B.aux[d];
        if (x.kind != y.kind || x.layer != y.layer || x.ref_layer != y.ref_layer || x.ents.size() != y.ents.size()) return 0;
        if (!x.ents.empty() && memcmp(x.ents.data(), y.ents.data(), x.ents.size() * sizeof(pfnav_footprint))) return 0;
    }
    if (fields) {
        if (A.dtouch != B.dtouch) return 0;
        for (int s = 0; s < P.max; s++)
            if (P.has[s] && memcmp(A.fields.data() + (size_t)s * 8192, B.fields.data() + (size_t)s * 8192, 8192)) return 0;
    }
    return 1;
}

// counters: used, nzone, nfree, tick
void emu_pc_counts(void *h, int64_t *out)
{
    const emu_ctx &E = *(const emu_ctx *)h;
    out[0] = E.P.used; out[1] = E.P.nzone; out[2] = (int64_t)E.P.free_list.size(); out[3] = E.tick_no;
}

uint64_t emu_pc_digest(const uint8_t *cost, const uint16_t *blk, const uint16_t *liid, const uint16_t *fmask, int nlayers,
                       int chunk_w, int chunk_h, float map_x, float map_z, const uint16_t *enemies)
{
    return pf_map_digest_host(cost, blk, liid, fmask, nlayers, chunk_w, chunk_h, map_x, map_z, enemies);
}

// the per-tile and per-block terms, for the restatement's order tests
uint64_t emu_pc_digest_tile(uint32_t t, uint32_t cost, uint32_t blk, uint32_t liid, uint32_t fmask)
{
    return pf_digest_tile(t, cost, blk, liid, fmask);
}
uint64_t emu_pc_digest_block(uint64_t b, int layer, int chunk) { return pf_digest_block(b, layer, chunk); }

}
