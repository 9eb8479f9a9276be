// pfnav_digest_host.h -- the state digests, CUDA-free: the hash primitives, the committed-map digest (which ties a saved
// pool to its map), and the digests of the device-resident game state that pfnav_state_digest computes on the device
// (pfnav_digest.cu). Each state digest is defined here as a function of bytes a checkpoint segment already holds
// (pfnav_checkpoint_host.h, pfnav_pool_host.h), so that the host can compute it from a save without a GPU:
// pf_digest_agents_segment and pf_digest_pool_segment are those functions, and the device kernels call the per-item
// terms below. tests/emu/digest_emu.cpp builds this header with g++.
//
// Every value is a wrapping 64-bit integer sum of per-item terms, or a chain h = splitmix64(h ^ x) over 64-bit words.
// splitmix64 is a bijection of 64-bit words and x -> h ^ x is one for a fixed h, so a chain is a bijection in each of its
// words when the others are fixed: changing any one 8-byte word always changes a chain, and with it any sum it is a term
// of. Sums do not depend on their order, so every reduction order (the device's atomics, the host loops) gives the same
// bits, and the sums of a job's members add up to a single context's.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include "pfnav_pool_host.h"
#include "pfnav_checkpoint_host.h"

// ------------------------------------------------------------------------------------------
// Map digest: a 64-bit value over the committed map images, so that a saved pool is restored only onto the map its
// fields were built on. Tile t = r * 64 + c of block (layer, chunk) gives the word v = cost | blk << 8 | liid << 24 |
// fmask << 40 (fmask: the faction bit mask of the tile, 0 where the context keeps none); the block's hash is the wrapping
// sum over its 4096 tiles of splitmix64(v ^ t * K); the map's value is the wrapping sum over blocks of
// splitmix64(block hash ^ mix(layer, chunk)), folded with nlayers, chunk_w, chunk_h, the map position and the enemy table
// (pf_digest_fold). Integer sums do not depend on their order, so every reduction order (the device's k_map_digest, the
// host loop below) gives the same bits.
// ------------------------------------------------------------------------------------------
#define PF_DIGEST_K   0xD6E8FEB86659FD93ull
#define PF_DIGEST_MIX 0xA0761D6478BD642Full

PF_HD uint64_t pf_splitmix64(uint64_t x)
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
PF_HD uint64_t pf_digest_tile(uint32_t t, uint32_t cost, uint32_t blk, uint32_t liid, uint32_t fmask)
{
    const uint64_t v = (uint64_t)cost | (uint64_t)blk << 8 | (uint64_t)liid << 24 | (uint64_t)fmask << 40;
    return pf_splitmix64(v ^ (uint64_t)t * PF_DIGEST_K);
}
PF_HD uint64_t pf_digest_block(uint64_t block_hash, int layer, int chunk)
{
    return pf_splitmix64(block_hash ^ ((uint64_t)(uint32_t)layer << 32 | (uint32_t)chunk) * PF_DIGEST_MIX);
}
PF_HD uint64_t pf_digest_fold(uint64_t blocks, int nlayers, int chunk_w, int chunk_h, float map_x, float map_z,
                              const uint16_t enemies[16])
{
    uint32_t bx, bz;
    memcpy(&bx, &map_x, 4); memcpy(&bz, &map_z, 4);
    const uint64_t v[5] = {(uint64_t)nlayers, (uint64_t)chunk_w, (uint64_t)chunk_h, bx, bz};
    uint64_t h = blocks;
    for (uint64_t x : v) h = pf_splitmix64(h ^ x);
    for (int f = 0; f < 16; f++) h = pf_splitmix64(h ^ enemies[f]);
    return h;
}
// The digest over chunk-blocked images ([layer][chunk][64][64], the host mirrors' layout); fmask may be NULL (zeros).
static inline uint64_t pf_map_digest_host(const uint8_t *cost, const uint16_t *blk, const uint16_t *liid, const uint16_t *fmask,
                                          int nlayers, int chunk_w, int chunk_h, float map_x, float map_z, const uint16_t enemies[16])
{
    const int chunks = chunk_w * chunk_h;
    uint64_t sum = 0;
    for (int l = 0; l < nlayers; l++)
        for (int c = 0; c < chunks; c++) {
            const size_t base = ((size_t)l * chunks + c) * 4096;
            uint64_t b = 0;
            for (uint32_t t = 0; t < 4096; t++)
                b += pf_digest_tile(t, cost[base + t], blk[base + t], liid[base + t], fmask ? fmask[base + t] : 0);
            sum += pf_digest_block(b, l, c);
        }
    return pf_digest_fold(sum, nlayers, chunk_w, chunk_h, map_x, map_z, enemies);
}


// ------------------------------------------------------------------------------------------
// State digests.
//   population  the wrapping sum, over the uids u of the context's own range, of the row hash of u: the chain that starts
//               at splitmix64(u * K ^ tables ^ SEED_ROW) and takes, for each 16-byte word of the row pfnav_agents_save
//               writes for u (pfnav_checkpoint_host.h: agent, then movestate, movestate_ext, formation and blocking records
//               where the tables exist), its low then its high 8 bytes.
//   blocks      the same sum restricted to the uids [b * 2^k, (b + 1) * 2^k), for b < ceil(n_total / 2^k): a member's
//               array is zero outside its range, so members' arrays add up element-wise to a single context's.
//   flocks      the chain from splitmix64(nflocks ^ SEED_FLOCK) over the 8-byte words of the flock table, in order.
//   records     the wrapping sum over the whole population of the record hash of (u, the 24-byte neighbour record of u):
//               the chain from splitmix64(u * K ^ SEED_REC) over the record's three 8-byte words {px, pz}, {vx, vz},
//               {radius, state << 24 | flags & 0xFFFFFF}. The record is derived from the agent record, so the host
//               computes it from the segments' rows; each segment gives the sum over its own rows.
//   map         the committed-map digest above.
//   pool        step(host chain, device sum): the host chain runs from splitmix64(bytes ^ SEED_POOL) over the 8-byte
//               words of the segment pfnav_pool_save writes, from its start up to the device touch stamps, with the
//               header's map digest word taken as zero (the map is a component of its own); the device sum is the
//               wrapping sum of pf_digest_touch(s, device stamp of s) over every slot s < max and, for every slot s with
//               a `has` byte, of pf_digest_slot(s, the sum over the 512 16-byte words w of its flow then LOS bytes of
//               pf_digest_field_word(w, word)).
// ------------------------------------------------------------------------------------------
#define PF_DIGEST_SEED_ROW   0x8EBC6AF09C88C6E3ull
#define PF_DIGEST_SEED_REC   0x589965CC75374CC3ull
#define PF_DIGEST_SEED_FLOCK 0x1D8E4E27C47D124Full
#define PF_DIGEST_SEED_POOL  0xE7037ED1A0B428DBull
#define PF_DIGEST_SEED_FIELD 0x2D358DCCAA6C78A5ull
#define PF_DIGEST_SEED_TOUCH 0x8BB84B93962EACC9ull
#define PF_DIGEST_BLOCK_MIN  6                  // the range of block_log2: a warp's 32 uids never span two blocks
#define PF_DIGEST_BLOCK_MAX  20

PF_HD uint64_t pf_digest_step(uint64_t h, uint64_t x) { return pf_splitmix64(h ^ x); }
// one 16-byte word of a chain: its low 8 bytes, then its high 8 bytes
PF_HD uint64_t pf_digest_word(uint64_t h, uint64_t lo, uint64_t hi) { return pf_digest_step(pf_digest_step(h, lo), hi); }
PF_HD uint64_t pf_digest_row_begin(uint64_t uid, uint32_t tables)
{
    return pf_splitmix64(uid * PF_DIGEST_K ^ (uint64_t)tables ^ PF_DIGEST_SEED_ROW);
}
PF_HD uint64_t pf_digest_record(uint64_t uid, uint64_t w0, uint64_t w1, uint64_t w2)
{
    return pf_digest_step(pf_digest_word(pf_splitmix64(uid * PF_DIGEST_K ^ PF_DIGEST_SEED_REC), w0, w1), w2);
}
PF_HD uint64_t pf_digest_touch(uint32_t slot, uint32_t stamp)
{
    return pf_splitmix64(((uint64_t)slot << 32 | stamp) ^ PF_DIGEST_SEED_TOUCH);
}
PF_HD uint64_t pf_digest_field_word(uint32_t w, uint64_t lo, uint64_t hi)
{
    return pf_digest_word(pf_splitmix64((uint64_t)w * PF_DIGEST_K ^ PF_DIGEST_SEED_FIELD), lo, hi);
}
PF_HD uint64_t pf_digest_slot(uint32_t slot, uint64_t field_sum)
{
    return pf_splitmix64(field_sum ^ (uint64_t)slot * PF_DIGEST_MIX ^ PF_DIGEST_SEED_POOL);
}
static inline size_t pf_digest_nblocks(size_t n_total, int k) { return (n_total + ((size_t)1 << k) - 1) >> k; }

static inline uint64_t pf_digest_load64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }

// the neighbour record's three words of an agent record, as k_make_records and k_entity_apply pack it
static inline void pf_digest_record_words(const pfnav_agent &a, uint64_t w[3])
{
    uint32_t v[6];
    memcpy(&v[0], &a.pos[0], 4); memcpy(&v[1], &a.pos[1], 4);
    memcpy(&v[2], &a.velocity[0], 4); memcpy(&v[3], &a.velocity[1], 4);
    memcpy(&v[4], &a.radius, 4);
    v[5] = (a.state << 24) | (a.flags & 0xFFFFFFu);
    for (int i = 0; i < 3; i++) w[i] = (uint64_t)v[2 * i] | (uint64_t)v[2 * i + 1] << 32;
}

static inline uint64_t pf_digest_flocks(const pfnav_flock *flocks, size_t nflocks)
{
    uint64_t h = pf_splitmix64((uint64_t)nflocks ^ PF_DIGEST_SEED_FLOCK);
    const uint8_t *p = (const uint8_t *)flocks;
    for (size_t i = 0; i < nflocks * sizeof(pfnav_flock) / 8; i++) h = pf_digest_step(h, pf_digest_load64(p + i * 8));
    return h;
}

// the host chain of the pool digest over a segment's first `bytes` bytes (a multiple of 8: the offset of the device touch
// stamps), the header's map digest word taken as zero
static inline uint64_t pf_digest_pool_host(const uint8_t *seg, size_t bytes)
{
    uint64_t h = pf_splitmix64((uint64_t)bytes ^ PF_DIGEST_SEED_POOL);
    for (size_t o = 0; o < bytes; o += 8)
        h = pf_digest_step(h, o == offsetof(pf_pool_header, digest) ? 0 : pf_digest_load64(seg + o));
    return h;
}

// the field sum of one stored slot's 8192 bytes (flow then LOS), the term pf_digest_slot takes
static inline uint64_t pf_digest_field_sum(const uint8_t *fields)
{
    uint64_t s = 0;
    for (uint32_t w = 0; w < 512; w++)
        s += pf_digest_field_word(w, pf_digest_load64(fields + w * 16), pf_digest_load64(fields + w * 16 + 8));
    return s;
}

// What one checkpoint segment contributes: its population and records sums over its rows, the flock chain of the table it
// carries, and its header.
struct pf_digest_agents {
    uint64_t population = 0, flocks = 0, records = 0;
    pf_ckpt_header h;
};

// The digests of one pfnav_agents_save segment (size bytes). blocks_out, when given, has pf_digest_nblocks(n_total, k)
// entries and each row's hash is added to entry uid >> k (the caller zeroes it; several segments add into one array).
// Returns NULL, or what is wrong with the segment's header or size (nothing is written then).
static inline const char *pf_digest_agents_segment(const void *seg, size_t size, int k, uint64_t *blocks_out, pf_digest_agents *out)
{
    if (!seg || size < sizeof(pf_ckpt_header)) return "segment shorter than its header";
    if (k < PF_DIGEST_BLOCK_MIN || k > PF_DIGEST_BLOCK_MAX) return "block_log2 outside 6..20";
    const uint8_t *b = (const uint8_t *)seg;
    pf_ckpt_header h;
    memcpy(&h, b, sizeof(h));
    if (h.magic != PF_CKPT_MAGIC || h.version != PF_CKPT_VERSION) return "not a checkpoint segment of this version";
    if (memcmp(h.rec_size, pf_ckpt_sizes, sizeof(h.rec_size))) return "checkpoint record sizes differ from this library's";
    if ((h.tables & ~PF_CKPT_TABLES) || h.lo > h.hi || h.hi > h.n_total || h.n_total >= (1u << 31) || h.nflocks >= (1u << 24))
        return "checkpoint header out of range";
    if (size != pf_ckpt_bytes(h.tables, h.nflocks, h.hi - h.lo)) return "segment size does not match its header";
    const pf_ckpt_row R = pf_ckpt_row_of(h.tables);
    const uint8_t *rows = b + sizeof(pf_ckpt_header) + (size_t)h.nflocks * sizeof(pfnav_flock);
    pf_digest_agents d;
    d.h = h;
    d.flocks = pf_digest_flocks((const pfnav_flock *)(b + sizeof(pf_ckpt_header)), h.nflocks);
    for (uint64_t u = h.lo; u < h.hi; u++) {
        const uint8_t *row = rows + (u - h.lo) * R.words * 16;
        uint64_t x = pf_digest_row_begin(u, h.tables);
        for (uint32_t q = 0; q < R.words; q++) x = pf_digest_word(x, pf_digest_load64(row + q * 16), pf_digest_load64(row + q * 16 + 8));
        d.population += x;
        if (blocks_out) blocks_out[u >> k] += x;
        pfnav_agent a;
        memcpy(&a, row, sizeof(a));
        uint64_t w[3];
        pf_digest_record_words(a, w);
        d.records += pf_digest_record(u, w[0], w[1], w[2]);
    }
    *out = d;
    return nullptr;
}

// The pool digest of one pfnav_pool_save segment (size bytes) into *out. Returns NULL, or what is wrong with its header or
// size (nothing is written then).
static inline const char *pf_digest_pool_segment(const void *seg, size_t size, uint64_t *out)
{
    if (!seg || size < sizeof(pf_pool_header)) return "segment shorter than its header";
    const uint8_t *b = (const uint8_t *)seg;
    pf_pool_header h;
    memcpy(&h, b, sizeof(h));
    if (h.magic != PF_POOL_MAGIC || h.version != PF_POOL_VERSION) return "not a pool segment of this version";
    if (h.ndests < 0 || h.max < 0 || h.nstored > (uint32_t)h.max) return "pool header out of range";
    const size_t nkeys = (size_t)h.ndests * h.chunk_w * h.chunk_h;
    const pf_pool_layout L = pf_pool_layout_of(nkeys, (size_t)h.max, h.nfree, h.naux, h.nfp, h.nstored);
    if (size != L.size) return "segment size does not match its header";
    uint64_t dev = 0;
    uint32_t b_at = 0;
    for (int s = 0; s < h.max; s++) {
        uint32_t stamp;
        memcpy(&stamp, b + L.dtouch + (size_t)s * 4, 4);
        dev += pf_digest_touch((uint32_t)s, stamp);
        if (b[L.has + s] && b_at < h.nstored) dev += pf_digest_slot((uint32_t)s, pf_digest_field_sum(b + L.fields + (size_t)b_at++ * 8192));
    }
    if (b_at != h.nstored) return "stored field count does not match the has bytes";
    *out = pf_digest_step(pf_digest_pool_host(b, L.dtouch), dev);
    return nullptr;
}
