// pfnav_los_kernel.cuh -- the device code of the LOS field kernels k_los_b (byte-state heap replay) and k_los_level
// (level-parallel pass with a certificate, falling back to the replay), kept in a header of its own so that tests/emu
// can run the SAME source on CPU threads (tests/emu/los_emu.cpp defines the CUDA keywords and warp intrinsics it uses as
// plain C++); pfnav_fields.cu includes it. Also the bit helpers and FlowGrids that the other field kernels share.
// Needs: <stdint.h>, pfnav.h, uint4 and the warp intrinsics.
#pragma once

// ------------------------------------------------------------------------------------------
// bit helpers
// ------------------------------------------------------------------------------------------
// 4 byte-masks (0xFF/0x00) -> 4 bits
__device__ __forceinline__ uint32_t bytemask_to_bits(uint32_t m)
{
    return (((m & 0x01010101u) * 0x01020408u) >> 24) & 0xFu;
}
// bits for 16 cost bytes: impassable (==0xFF) and "not unit" (!= 1)
__device__ __forceinline__ void cost16_bits(const uint4 v, uint32_t &imp, uint32_t &nonunit)
{
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    imp = 0; nonunit = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        imp |= bytemask_to_bits(__vcmpeq4(w[i], 0xFFFFFFFFu)) << (4 * i);
        nonunit |= bytemask_to_bits(__vcmpne4(w[i], 0x01010101u)) << (4 * i);
    }
}
// bits for 8 u16 blockers: nonzero
__device__ __forceinline__ uint32_t blk8_bits(const uint4 v)
{
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t r = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        uint32_t b = ((w[i] & 0xFFFFu) ? 1u : 0u) | ((w[i] >> 16) ? 2u : 0u);
        r |= b << (2 * i);
    }
    return r;
}
// 4 bits -> 4 bytes (bit j -> bit 0 of byte j)
__device__ __forceinline__ uint32_t spread4(uint32_t x) { return ((x & 0xFu) * 0x00204081u) & 0x01010101u; }

__device__ __forceinline__ uint64_t shfl_up64(uint64_t v, uint32_t lane)
{
    uint32_t lo = __shfl_up_sync(0xffffffffu, (uint32_t)v, 1);
    uint32_t hi = __shfl_up_sync(0xffffffffu, (uint32_t)(v >> 32), 1);
    return lane == 0 ? 0ull : (((uint64_t)hi << 32) | lo);
}
__device__ __forceinline__ uint64_t shfl_down64(uint64_t v, uint32_t lane)
{
    uint32_t lo = __shfl_down_sync(0xffffffffu, (uint32_t)v, 1);
    uint32_t hi = __shfl_down_sync(0xffffffffu, (uint32_t)(v >> 32), 1);
    return lane == 31 ? 0ull : (((uint64_t)hi << 32) | lo);
}

struct FlowGrids {
    const uint8_t *cost;     // [layer][H64][W64]
    const uint16_t *blk;
    const uint16_t *liid;
    const uint8_t *unit;     // [layer][chunks]
    int W64, H64, chunk_w, chunk_h;
    const uint16_t *fmask;   // [layer][H64][W64] bit f <=> faction f holds a blocker refcount on the tile
    uint16_t enemies[16];    // enemies[f]: factions at war with f
};

// ------------------------------------------------------------------------------------------
// K3: LOS field. One warp per field.
// ------------------------------------------------------------------------------------------
#define LOS_WARPS_PER_CTA 4
// previous-chunk field bytes may have been written by another SM during this launch (dependency-driven
// scheduling): read them through L2
#define LOS_PREV_LOAD(p) __ldcg(p)

struct LosMapInfo {
    float map_x, map_z;
};

#ifndef pf_globaltimer
__device__ __forceinline__ unsigned long long pf_globaltimer()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#endif

// OR 64 bits into a shared-memory row with two native 32-bit reductions (a 64-bit shared atomicOr
// compiles to a compare-and-swap spin loop)
__device__ __forceinline__ void or_row(uint64_t *row, uint64_t bits)
{
    unsigned *w = reinterpret_cast<unsigned *>(row);
    const unsigned lo = (unsigned)bits, hi = (unsigned)(bits >> 32);
    if (lo) atomicOr(w, lo);
    if (hi) atomicOr(w + 1, hi);
}

// Byte-state variant of the LOS replay (k_los_b): one state byte per tile in a 66 x 66 array whose border ring
// carries LB_BORDER, so the four neighbour tests of a pop are four byte loads + mask compares with no bounds
// checks and no 64-bit variable shifts (the bit-row form spends ~75 of its ~300 instructions per pop on those).
#define LB_BLK    0x01   /* wavefront_blocked                                             */
#define LB_OPEN   0x02   /* passable for this request and cost <= 1                        */
#define LB_ASG    0x04   /* integration_field < INF (was pushed / is a seed)               */
#define LB_VIS    0x08   /* visible                                                        */
#define LB_PASS   0x10   /* plain passable (field_is_los_corner, field.c:435)              */
#define LB_BORDER 0x20   /* outside the chunk                                              */
#define LB_W 66
struct __align__(16) LosSmemB {
    uint8_t  st[LB_W * LB_W + 12];   // 4368
    uint64_t blkrow[64], visrow[64]; // bit rows for the final padding pass (k_los_level: BLK while it runs)
    union {
        uint16_t heap[4104];
        struct {                     // k_los_level, which has no heap until it falls back to the replay
            uint64_t walk[64];       // tiles of this level's lines after their first
            int32_t  esrc[64];       // edge seeding: 1 + the largest source index whose line covers an edge tile
            uint16_t list[32];       // one round of trigger tiles, r << 6 | c
        } lv;
    };
};
static_assert(sizeof(LosSmemB) % 16 == 0, "LosSmemB must keep 16-byte alignment per warp");

// field_create_wavefront_blocked_line (field.c:463-517) on the byte array
__device__ void los_blocked_line_b(LosSmemB &s, const LosMapInfo mi, int tgt_cr, int tgt_cc, int tgt_r, int tgt_c,
                                   int cr, int cc, int r, int c)
{
    const float tbx = (mi.map_x - (float)(tgt_cc * 256)) - (float)(tgt_c * 4);
    const float tbz = (mi.map_z + (float)(tgt_cr * 256)) + (float)(tgt_r * 4);
    const float cbx = (mi.map_x - (float)(cc * 256)) - (float)(c * 4);
    const float cbz = (mi.map_z + (float)(cr * 256)) + (float)(r * 4);
    const float tcx = tbx - 4.0f / 2.0f, tcz = tbz + 4.0f / 2.0f;
    const float ccx = cbx - 4.0f / 2.0f, ccz = cbz + 4.0f / 2.0f;
    float sx_ = tcx - ccx, sz_ = tcz - ccz;
    const float len = sqrtf(sx_ * sx_ + sz_ * sz_);
    sx_ = sx_ / len;
    sz_ = sz_ / len;
    if (!(len > 0.0f)) {
        // line from the target tile to itself: NaN slope, INT_MIN deltas, wrapped error term -- the reference walks the
        // row towards column 0 (see los_blocked_line)
        for (int idx0 = (r + 1) * LB_W + (c + 1); !(s.st[idx0] & LB_BORDER); idx0--) s.st[idx0] |= LB_BLK;
        return;
    }
    const int dx = abs((int)(sx_ * 1000));
    const int dy = -abs((int)(sz_ * 1000));
    const int sx = sx_ > 0.0f ? 1 : -1;
    const int sy = sz_ < 0.0f ? 1 : -1;
    int err = dx + dy, e2;
    int idx = (r + 1) * LB_W + (c + 1);
    uint8_t v = s.st[idx];
    // the walk ends on the border ring (LB_BORDER), which is never written
    while (!(v & LB_BORDER)) {
        s.st[idx] = v | LB_BLK;
        e2 = 2 * err;
        if (e2 >= dy) { err += dy; idx += sx; }
        if (e2 <= dx) { err += dx; idx += sy * LB_W; }
        v = s.st[idx];
    }
}

// Heap of the byte-state kernel: entries = prio2 << 13 | padded index ((r + 1) * 66 + c + 1 < 8192), so that a pop needs
// no unpacking and no address arithmetic before its four state loads. heap_remove_root is heap_pop without the read of
// the root: the caller reads h[1] first and issues the neighbour loads BEFORE the sift, whose dependent chain then hides them.
__device__ __forceinline__ void heap_remove_root13(uint16_t *h, int &size, uint32_t lowp)
{
    const uint16_t x = h[size];
    size--;
    int root = 1;
    if ((uint32_t)(x >> 13) != lowp) {
        const uint32_t *h2 = reinterpret_cast<const uint32_t *>(h);      // children 2k, 2k+1 share one aligned word
        while (true) {
            const int l = root * 2;
            if (l > size) break;
            const uint32_t two = h2[root];
            const bool dl = ((two >> 13) & 0x7u) == lowp, dr = l < size && (two >> 29) == lowp;
            if (!(dl || dr)) break;
            h[root] = (uint16_t)(dl ? two : two >> 16);
            root = dl ? l : l + 1;
        }
    }
    h[root] = x;
}

__device__ __forceinline__ const uint8_t *los_prev_field(const uint8_t *fields, const int32_t *out_slot, const pfnav_los_req &q)
{
    return fields + (size_t)(q.prev_index >= 0 ? (out_slot ? out_slot[q.prev_index] : q.prev_index) : q._pad) * 4096;
}

// which edge of this chunk is shared with the previous chunk (field.c:2122-2196): `horizontal` = the edge is a column
__device__ __forceinline__ void los_edge_of(const pfnav_los_req &q, bool &horizontal, int &curr_edge, int &prev_edge)
{
    if (q.prev_chunk_r < q.chunk_r)      { horizontal = false; curr_edge = 0;  prev_edge = 63; }
    else if (q.prev_chunk_r > q.chunk_r) { horizontal = false; curr_edge = 63; prev_edge = 0;  }
    else if (q.prev_chunk_c < q.chunk_c) { horizontal = true;  curr_edge = 0;  prev_edge = 63; }
    else                                 { horizontal = true;  curr_edge = 63; prev_edge = 0;  }
}

// The tile bits of one chunk row for one request: passb = plain passable (the corner rule, field.c:435), openb = passable
// for the request (field_tile_passable_no_enemies for an attacking one, field.c:179) with cost <= 1
__device__ __forceinline__ void los_stage_row(const FlowGrids &g, const pfnav_los_req &q, int row, uint64_t &passb, uint64_t &openb)
{
    const size_t off = ((size_t)q.layer * g.H64 + q.chunk_r * 64 + row) * g.W64 + q.chunk_c * 64;
    const uint4 *pc = reinterpret_cast<const uint4 *>(g.cost + off);
    const uint4 *pb = reinterpret_cast<const uint4 *>(g.blk + off);
    uint64_t p = 0, blocked = 0, gt1 = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const uint4 v = __ldg(pc + j);
        uint32_t imp, n1;
        cost16_bits(v, imp, n1);
        p |= (uint64_t)((~imp) & 0xFFFFu) << (16 * j);
        // cost > 1  <=>  cost not in {0, 1}
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t g1 = 0;
#pragma unroll
        for (int e = 0; e < 4; e++)
            g1 |= bytemask_to_bits(__vcmpgtu4(w[e], 0x01010101u)) << (4 * e);
        gt1 |= (uint64_t)g1 << (16 * j);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) blocked |= (uint64_t)blk8_bits(__ldg(pb + j)) << (8 * j);
    // an "attacking" request (dest_id carries a faction, field.c:2095) walks over tiles blocked only by its
    // enemies (field_tile_passable_no_enemies, field.c:179); the corner test keeps the plain rule (field.c:435)
    uint64_t blocked_f = blocked;
    if (q.faction_id != PFNAV_FACTION_ID_NONE && blocked) {
        const uint16_t en = g.enemies[q.faction_id & 0xF];
        const uint16_t *pf = g.fmask + off;
        for (uint64_t rest = blocked; rest; rest &= rest - 1) {
            const int c = __ffsll((long long)rest) - 1;
            if ((pf[c] & ~en) == 0) blocked_f &= ~(1ull << c);
        }
    }
    passb = p & ~blocked;
    openb = p & ~blocked_f & ~gt1;
}

// field_pad_wavefront (field.c:519) and the store: clear `visible` within 1 tile of a blocked tile, from the bit rows
// s.blkrow / s.visrow, and write the field's bytes (bit 0 visible, bit 1 wavefront_blocked)
__device__ __forceinline__ void los_store_b(const LosSmemB &s, uint8_t *dst, uint32_t lane)
{
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        const int row = 2 * lane + rr;
        uint64_t b = s.blkrow[row];
        if (row > 0) b |= s.blkrow[row - 1];
        if (row < 63) b |= s.blkrow[row + 1];
        b = b | (b << 1) | (b >> 1);
        const uint64_t vis = s.visrow[row] & ~b, w = s.blkrow[row];
        uint4 *d4 = reinterpret_cast<uint4 *>(dst + row * 64);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            uint32_t o[4];
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int sh = j * 16 + e * 4;
                o[e] = spread4((uint32_t)(vis >> sh)) | (spread4((uint32_t)(w >> sh)) << 1);
            }
            d4[j] = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}

// One whole field by the byte-state replay: stage, lane 0 replays the reference heap, pad and store. Returns the
// number of heap pops (lane 0; 0 on the other lanes).
__device__ unsigned los_field_replay_b(LosSmemB &s, const FlowGrids &g, const LosMapInfo mi, const pfnav_los_req &q,
                                       const uint8_t *fields, const int32_t *out_slot, uint8_t *dst, uint32_t lane)
{
    // ---- stage tile -> state bytes (2 rows per lane) ----
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        const int row = 2 * lane + rr;
        uint64_t passb, openb;
        los_stage_row(g, q, row, passb, openb);
        uint8_t *rowp = s.st + (row + 1) * LB_W + 1;
#pragma unroll 8
        for (int c = 0; c < 64; c++)
            rowp[c] = (uint8_t)((((passb >> c) & 1) ? LB_PASS : 0) | (((openb >> c) & 1) ? LB_OPEN : 0));
        rowp[-1] = LB_BORDER; rowp[64] = LB_BORDER;
    }
    for (int c = lane; c < LB_W; c += 32) { s.st[c] = LB_BORDER; s.st[65 * LB_W + c] = LB_BORDER; }
    __syncwarp();

    unsigned npops = 0;
    if (lane == 0) {
        uint16_t *h = s.heap;
        int size = 0;
        const bool dest_chunk = (q.chunk_r == q.tgt_chunk_r && q.chunk_c == q.tgt_chunk_c);
        if (dest_chunk) {
            h[++size] = (uint16_t)((q.tgt_tile_r + 1) * LB_W + q.tgt_tile_c + 1);
            s.st[(q.tgt_tile_r + 1) * LB_W + q.tgt_tile_c + 1] |= LB_ASG;
        } else {
            // carry the shared edge over from the previous chunk's field (field.c:2122-2196)
            const uint8_t *prev = los_prev_field(fields, out_slot, q);
            bool horizontal; int curr_edge, prev_edge;
            los_edge_of(q, horizontal, curr_edge, prev_edge);
            for (int e = 0; e < 64; e++) {
                const int r = horizontal ? e : curr_edge, c = horizontal ? curr_edge : e;
                const uint8_t pv = LOS_PREV_LOAD(horizontal ? prev + e * 64 + prev_edge : prev + prev_edge * 64 + e);
                const int idx = (r + 1) * LB_W + c + 1;
                // struct assignment overwrites both flags of the edge tile
                s.st[idx] = (uint8_t)((s.st[idx] & ~(LB_VIS | LB_BLK)) | ((pv & 1) ? LB_VIS : 0) | ((pv & 2) ? LB_BLK : 0));
                if (pv & 2)
                    los_blocked_line_b(s, mi, q.tgt_chunk_r, q.tgt_chunk_c, q.tgt_tile_r, q.tgt_tile_c,
                                       q.chunk_r, q.chunk_c, r, c);
                if (pv & 1) {
                    h[++size] = (uint16_t)idx;                // priority 0: an append, all seeds are equal
                    s.st[idx] |= LB_ASG;
                }
            }
        }
        while (size > 0) {
            npops++;
            const uint32_t cur = h[1];
            const uint32_t pidx = cur & 0x1FFFu;
            const uint16_t nprio = (uint16_t)((((cur >> 13) + 1) & 3) << 13);
            uint8_t *ctr = s.st + pidx;
            // neighbour order of field_neighbours_grid_los: (-1,0) (0,-1) (0,+1) (+1,0); the four states are read
            // before anything of this pop is written (the list is collected first, field.c:2205) -- and before the
            // sift, which touches only the heap array
            const uint32_t s0 = ctr[-LB_W], s1 = ctr[-1], s2 = ctr[1], s3 = ctr[LB_W];
            heap_remove_root13(h, size, cur >> 13);
            const uint32_t TM = LB_BLK | LB_BORDER | LB_OPEN;
            const bool v0 = (s0 & TM) == LB_OPEN, v1 = (s1 & TM) == LB_OPEN, v2 = (s2 & TM) == LB_OPEN, v3 = (s3 & TM) == LB_OPEN;
            const bool p0 = v0 && !(s0 & LB_ASG), p1 = v1 && !(s1 & LB_ASG), p2 = v2 && !(s2 & LB_ASG), p3 = v3 && !(s3 & LB_ASG);
            if (v0) ctr[-LB_W] = (uint8_t)(s0 | LB_VIS | LB_ASG);
            if (v1) ctr[-1] = (uint8_t)(s1 | LB_VIS | LB_ASG);
            if (v2) ctr[1] = (uint8_t)(s2 | LB_VIS | LB_ASG);
            if (v3) ctr[LB_W] = (uint8_t)(s3 | LB_VIS | LB_ASG);
            const uint16_t base0 = (uint16_t)(nprio | pidx);
            int sz = size;
            if (p0) h[++sz] = (uint16_t)(base0 - LB_W);
            if (p1) h[++sz] = (uint16_t)(base0 - 1);
            if (p2) h[++sz] = (uint16_t)(base0 + 1);
            if (p3) h[++sz] = (uint16_t)(base0 + LB_W);
            size = sz;
            if (!((s0 & TM) && (s1 & TM) && (s2 & TM) && (s3 & TM))) {
                // an impassable (or cost > 1) neighbour that is inside the chunk and not wavefront-blocked:
                // field_is_los_corner (field.c:435), then the blocked line
                const int r = (int)(pidx / LB_W) - 1, c = (int)(pidx % LB_W) - 1;
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const uint32_t se = e == 0 ? s0 : e == 1 ? s1 : e == 2 ? s2 : s3;
                    if (se & TM) continue;
                    const int rr = e == 0 ? r - 1 : e == 3 ? r + 1 : r, cc = e == 1 ? c - 1 : e == 2 ? c + 1 : c;
                    const uint8_t *nb = s.st + (rr + 1) * LB_W + (cc + 1);
                    bool corner = false;
                    if (rr > 0 && rr < 63) corner = ((nb[-LB_W] ^ nb[LB_W]) & LB_PASS) != 0;
                    if (!corner && cc > 0 && cc < 63) corner = ((nb[-1] ^ nb[1]) & LB_PASS) != 0;
                    if (!corner) continue;
                    los_blocked_line_b(s, mi, q.tgt_chunk_r, q.tgt_chunk_c, q.tgt_tile_r, q.tgt_tile_c,
                                       q.chunk_r, q.chunk_c, rr, cc);
                }
            }
        }
    }
    __syncwarp();
    // ---- bytes -> bit rows for the padding pass ----
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        const int row = 2 * lane + rr;
        const uint8_t *rowp = s.st + (row + 1) * LB_W + 1;
        uint64_t bb = 0, vv = 0;
#pragma unroll 8
        for (int c = 0; c < 64; c++) {
            const uint32_t v = rowp[c];
            bb |= (uint64_t)(v & LB_BLK) << c;
            vv |= (uint64_t)((v >> 3) & 1) << c;
        }
        s.blkrow[row] = bb; s.visrow[row] = vv;
    }
    __syncwarp();
    los_store_b(s, dst, lane);
    return npops;
}

// Dependency-driven scheduling shared by k_los_b and k_los_level: requests are sorted so that a request's prev_index is
// smaller than its own index; warps take indices in order from a global counter and wait (only) for the one field they
// depend on. No barrier between dependency levels: the LOS phase costs the slowest chain, not the sum over levels of the
// slowest field of each level. Returns the request index (>= n: no more work); t_take / t_ready are set on lane 0 when
// tracing.
__device__ __forceinline__ int los_take(const pfnav_los_req *__restrict__ reqs, int n, unsigned *counter, const int *done,
                                        const unsigned long long *trace, uint32_t lane, pfnav_los_req &q,
                                        unsigned long long &t_take, unsigned long long &t_ready)
{
    int i = 0;
    if (lane == 0) i = (int)atomicAdd(counter, 1u);
    i = __shfl_sync(0xffffffffu, i, 0);
    if (i >= n) return i;
    q = reqs[i];
    if (trace && lane == 0) t_take = pf_globaltimer();
    if (q.prev_index >= 0) {
        if (lane == 0) {
            const volatile int *flag = done + q.prev_index;
            while (*flag == 0) __nanosleep(100);
        }
        __syncwarp();
        __threadfence();
    }
    if (trace && lane == 0) t_ready = pf_globaltimer();
    return i;
}

// A chunk other than the destination whose shared edge with the previous chunk carries no `visible` and no
// `wavefront_blocked` tile starts with an empty frontier and draws no line (field.c:2157-2195): the field is all zero.
// Most chunks far from the goal end here. Returns true when it zero-filled the field.
__device__ __forceinline__ bool los_zero_shortcut(const pfnav_los_req &q, const uint8_t *fields, const int32_t *out_slot,
                                                  uint8_t *dst, uint32_t lane)
{
    if (q.chunk_r == q.tgt_chunk_r && q.chunk_c == q.tgt_chunk_c) return false;
    const uint8_t *prev = los_prev_field(fields, out_slot, q);
    bool horiz; int ce, pe;
    los_edge_of(q, horiz, ce, pe);
    uint32_t any = 0;
    for (int e = lane; e < 64; e += 32) any |= LOS_PREV_LOAD(horiz ? prev + e * 64 + pe : prev + pe * 64 + e);
    if (__any_sync(0xffffffffu, any != 0)) return false;
    uint4 *d4 = reinterpret_cast<uint4 *>(dst);
    for (int j = lane; j < 256; j += 32) d4[j] = make_uint4(0, 0, 0, 0);
    return true;
}

// Publish field i (its bytes are stored): the done flag its dependants wait on, and the trace record
// {taken, dependency satisfied, finished, (prev_index + 1) << 32 | word}
__device__ __forceinline__ void los_finish(int *done, unsigned long long *trace, int i, const pfnav_los_req &q, uint32_t lane,
                                           unsigned long long t_take, unsigned long long t_ready, unsigned word)
{
    __threadfence();
    __syncwarp();
    if (lane == 0) {
        *(volatile int *)(done + i) = 1;
        if (trace) {
            const unsigned long long t_done = pf_globaltimer();
            trace[4 * (size_t)i] = t_take; trace[4 * (size_t)i + 1] = t_ready; trace[4 * (size_t)i + 2] = t_done;
            trace[4 * (size_t)i + 3] = ((unsigned long long)(unsigned)(q.prev_index + 1) << 32) | word;
        }
    }
}

__global__ void __launch_bounds__(LOS_WARPS_PER_CTA * 32)
k_los_b(FlowGrids g, LosMapInfo mi, const pfnav_los_req *__restrict__ reqs, int n,
      uint8_t *fields, const int32_t *__restrict__ out_slot, unsigned *counter, int *done,
      unsigned long long *trace)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    LosSmemB &s = reinterpret_cast<LosSmemB *>(smem_raw)[warp];
    for (;;) {
        pfnav_los_req q;
        unsigned long long t_take = 0, t_ready = 0;
        const int i = los_take(reqs, n, counter, done, trace, lane, q, t_take, t_ready);
        if (i >= n) break;
        uint8_t *dst = fields + (size_t)(out_slot ? out_slot[i] : i) * 4096;
        if (los_zero_shortcut(q, fields, out_slot, dst, lane)) {
            los_finish(done, trace, i, q, lane, t_take, t_ready, 0);
            continue;
        }
        const unsigned npops = los_field_replay_b(s, g, mi, q, fields, out_slot, dst, lane);
        los_finish(done, trace, i, q, lane, t_take, t_ready, npops + 1);
    }
}

// ------------------------------------------------------------------------------------------
// Level-parallel LOS field (k_los_level)
// ------------------------------------------------------------------------------------------
// The reference's heap only ever holds priorities d and d + 1, so its pops run level by level: a breadth-first search.
// Within a level, `integration_field < INF` (ASG) and `visible` (VIS) only grow: they are unions over the level's pops,
// whatever their order. What the order can change is `wavefront_blocked` (BLK): a line drawn while the level runs can
// hide a tile from a later pop of the same level. Each line is a fixed function of its corner tile and the target, and
// the corner test reads only the static passable bits. So the level computed from the BLK of the level's start is
// exact unless a line drawn in the level covers, after its own first tile, a tile N of the level's neighbourhood that
// was not blocked at the level's start and that is (a) open and not yet visible, or (b) the first tile of another line
// of the level. That is the certificate; when it fails, the field is built again by the byte-state replay.
// FLAT bit rows, two per lane as in the other bit-row kernels: row 2 * lane (suffix 0) and 2 * lane + 1 (suffix 1).
#define LOS_INNER_COLS 0x7FFFFFFFFFFFFFFEull

// field_create_wavefront_blocked_line (field.c:463-517) into BLK (s.blkrow, every tile) and WALK (s.lv.walk, every tile
// after the first). src >= 0: a line of the edge seeding, from edge tile `src`; its tiles on the edge also record in
// s.lv.esrc the largest source that covers them.
__device__ __forceinline__ void los_level_line(LosSmemB &s, const LosMapInfo mi, const pfnav_los_req &q, int r, int c, int src,
                               bool horizontal, int curr_edge)
{
    const float tbx = (mi.map_x - (float)(q.tgt_chunk_c * 256)) - (float)(q.tgt_tile_c * 4);
    const float tbz = (mi.map_z + (float)(q.tgt_chunk_r * 256)) + (float)(q.tgt_tile_r * 4);
    const float cbx = (mi.map_x - (float)(q.chunk_c * 256)) - (float)(c * 4);
    const float cbz = (mi.map_z + (float)(q.chunk_r * 256)) + (float)(r * 4);
    const float tcx = tbx - 4.0f / 2.0f, tcz = tbz + 4.0f / 2.0f;
    const float ccx = cbx - 4.0f / 2.0f, ccz = cbz + 4.0f / 2.0f;
    float sx_ = tcx - ccx, sz_ = tcz - ccz;
    const float len = sqrtf(sx_ * sx_ + sz_ * sz_);
    sx_ = sx_ / len;
    sz_ = sz_ / len;
    if (!(len > 0.0f)) {
        // the target tile itself (see los_blocked_line): the row from the tile to column 0. Only the destination chunk
        // holds the target, and it seeds no edge, so this is never an edge-seeding line.
        or_row(&s.blkrow[r], (c == 63) ? ~0ull : ((2ull << c) - 1));
        or_row(&s.lv.walk[r], (1ull << c) - 1);
        return;
    }
    const int dx = abs((int)(sx_ * 1000));
    const int dy = -abs((int)(sz_ * 1000));
    const int sx = sx_ > 0.0f ? 1 : -1;
    const int sy = sz_ < 0.0f ? 1 : -1;
    int err = dx + dy, e2;
    int rr = r, c2 = c;
    int acc_row = rr;
    uint64_t acc = 0, wacc = 0, wmask = 0;
    do {
        if (rr != acc_row) { or_row(&s.blkrow[acc_row], acc); or_row(&s.lv.walk[acc_row], wacc); acc_row = rr; acc = 0; wacc = 0; }
        const uint64_t bit = 1ull << c2;
        acc |= bit;
        wacc |= bit & wmask;
        wmask = ~0ull;
        if (src >= 0 && (horizontal ? c2 : rr) == curr_edge) atomicMax(&s.lv.esrc[horizontal ? rr : c2], src + 1);
        e2 = 2 * err;
        if (e2 >= dy) { err += dy; c2 += sx; }
        if (e2 <= dx) { err += dx; rr += sy; }
    } while (rr >= 0 && rr < 64 && c2 >= 0 && c2 < 64);
    or_row(&s.blkrow[acc_row], acc);
    or_row(&s.lv.walk[acc_row], wacc);
}

// The level-parallel pass over one field. Returns true with s.blkrow / s.visrow holding the field's BLK and VIS rows,
// false as soon as the certificate fails. npops (when counted): the heap pops the replay would make, |ASG|.
__device__ bool los_field_level(LosSmemB &s, const FlowGrids &g, const LosMapInfo mi, const pfnav_los_req &q,
                                const uint8_t *fields, const int32_t *out_slot, uint32_t lane, bool count, unsigned &npops)
{
    const uint32_t FULL = 0xffffffffu;
    const int r0 = 2 * lane, r1 = 2 * lane + 1;
    uint64_t pass0, open0, pass1, open1;
    los_stage_row(g, q, r0, pass0, open0);
    los_stage_row(g, q, r1, pass1, open1);
    // field_is_los_corner (field.c:435): the passable bits above / below differ (rows 1..62), or those left / right do
    // (columns 1..62)
    const uint64_t pass_up = shfl_up64(pass1, lane), pass_dn = shfl_down64(pass0, lane);
    const uint64_t cor0 = (r0 > 0 ? pass_up ^ pass1 : 0ull) | (((pass0 << 1) ^ (pass0 >> 1)) & LOS_INNER_COLS);
    const uint64_t cor1 = (r1 < 63 ? pass0 ^ pass_dn : 0ull) | (((pass1 << 1) ^ (pass1 >> 1)) & LOS_INNER_COLS);
    s.blkrow[r0] = 0; s.blkrow[r1] = 0;
    s.lv.esrc[r0] = 0; s.lv.esrc[r1] = 0;
    uint64_t asg0 = 0, asg1 = 0, vis0 = 0, vis1 = 0;
    __syncwarp();
    if (q.chunk_r == q.tgt_chunk_r && q.chunk_c == q.tgt_chunk_c) {
        // the destination chunk seeds the target tile alone, with ASG only
        if (q.tgt_tile_r == r0) asg0 = 1ull << q.tgt_tile_c;
        if (q.tgt_tile_r == r1) asg1 = 1ull << q.tgt_tile_c;
    } else {
        // the edge loop of field.c:2122-2196. Its struct assignment overwrites the BLK bit that lines of EARLIER edge tiles
        // set on an edge tile, so an edge tile ends blocked iff it carries the flag itself or a line from a LATER edge tile
        // covers it; any other tile is the OR of all edge lines.
        const uint8_t *prev = los_prev_field(fields, out_slot, q);
        bool horizontal; int curr_edge, prev_edge;
        los_edge_of(q, horizontal, curr_edge, prev_edge);
        const uint32_t pva = LOS_PREV_LOAD(horizontal ? prev + lane * 64 + prev_edge : prev + prev_edge * 64 + lane);
        const uint32_t pvb = LOS_PREV_LOAD(horizontal ? prev + (lane + 32) * 64 + prev_edge : prev + prev_edge * 64 + lane + 32);
        const uint64_t seen = (uint64_t)__ballot_sync(FULL, pva & 1) | ((uint64_t)__ballot_sync(FULL, pvb & 1) << 32);
        const uint64_t flag = (uint64_t)__ballot_sync(FULL, pva & 2) | ((uint64_t)__ballot_sync(FULL, pvb & 2) << 32);
        if (pva & 2) los_level_line(s, mi, q, horizontal ? lane : curr_edge, horizontal ? curr_edge : lane, lane, horizontal, curr_edge);
        if (pvb & 2) los_level_line(s, mi, q, horizontal ? lane + 32 : curr_edge, horizontal ? curr_edge : lane + 32, lane + 32,
                                    horizontal, curr_edge);
        __syncwarp();
        const uint64_t fin = flag | (uint64_t)__ballot_sync(FULL, s.lv.esrc[lane] > (int)lane + 1) |
                             ((uint64_t)__ballot_sync(FULL, s.lv.esrc[lane + 32] > (int)lane + 33) << 32);
        if (horizontal) {
            const uint64_t eb = 1ull << curr_edge;
            s.blkrow[r0] = (s.blkrow[r0] & ~eb) | (((fin >> r0) & 1) ? eb : 0ull);
            s.blkrow[r1] = (s.blkrow[r1] & ~eb) | (((fin >> r1) & 1) ? eb : 0ull);
            asg0 = ((seen >> r0) & 1) ? eb : 0ull;
            asg1 = ((seen >> r1) & 1) ? eb : 0ull;
        } else {
            if (r0 == curr_edge) { s.blkrow[r0] = fin; asg0 = seen; }
            if (r1 == curr_edge) { s.blkrow[r1] = fin; asg1 = seen; }
        }
        vis0 = asg0; vis1 = asg1;
    }
    __syncwarp();

    uint64_t f0 = asg0, f1 = asg1;
    for (;;) {
        // N: the 4-neighbours of the frontier inside the chunk; NB: those not blocked at the level's start
        const uint64_t up = shfl_up64(f1, lane), dn = shfl_down64(f0, lane);
        const uint64_t nb0 = ((f0 << 1) | (f0 >> 1) | up | f1) & ~s.blkrow[r0];
        const uint64_t nb1 = ((f1 << 1) | (f1 >> 1) | f0 | dn) & ~s.blkrow[r1];
        const uint64_t vs0 = vis0, vs1 = vis1;
        vis0 |= nb0 & open0; vis1 |= nb1 & open1;
        f0 = nb0 & open0 & ~asg0; f1 = nb1 & open1 & ~asg1;
        asg0 |= f0; asg1 |= f1;
        // the corner neighbours, each the first tile of a line
        const uint64_t t0 = nb0 & ~open0 & cor0, t1 = nb1 & ~open1 & cor1;
        if (__any_sync(FULL, (t0 | t1) != 0)) {
            s.lv.walk[r0] = 0; s.lv.walk[r1] = 0;
            __syncwarp();
            // rounds of up to 32 lines, one per lane, taken in lane order from the warp's trigger bits
            uint64_t rest0 = t0, rest1 = t1;
            for (;;) {
                const int cnt = __popcll(rest0) + __popcll(rest1);
                int incl = cnt;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const int y = __shfl_up_sync(FULL, incl, d);
                    if ((int)lane >= d) incl += y;
                }
                const int total = __shfl_sync(FULL, incl, 31);
                if (total == 0) break;
                for (int pos = incl - cnt; pos < 32 && (rest0 | rest1); pos++) {
                    const bool lo = rest0 != 0;
                    const uint64_t w = lo ? rest0 : rest1;
                    const int c = __ffsll((long long)w) - 1;
                    s.lv.list[pos] = (uint16_t)(((lo ? r0 : r1) << 6) | c);
                    if (lo) rest0 &= rest0 - 1; else rest1 &= rest1 - 1;
                }
                __syncwarp();
                if ((int)lane < total) {
                    const int t = s.lv.list[lane];
                    los_level_line(s, mi, q, t >> 6, t & 63, -1, false, 0);
                }
                __syncwarp();
            }
#ifndef LOS_LEVEL_NO_CERTIFICATE
            const uint64_t w0 = s.lv.walk[r0], w1 = s.lv.walk[r1];
            const uint64_t bad = (w0 & nb0 & ((open0 & ~vs0) | t0)) | (w1 & nb1 & ((open1 & ~vs1) | t1));
            if (__any_sync(FULL, bad != 0)) return false;
#endif
        }
        if (!__any_sync(FULL, (f0 | f1) != 0)) break;
    }
    s.visrow[r0] = vis0; s.visrow[r1] = vis1;
    if (count) npops = __reduce_add_sync(FULL, (unsigned)(__popcll(asg0) + __popcll(asg1)));
    __syncwarp();
    return true;
}

// trace word 4, low half: 1 + heap pops, with LOS_TRACE_REPLAYED set when the certificate failed and the field was
// built by the replay
#define LOS_TRACE_REPLAYED 0x80000000u

__global__ void __launch_bounds__(LOS_WARPS_PER_CTA * 32)
k_los_level(FlowGrids g, LosMapInfo mi, const pfnav_los_req *__restrict__ reqs, int n,
            uint8_t *fields, const int32_t *__restrict__ out_slot, unsigned *counter, int *done,
            unsigned long long *trace)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    LosSmemB &s = reinterpret_cast<LosSmemB *>(smem_raw)[warp];
    for (;;) {
        pfnav_los_req q;
        unsigned long long t_take = 0, t_ready = 0;
        const int i = los_take(reqs, n, counter, done, trace, lane, q, t_take, t_ready);
        if (i >= n) break;
        uint8_t *dst = fields + (size_t)(out_slot ? out_slot[i] : i) * 4096;
        if (los_zero_shortcut(q, fields, out_slot, dst, lane)) {
            los_finish(done, trace, i, q, lane, t_take, t_ready, 0);
            continue;
        }
        unsigned npops = 0, word;
#ifdef LOS_LEVEL_ALWAYS_REPLAY
        const bool certified = false;
#else
        const bool certified = los_field_level(s, g, mi, q, fields, out_slot, lane, trace != nullptr, npops);
#endif
        if (certified) {
            los_store_b(s, dst, lane);
            word = npops + 1;
        } else {
            __syncwarp();
            npops = los_field_replay_b(s, g, mi, q, fields, out_slot, dst, lane);
            word = (npops + 1) | LOS_TRACE_REPLAYED;
        }
        los_finish(done, trace, i, q, lane, t_take, t_ready, word);
    }
}
