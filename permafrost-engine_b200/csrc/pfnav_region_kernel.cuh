// pfnav_region_kernel.cuh -- the device code of k_region_fields (region / zone / entity fields), kept in a header of
// its own so that tests/emu can run the SAME source on CPU threads (tests/emu/region_emu.cpp defines the CUDA
// keywords it uses as plain C++ and a barrier); pfnav_region.cu includes it inside its anonymous namespace.
// Needs: <stdint.h>, pfnav_region_req and the PFNAV_REGION_* flags (include/pfnav.h), min().
#pragma once

enum : uint8_t {
    RG_EXISTS = 1,     // inside the map (M_Tile_RelativeDesc, tile.c:391)
    RG_PASSP  = 2,     // field_tile_passable (field.c:117)
    RG_PASSM  = 4,     // passable under the request's enemy mask (field_tile_passable_no_enemies, field.c:179)
    RG_OVL    = 8,     // nav_cell_overlay::blocked
    RG_ENT    = 16,    // may be entered by the current integration pass
    RG_COMP   = 32,    // part of the blocked island flooded from `start`
    RG_SEED   = 64,    // zero-cost source of the current integration pass
    RG_INCL   = 128    // inside the map-clamped region of the fix-up flood
};

#define RG_INF 0xFFFFFFFFu
#ifndef RG_THREADS
#define RG_THREADS 256
#endif

struct RegionGrids {
    const uint8_t *cost; const uint16_t *blk; const uint16_t *fmask;   // [layer][H64][W64]
    int W64, H64;
};

struct RegionSmem {
    uint32_t *dist; uint8_t *cst; uint8_t *flg; int dim, N;
};

__device__ __forceinline__ void region_gather(const RegionGrids &g, const RegionSmem &s, int layer, int base_r, int base_c,
                                              uint16_t enemies, const int32_t *ov, int nov)
{
    const size_t lbase = (size_t)layer * g.W64 * g.H64;
    for (int i = threadIdx.x; i < s.N; i += RG_THREADS) {
        const int r = i / s.dim, c = i - r * s.dim;
        const int ar = base_r + r, ac = base_c + c;
        uint8_t f = 0, cv = 0;
        if (ar >= 0 && ar < g.H64 && ac >= 0 && ac < g.W64) {
            const size_t off = lbase + (size_t)ar * g.W64 + ac;
            cv = g.cost[off];
            const uint16_t b = g.blk[off];
            f = RG_EXISTS;
            if (cv != 0xFF) {
                if (b == 0) f |= RG_PASSP | RG_PASSM;
                else if (enemies != 0 && (g.fmask[off] & ~enemies) == 0) f |= RG_PASSM;
            }
        }
        s.cst[i] = cv; s.flg[i] = f;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < nov; k += RG_THREADS) {        // build_overlay_mask (field.c:571)
        const int dr = ov[2 * k] - base_r, dc = ov[2 * k + 1] - base_c;
        if (dr >= 0 && dr < s.dim && dc >= 0 && dc < s.dim) s.flg[dr * s.dim + dc] |= RG_OVL;
    }
    __syncthreads();
}

// relaxation to the shortest-distance fixed point over the RG_ENT cells (sources: dist == 0 on entry)
__device__ __forceinline__ void region_relax(const RegionSmem &s)
{
    const int dim = s.dim, N = s.N;
    // a thread owns `per` consecutive cells; per is made odd so that the lanes of a warp, which walk their runs in
    // lock step, hit 32 different shared-memory banks (an even run length of 36 or 64 words is a 4- / 32-way conflict)
    const int per = ((N + RG_THREADS - 1) / RG_THREADS) | 1;
    const int lo = min((int)threadIdx.x * per, N), hi = min(lo + per, N);
    // (row, column) of the run's first and last cell; the sweeps step them instead of dividing per cell
    const int r_lo = lo / dim, c_lo = lo - r_lo * dim;
    const int last = hi > lo ? hi - 1 : lo, r_hi = last / dim, c_hi = last - r_hi * dim;
    bool fwd = true;
    while (true) {
        bool changed = false;
        int i = fwd ? lo : hi - 1, r = fwd ? r_lo : r_hi, c = fwd ? c_lo : c_hi;
        for (int k = 0; k < hi - lo; k++) {
            if (s.flg[i] & RG_ENT) {
                uint32_t m = RG_INF;
                if (r > 0) m = min(m, s.dist[i - dim]);
                if (r < dim - 1) m = min(m, s.dist[i + dim]);
                if (c > 0) m = min(m, s.dist[i - 1]);
                if (c < dim - 1) m = min(m, s.dist[i + 1]);
                if (m != RG_INF) {
                    const uint32_t nd = m + s.cst[i];
                    if (nd < s.dist[i]) { s.dist[i] = nd; changed = true; }
                }
            }
            if (fwd) { i++; if (++c == dim) { c = 0; r++; } }
            else     { i--; if (--c < 0) { c = dim - 1; r--; } }
        }
        fwd = !fwd;
        if (!__syncthreads_or(changed)) break;
    }
}

// field_flow_dir (field.c:355) over the integer integration values; note the last test's `c < rdim - 1`
__device__ __forceinline__ uint32_t region_flow_dir(const uint32_t *f, int n, int r, int c)
{
    const int i = r * n + c;
    const bool up = r > 0, dn = r < n - 1, lf = c > 0, rt = c < n - 1;
    const uint32_t N_ = up ? f[i - n] : RG_INF, S_ = dn ? f[i + n] : RG_INF;
    const uint32_t W_ = lf ? f[i - 1] : RG_INF, E_ = rt ? f[i + 1] : RG_INF;
    uint32_t mc = min(min(N_, S_), min(W_, E_));
    const uint32_t NW = (up && lf) ? f[i - n - 1] : RG_INF, NE = (up && rt) ? f[i - n + 1] : RG_INF;
    const uint32_t SW = (dn && lf) ? f[i + n - 1] : RG_INF, SE = (dn && rt) ? f[i + n + 1] : RG_INF;
    if (up && lf && N_ != RG_INF && W_ != RG_INF) mc = min(mc, NW);
    if (up && rt && N_ != RG_INF && E_ != RG_INF) mc = min(mc, NE);
    if (dn && lf && S_ != RG_INF && W_ != RG_INF) mc = min(mc, SW);
    if (dn && rt && S_ != RG_INF && E_ != RG_INF) mc = min(mc, SE);
    // enum flow_dir: FD_NONE 0, NW 1, N 2, NE 3, W 4, E 5, SW 6, S 7, SE 8
    if (up && N_ == mc) return 2;
    if (dn && S_ == mc) return 7;
    if (rt && E_ == mc) return 5;
    if (lf && W_ == mc) return 4;
    if (up && lf && NW == mc) return 1;
    if (up && rt && NE == mc) return 3;
    if (dn && lf && SW == mc) return 6;
    if (dn && rt && SE == mc) return 8;
    return 0;
}

__global__ void __launch_bounds__(RG_THREADS, 4) k_region_fields(RegionGrids g, int dim, const pfnav_region_req *__restrict__ reqs,
                                                              int n, const int32_t *__restrict__ seeds,
                                                              const int32_t *__restrict__ overlay, uint8_t *__restrict__ fields,
                                                              int chunk_out, const uint32_t *__restrict__ seed_bits = nullptr,
                                                              const int32_t *__restrict__ out_slot = nullptr)
{
    extern __shared__ uint32_t rg_smem[];
    RegionSmem s;
    s.dim = dim; s.N = dim * dim;
    s.dist = rg_smem; s.cst = reinterpret_cast<uint8_t *>(s.dist + s.N); s.flg = s.cst + s.N;
    const int N = s.N, half = dim / 2, tid = threadIdx.x;

    for (int q = blockIdx.x; q < n; q += gridDim.x) {
        const pfnav_region_req rq = reqs[q];
        // out_slot: field q goes to its pool slot instead of position q
        uint8_t *out = fields + (size_t)(out_slot ? out_slot[q] : q) * (chunk_out ? 4096 : N / 2);
        const int32_t *ov = overlay + 2 * (size_t)rq.overlay_off;
        __syncthreads();

        if (chunk_out) {
            // TARGET_ZONE chunk field (field_update_zone, field.c:1810): the chunk (center_r, center_c) padded by
            // half a chunk; field_build_flow_region (field.c:762) writes the chunk's 64 x 64 window of an
            // initialised (all FD_NONE) field, one direction per byte
            const int roff = (rq.center_r > 0 && dim > 64) ? 32 : 0, coff = (rq.center_c > 0 && dim > 64) ? 32 : 0;
            const int base_r = rq.center_r * 64 - roff, base_c = rq.center_c * 64 - coff;
            const int32_t *sd = seeds + 2 * (size_t)rq.seed_off;
            region_gather(g, s, rq.layer, base_r, base_c, 0, ov, 0);
            // seed_bits: the frontier as dim x dim bits (row-major, N / 32 words per field) instead of a tile list
            const uint32_t *bits = seed_bits ? seed_bits + (size_t)q * (N / 32) : nullptr;
            for (int i = tid; i < N; i += RG_THREADS) {
                const uint8_t f = s.flg[i];
                s.dist[i] = (bits && ((bits[i >> 5] >> (i & 31)) & 1u)) ? 0u : RG_INF;
                if ((f & (RG_EXISTS | RG_PASSP)) == (RG_EXISTS | RG_PASSP)) s.flg[i] = f | RG_ENT;
            }
            __syncthreads();
            for (int k = tid; k < rq.seed_n; k += RG_THREADS) {
                const int dr = sd[2 * k] - base_r, dc = sd[2 * k + 1] - base_c;
                if (dr >= 0 && dr < dim && dc >= 0 && dc < dim) s.dist[dr * dim + dc] = 0;
            }
            __syncthreads();
            region_relax(s);
            for (int t = tid; t < 4096; t += RG_THREADS) {
                const int r = (t >> 6) + roff, c = (t & 63) + coff;
                const uint32_t d = s.dist[r * dim + c];
                out[t] = (d != RG_INF && d != 0) ? (uint8_t)region_flow_dir(s.dist, dim, r, c) : (uint8_t)0;
            }
            continue;
        }

        if (rq.flags & PFNAV_REGION_CREATE) {
            int base_r = rq.center_r - half, base_c = rq.center_c - half;
            const int32_t *sd = seeds + 2 * (size_t)rq.seed_off;
            if (rq.flags & PFNAV_REGION_CELL) {              // field.c:2477-2482
                if (sd[0] - base_r >= dim) base_r = sd[0] - (dim - 1);
                if (sd[1] - base_c >= dim) base_c = sd[1] - (dim - 1);
            }
            region_gather(g, s, rq.layer, base_r, base_c, rq.enemies, ov, rq.overlay_n);
            for (int i = tid; i < N; i += RG_THREADS) {
                const uint8_t f = s.flg[i];
                s.dist[i] = RG_INF;
                if ((f & (RG_EXISTS | RG_PASSM | RG_OVL)) == (RG_EXISTS | RG_PASSM)) s.flg[i] = f | RG_ENT;
            }
            __syncthreads();
            for (int k = tid; k < rq.seed_n; k += RG_THREADS) {
                const int dr = sd[2 * k] - base_r, dc = sd[2 * k + 1] - base_c;
                if (dr >= 0 && dr < dim && dc >= 0 && dc < dim) s.dist[dr * dim + dc] = 0;
            }
            __syncthreads();
            region_relax(s);
            // field_build_flow_unaligned (field.c:804): unreached cells keep the memset's 0 == FD_NONE
            for (int b = tid; b < N / 2; b += RG_THREADS) {
                const int r = b / half, c = (b - r * half) * 2;
                uint32_t hi = 0, lo = 0;
                const uint32_t d0 = s.dist[r * dim + c], d1 = s.dist[r * dim + c + 1];
                if (d0 != RG_INF && d0 != 0) hi = region_flow_dir(s.dist, dim, r, c);
                if (d1 != RG_INF && d1 != 0) lo = region_flow_dir(s.dist, dim, r, c + 1);
                out[b] = (uint8_t)((hi << 4) | lo);
            }
            __syncthreads();
        }

        if (rq.flags & PFNAV_REGION_FIXUP) {
            // the fix-up's own base: the create call's target shift is not repeated (field.c:2650-2657)
            const int base_r = rq.center_r - half, base_c = rq.center_c - half;
            // clamped_region (field.c:1892): extents are end - base
            const int cb_r = base_r >= 0 ? base_r : 0, cb_c = base_c >= 0 ? base_c : 0;
            const int ce_r = rq.center_r + half < g.H64 ? rq.center_r + half : g.H64 - 1;
            const int ce_c = rq.center_c + half < g.W64 ? rq.center_c + half : g.W64 - 1;
            const int reg_r = ce_r - cb_r, reg_c = ce_c - cb_c;
            const int wr0 = cb_r - base_r, wc0 = cb_c - base_c;      // the clamped window inside the dim x dim cells
            const int sr = rq.start_r - base_r, sc = rq.start_c - base_c;
            const bool start_ok = sr >= wr0 && sr < wr0 + reg_r && sc >= wc0 && sc < wc0 + reg_c;
            region_gather(g, s, rq.layer, base_r, base_c, rq.enemies, ov, rq.overlay_n);
            for (int i = tid; i < N; i += RG_THREADS) {
                const int r = i / dim, c = i - r * dim;
                uint8_t f = s.flg[i];
                if (r >= wr0 && r < wr0 + reg_r && c >= wc0 && c < wc0 + reg_c && (f & RG_EXISTS)) f |= RG_INCL;
                s.flg[i] = f;
            }
            __syncthreads();
            if (start_ok) {
                if (reg_r >= reg_c) {
                    // field_passable_frontier (field.c:1441) as a reachability fixed point
                    if (tid == 0) s.flg[sr * dim + sc] |= (s.flg[sr * dim + sc] & RG_PASSP) ? RG_SEED : RG_COMP;
                    __syncthreads();
                    const int per = ((N + RG_THREADS - 1) / RG_THREADS) | 1;
                    const int lo = min(tid * per, N), hi = min(lo + per, N);
                    bool fwd = true;
                    while (true) {
                        bool changed = false;
                        for (int k = 0; k < hi - lo; k++) {
                            const int i = fwd ? lo + k : hi - 1 - k;
                            const uint8_t f = s.flg[i];
                            if ((f & (RG_INCL | RG_PASSP | RG_COMP)) != RG_INCL) continue;
                            const int r = i / dim, c = i - r * dim;
                            uint8_t nb = 0;
                            if (r > 0) nb |= s.flg[i - dim];
                            if (r < dim - 1) nb |= s.flg[i + dim];
                            if (c > 0) nb |= s.flg[i - 1];
                            if (c < dim - 1) nb |= s.flg[i + 1];
                            if (nb & RG_COMP) { s.flg[i] = f | RG_COMP; changed = true; }
                        }
                        fwd = !fwd;
                        if (!__syncthreads_or(changed)) break;
                    }
                    for (int i = tid; i < N; i += RG_THREADS) {
                        const uint8_t f = s.flg[i];
                        if ((f & (RG_INCL | RG_PASSP)) != (RG_INCL | RG_PASSP)) continue;
                        const int r = i / dim, c = i - r * dim;
                        uint8_t nb = 0;
                        if (r > 0) nb |= s.flg[i - dim];
                        if (r < dim - 1) nb |= s.flg[i + dim];
                        if (c > 0) nb |= s.flg[i - 1];
                        if (c < dim - 1) nb |= s.flg[i + 1];
                        if (nb & RG_COMP) s.flg[i] = f | RG_SEED;
                    }
                    __syncthreads();
                } else {
                    // rows < columns: visited_idx (field.c:1431) aliases; replay the breadth-first order literally
                    uint8_t *visited = reinterpret_cast<uint8_t *>(s.dist);
                    uint16_t *queue = reinterpret_cast<uint16_t *>(visited + N);
                    for (int i = tid; i < N; i += RG_THREADS) visited[i] = 0;
                    __syncthreads();
                    if (tid == 0) {
                        int head = 0, tail = 0;
                        queue[tail++] = (uint16_t)(sr * dim + sc);
                        visited[(sr - wr0) * reg_r + (sc - wc0)] = 1;
                        while (head < tail) {
                            const int i = queue[head++];
                            const uint8_t f = s.flg[i];
                            if (f & RG_PASSP) { s.flg[i] = f | RG_SEED; continue; }
                            const int r = i / dim, c = i - r * dim;
                            const int nr[4] = {r, r, r - 1, r + 1}, nc[4] = {c - 1, c + 1, c, c};   // field.c:1492-1497
#pragma unroll
                            for (int e = 0; e < 4; e++) {
                                if (nr[e] < wr0 || nr[e] >= wr0 + reg_r || nc[e] < wc0 || nc[e] >= wc0 + reg_c) continue;
                                const int j = nr[e] * dim + nc[e];
                                if (!(s.flg[j] & RG_EXISTS)) continue;
                                const int v = (nr[e] - wr0) * reg_r + (nc[e] - wc0);
                                if (visited[v]) continue;
                                visited[v] = 1;
                                queue[tail++] = (uint16_t)j;
                            }
                        }
                    }
                    __syncthreads();
                }
                // field_build_integration_nonpass_region (field.c:678): only non-passable or overlay-blocked tiles
                for (int i = tid; i < N; i += RG_THREADS) {
                    const uint8_t f = s.flg[i];
                    s.dist[i] = (f & RG_SEED) ? 0u : RG_INF;
                    const bool ent = (f & RG_EXISTS) && !((f & RG_PASSP) && !(f & RG_OVL));
                    s.flg[i] = ent ? (f | RG_ENT) : (f & ~RG_ENT);
                }
                __syncthreads();
                region_relax(s);
                for (int b = tid; b < N / 2; b += RG_THREADS) {
                    const int r = b / half, c = (b - r * half) * 2;
                    const uint32_t d0 = s.dist[r * dim + c], d1 = s.dist[r * dim + c + 1];
                    const bool u0 = d0 != RG_INF && d0 != 0 && (s.flg[r * dim + c] & RG_EXISTS);
                    const bool u1 = d1 != RG_INF && d1 != 0 && (s.flg[r * dim + c + 1] & RG_EXISTS);
                    if (!(u0 || u1)) continue;
                    uint32_t v = out[b];
                    if (u0) v = (v & 0x0Fu) | (region_flow_dir(s.dist, dim, r, c) << 4);
                    if (u1) v = (v & 0xF0u) | region_flow_dir(s.dist, dim, r, c + 1);
                    out[b] = (uint8_t)v;
                }
            }
        }
    }
}

