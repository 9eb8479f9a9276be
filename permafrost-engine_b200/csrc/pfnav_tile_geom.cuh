// pfnav_tile_geom.cuh -- the reference's tile geometry in its own float arithmetic, shared by the blocker
// rasterisation (pfnav_blockers.cu) and the entity-field footprints (pfnav_region.cu). Both include it inside
// their anonymous namespace.
//
// Restates (reference file:line):
//   M_Tile_DescForPoint2D / M_Tile_Bounds / M_Tile_AllUnderCircle      src/map/tile.c:547, 356, 687
//   C_CircleRectIntersection, C_PointInsideRect2D, C_LineCircleIntersection
//                                                                      src/phys/collision.c:997-1027, 756-768, 960-996
//   M_Tile_Contour as a bit-row dilation                               src/map/tile.c:759
#pragma once

struct td { int chunk_r, chunk_c, tile_r, tile_c; };
struct v2f { float x, z; };
struct geom { float map_x, map_z; int chunk_w, chunk_h; };
#define EPS_COLL (1.0f / 1024.0f)          // collision.c:64
#define HD __host__ __device__ __forceinline__

// The reference's float / double expressions, one rounding per operation: the device compiler must not contract
// a*b+c into an FMA (the host compiler does not: x86-64 baseline has none), so every operation is spelled out.
#ifdef __CUDA_ARCH__
HD float  f_add(float a, float b) { return __fadd_rn(a, b); }
HD float  f_sub(float a, float b) { return __fsub_rn(a, b); }
HD float  f_mul(float a, float b) { return __fmul_rn(a, b); }
HD float  f_div(float a, float b) { return __fdiv_rn(a, b); }
HD double d_add(double a, double b) { return __dadd_rn(a, b); }
HD double d_sub(double a, double b) { return __dsub_rn(a, b); }
HD double d_mul(double a, double b) { return __dmul_rn(a, b); }
HD double d_div(double a, double b) { return __ddiv_rn(a, b); }
HD double d_sqrt(double a) { return __dsqrt_rn(a); }
#else
HD float  f_add(float a, float b) { return a + b; }
HD float  f_sub(float a, float b) { return a - b; }
HD float  f_mul(float a, float b) { return a * b; }
HD float  f_div(float a, float b) { return a / b; }
HD double d_add(double a, double b) { return a + b; }
HD double d_sub(double a, double b) { return a - b; }
HD double d_mul(double a, double b) { return a * b; }
HD double d_div(double a, double b) { return a / b; }
HD double d_sqrt(double a) { return sqrt(a); }
#endif
HD double d_sq(float a) { return d_mul((double)a, (double)a); }     // pow(a, 2)
HD float  f_dot(v2f a, v2f b) { return f_add(f_mul(a.x, b.x), f_mul(a.z, b.z)); }

HD bool point_inside_rect(v2f p, v2f a, v2f b, v2f d)
{
    const v2f ap = {f_sub(p.x, a.x), f_sub(p.z, a.z)}, ab = {f_sub(b.x, a.x), f_sub(b.z, a.z)}, ad = {f_sub(d.x, a.x), f_sub(d.z, a.z)};
    const float ap_ab = f_dot(ap, ab), ap_ad = f_dot(ap, ad);
    return (ap_ab >= 0.0f && ap_ab <= f_dot(ab, ab)) && (ap_ad >= 0.0f && ap_ad <= f_dot(ad, ad));
}

HD bool line_circle(float ax, float az, float bx, float bz, v2f c, float radius)
{
    const float dx = f_sub(bx, ax), dz = f_sub(bz, az);
    const float A = (float)d_add(d_sq(dx), d_sq(dz));
    const float B = f_mul(2.0f, f_add(f_mul(dx, f_sub(ax, c.x)), f_mul(dz, f_sub(az, c.z))));
    const float C = (float)d_sub(d_add(d_sq(f_sub(ax, c.x)), d_sq(f_sub(az, c.z))), d_sq(radius));
    const float det = (float)d_sub(d_sq(B), (double)f_mul(f_mul(4.0f, A), C));
    float t;
    if (det < 0.0f || A < EPS_COLL) return false;
    else if (det == 0.0f) t = f_div(-B, f_mul(2.0f, A));
    else {
        const double root = d_sqrt((double)det), two_a = (double)f_mul(2.0f, A);
        const float t1 = (float)d_div(d_add((double)(-B), root), two_a), t2 = (float)d_div(d_sub((double)(-B), root), two_a);
        t = t1 < t2 ? t1 : t2;
    }
    if (t < 0.0f || t > 1.0f) return false;
    return true;
}

// C_CircleRectIntersection (collision.c:997); rect = {x, z, width, height}, x decreasing with the column
HD bool circle_rect(v2f center, float radius, float rx, float rz, float w, float h)
{
    const v2f corners[4] = {{f_sub(rx, w), rz}, {rx, rz}, {rx, f_add(rz, h)}, {f_sub(rx, w), f_add(rz, h)}};
    if (point_inside_rect(center, corners[0], corners[1], corners[3])) return true;
    for (int i = 0; i < 4; i++) {
        const float ddx = f_sub(corners[i].x, center.x), ddz = f_sub(corners[i].z, center.z);
        if ((float)d_sqrt((double)f_add(f_mul(ddx, ddx), f_mul(ddz, ddz))) <= radius) return true;
    }
    for (int i = 0; i < 4; i++) {
        const v2f a = corners[i], b = corners[(i + 1) & 3];
        if (line_circle(a.x, a.z, b.x, b.z, center, radius)) return true;
    }
    return false;
}

HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// M_Tile_DescForPoint2D with the nav resolution (tile.c:547)
HD bool desc_for_point(const geom &g, float px, float pz, td *out)
{
    const float width = (float)(g.chunk_w * 256), height = (float)(g.chunk_h * 256);
    if (px > g.map_x || px < f_sub(g.map_x, width)) return false;
    if (pz < g.map_z || pz > f_add(g.map_z, height)) return false;
    int chunk_r = (int)(fabsf(f_sub(g.map_z, pz)) / 256.0f), chunk_c = (int)(fabsf(f_sub(g.map_x, px)) / 256.0f);
    chunk_r = clampi(chunk_r, 0, g.chunk_h - 1);
    chunk_c = clampi(chunk_c, 0, g.chunk_w - 1);
    const float bx = f_sub(g.map_x, chunk_c * 256.0f), bz = f_add(g.map_z, chunk_r * 256.0f);
    const int tile_r = (int)(fabsf(f_sub(bz, pz)) / 4.0f), tile_c = (int)(fabsf(f_sub(bx, px)) / 4.0f);
    out->chunk_r = chunk_r; out->chunk_c = chunk_c;
    out->tile_r = clampi(tile_r, 0, 63); out->tile_c = clampi(tile_c, 0, 63);
    return true;
}

// M_Tile_Bounds (tile.c:356) of the nav tile (ar, ac) + the circle test of M_Tile_AllUnderCircle (tile.c:687)
HD bool tile_under_circle(const geom &g, int ar, int ac, v2f c, float radius)
{
    const float bx = f_sub(f_sub(g.map_x, (float)((ac / 64) * 256)), (float)((ac % 64) * 4));
    const float bz = f_add(f_add(g.map_z, (float)((ar / 64) * 256)), (float)((ar % 64) * 4));
    return circle_rect(c, radius, bx, bz, 4.0f, 4.0f);
}

#ifdef __CUDACC__
// A circle and the rings around it as 32 x 32 bit rows, one warp per circle: lane = window row, bit = window column.
// The window's origin (r0, c0) puts the circle's centre tile at row / column nt + 3, which leaves room for three
// rings as long as 2 * nt + 7 <= 32 (nt = ceil(radius / 4)).
#define CIRCLE_MAX_NT 12

// M_Tile_AllUnderCircle (tile.c:687) into rows[0..31] (shared, zeroed by the caller; the warp synchronises). Tiles
// outside the map stay clear.
__device__ __forceinline__ void circle_rows(const geom &g, int H64, int W64, v2f c, float radius, int nt, int r0, int c0,
                                            unsigned *rows, int lane)
{
    const int side = 2 * nt + 1;
    for (int i = lane; i < side * side; i += 32) {
        const int dr = i / side, dc = i - dr * side;
        const int ar = r0 + 3 + dr, ac = c0 + 3 + dc;
        if (ar < 0 || ar >= H64 || ac < 0 || ac >= W64) continue;
        if (tile_under_circle(g, ar, ac, c, radius)) atomicOr(&rows[dr + 3], 1u << (dc + 3));
    }
    __syncwarp();
}

// the window's in-map columns of this lane's row (win = the window rows / columns in use)
__device__ __forceinline__ unsigned window_inmap(int H64, int W64, int r0, int c0, int win, int lane)
{
    const int lo = max(0, -c0), hi = min(win, W64 - c0);
    const unsigned colmask = hi > lo ? (((hi >= 32) ? 0xFFFFFFFFu : ((1u << hi) - 1u)) & ~((1u << lo) - 1u)) : 0u;
    const int myr = r0 + lane;
    return (lane < win && myr >= 0 && myr < H64) ? colmask : 0u;
}

// M_Tile_Contour (tile.c:759) of the bit rows m: the in-map tiles 8-adjacent to the set and not in it
__device__ __forceinline__ unsigned contour_rows(unsigned m, unsigned inmap, int lane)
{
    const unsigned h = m | (m << 1) | (m >> 1);
    unsigned up = __shfl_up_sync(0xFFFFFFFFu, h, 1), dn = __shfl_down_sync(0xFFFFFFFFu, h, 1);
    if (lane == 0) up = 0;
    if (lane == 31) dn = 0;
    return (h | up | dn) & ~m & inmap;
}
#endif
