// pfnav_clearpath_kernel.cuh -- the device code of ClearPath (G_ClearPath_NewVelocity, clearpath.c:694): velocity
// obstacles, the warp-cooperative solve, the one-pass emulation of the drop-furthest retry loop with its literal replay,
// and the two-phase split (phase A collects admissible intersections, phase B chooses). Kept in a header of its own so
// that tests/emu can run the SAME source on CPU threads (tests/emu/clearpath_emu.cpp defines the CUDA keywords and warp
// intrinsics it uses as plain C++); pfnav_agents.cu includes it. Also the v2 helpers the rest of the velocity update shares.
// Needs: <stdint.h>, <math.h>, pfnav.h and the warp intrinsics.
#pragma once

#define EPS_F (1.0f / 1024)
#define FULL 0xffffffffu

// ------------------------------------------------------------------------------------------
// vec2 helpers (pf_math.c:58-94) -- float storage, sqrt evaluated in double then rounded, which
// is the correctly rounded float sqrt.
// ------------------------------------------------------------------------------------------
struct v2 { float x, z; };
__device__ __forceinline__ v2 v2_add(v2 a, v2 b) { return {a.x + b.x, a.z + b.z}; }
__device__ __forceinline__ v2 v2_sub(v2 a, v2 b) { return {a.x - b.x, a.z - b.z}; }
__device__ __forceinline__ v2 v2_scale(v2 a, float s) { return {a.x * s, a.z * s}; }
__device__ __forceinline__ float v2_dot(v2 a, v2 b) { return a.x * b.x + a.z * b.z; }
__device__ __forceinline__ float v2_len(v2 a) { return sqrtf(a.x * a.x + a.z * a.z); }
__device__ __forceinline__ v2 v2_normal(v2 a) { float l = v2_len(a); return {a.x / l, a.z / l}; }
// vec2_truncate (movement.c:643)
__device__ __forceinline__ v2 v2_truncate(v2 a, float max_len)
{
    if (v2_len(a) > max_len) { a = v2_normal(a); a = v2_scale(a, max_len); }
    return a;
}

// ------------------------------------------------------------------------------------------
// ClearPath pieces
// ------------------------------------------------------------------------------------------
struct ray { v2 point, dir; };
struct cp_ent { v2 pos, vel; float radius; };

#define QNAN __int_as_float(0x7fc00000)

// slope used by C_InfiniteLineIntersection (collision.c:822): NaN marks a (near-)vertical line
__device__ __forceinline__ float line_slope(v2 dir) { return fabsf(dir.x) < EPS_F ? QNAN : (dir.z / dir.x); }

// C_InfiniteLineIntersection (collision.c:820) incl. the preserved "l2 vertical" y bug (:839-840),
// with the two slopes supplied by the caller
__device__ __forceinline__ bool line_isect_s(const v2 p1, const float s1, const v2 p2, const float s2, v2 &out)
{
    const bool n1 = isnan(s1), n2 = isnan(s2);
    if (n1 && n2) return false;
    if (fabsf(s1 - s2) < EPS_F) return false;
    if (n1 && !n2) {
        out.x = p1.x;
        out.z = (p1.x - p2.x) * s2 + p2.z;
    } else if (!n1 && n2) {
        out.x = p2.x;
        out.z = (p2.x - p1.x) * s1 + p2.z;
    } else {
        out.x = (s1 * p1.x - s2 * p2.x + p2.z - p1.z) / (s1 - s2);
        out.z = s2 * (out.x - p2.x) + p2.z;
    }
    return true;
}
__device__ __forceinline__ bool line_isect(const ray l1, const ray l2, v2 &out)
{
    return line_isect_s(l1.point, line_slope(l1.dir), l2.point, line_slope(l2.dir), out);
}

// (a / b < 0.0f) for |b| <= 1 without the division: the quotient of a non-zero a by such a b never
// underflows to zero, so only the signs (and NaNs, and b == +-0) matter. Bit-equivalent to the
// reference's four tests in C_RayRayIntersection2D (collision.c:861-871).
__device__ __forceinline__ bool quot_lt0(float a, float b)
{
    const bool bneg = signbit(b), bnum = (b == b);
    return bnum && ((a < 0.0f && !bneg) || (a > 0.0f && bneg));
}

// compute_vo_edges (clearpath.c:130)
__device__ __forceinline__ void vo_edges(const cp_ent ent, const cp_ent nb, v2 &right, v2 &left)
{
    v2 e2n = v2_normal(v2_sub(nb.pos, ent.pos));
    v2 r = {-e2n.z, e2n.x};
    r = v2_scale(r, nb.radius + ent.radius + 0.0f);
    const v2 rt = v2_add(nb.pos, r), lt = v2_sub(nb.pos, r);
    right = v2_normal(v2_sub(rt, ent.pos));
    left = v2_normal(v2_sub(lt, ent.pos));
}

#define CQ_CAP 160
struct VelSmem {
    cp_ent dyn[PFNAV_MAX_NEIGHBOURS];
    cp_ent stat[PFNAV_MAX_NEIGHBOURS];
    // rays, SoA (2 per velocity obstacle: even = left side, odd = right side)
    float rpx[4 * PFNAV_MAX_NEIGHBOURS], rpz[4 * PFNAV_MAX_NEIGHBOURS];
    float rdx[4 * PFNAV_MAX_NEIGHBOURS], rdz[4 * PFNAV_MAX_NEIGHBOURS];
    float rsl[4 * PFNAV_MAX_NEIGHBOURS];
    uint32_t near_id[128];
    float2 term[128];
    float cqx[CQ_CAP], cqz[CQ_CAP];      // candidate points awaiting the inside-PCR test
    int cqk[CQ_CAP];                      // their sequence index in the reference's push order
    // ---- one-pass emulation of the drop-furthest retry loop (clearpath_retry) ----
    uint8_t vo_src[64];                   // obstacle -> neighbour slot it was built from (dyn: 0..31, stat: 32..63)
    uint8_t nb_rank[64];                  // neighbour slot -> removal time 1.. (255: still there when the loop ends)
    uint8_t vo_rank[64];                  // obstacle -> removal time of its neighbour
    uint8_t vo_ord[64];                   // obstacles by decreasing removal time
    uint8_t cur[64];                      // working lists: dyn slots at [0, nd), stat slots at [32, 32 + ns)
    float   ndist[64];                    // neighbour slot -> distance from the entity
    uint8_t cqd[CQ_CAP];                  // death time of the queued candidates
};

// One velocity obstacle of inside_pcr (clearpath.c:252-287): is `test` strictly inside VO `i`?
// The reference normalises (test - apex) and compares a 2-D cross product with +-1/1024. Away from
// those thresholds the unnormalised cross product decides with certainty (margins of 1 % on the
// threshold versus ~1e-6 relative float error), so the sqrt and the two IEEE divisions are only paid
// in the thin band around a threshold, where the reference's exact sequence is replayed.
__device__ __forceinline__ bool vo_contains(const VelSmem &s, int i, v2 test)
{
    const float E_LO2 = (EPS_F * 0.99f) * (EPS_F * 0.99f), E_HI2 = (EPS_F * 1.01f) * (EPS_F * 1.01f);
    {   // left side: "left_of_vo" <=> det < EPS  -> not inside
        const int k = 2 * i;
        const v2 ptt = {test.x - s.rpx[k], test.z - s.rpz[k]};
        const float len2 = ptt.x * ptt.x + ptt.z * ptt.z;
        const float u = (ptt.z * s.rdx[k]) - (ptt.x * s.rdz[k]);
        const float u2 = u * u;
        bool decided = false, skip = false;
        if (len2 > E_HI2 && len2 < 1e30f) {             // |ptt| certainly >= EPS
            if (u <= 0.0f || u2 < E_LO2 * len2) { decided = true; skip = true; }        // det < EPS
            else if (u2 > E_HI2 * len2) { decided = true; skip = false; }               // det >= EPS
        }
        if (!decided) {
            const float len = sqrtf(len2);
            if (len < EPS_F) skip = true;
            else {
                const v2 n = {ptt.x / len, ptt.z / len};
                const float det = (n.z * s.rdx[k]) - (n.x * s.rdz[k]);
                skip = det < EPS_F;
            }
        }
        if (skip) return false;
    }
    {   // right side: "right_of_vo" <=> det > -EPS -> not inside
        const int k = 2 * i + 1;
        const v2 ptt = {test.x - s.rpx[k], test.z - s.rpz[k]};
        const float len2 = ptt.x * ptt.x + ptt.z * ptt.z;
        const float u = (ptt.z * s.rdx[k]) - (ptt.x * s.rdz[k]);
        const float u2 = u * u;
        bool decided = false, skip = false;
        if (len2 > E_HI2 && len2 < 1e30f) {
            if (u >= 0.0f || u2 < E_LO2 * len2) { decided = true; skip = true; }        // det > -EPS
            else if (u2 > E_HI2 * len2) { decided = true; skip = false; }               // det <= -EPS
        }
        if (!decided) {
            const float len = sqrtf(len2);
            if (len < EPS_F) skip = true;
            else {
                const v2 n = {ptt.x / len, ptt.z / len};
                const float det = (n.z * s.rdx[k]) - (n.x * s.rdz[k]);
                skip = det > -EPS_F;
            }
        }
        if (skip) return false;
    }
    return true;
}

// Drain the candidate queue: every lane keeps one candidate in flight and tests one velocity obstacle
// per iteration; a lane whose candidate is decided immediately takes the next one, so all lanes stay
// busy whatever the early-exit pattern of inside_pcr is. Keeps the per-lane first-minimum of
// compute_vnew (clearpath.c:368) on (distance, sequence index).
// The candidate a lane has in flight survives between two drains of the same solve (DrainLane): a drain that is not the
// last one of its solve returns as soon as the queue is empty and leaves the long-running candidates (the ones that pass
// obstacle after obstacle) in their lanes, where the next batch of candidates fills the idle lanes around them; only the
// final drain (`flush`) waits for the stragglers.
struct DrainLane { int busy = 0, vo = 0, myk = 0, vstart = 0; v2 myp = {0.0f, 0.0f}; };
// vstart: obstacle that swallowed this lane's previous candidate: tested first (any order is exact)

__device__ __forceinline__ void drain_candidates(const VelSmem &s, int qn, int nvo, const v2 ent_pos, const v2 des_v,
                                                 uint32_t lane, float &best, int &best_idx, v2 &best_p, int &any,
                                                 DrainLane &dl, bool flush)
{
    int next = 0;
    while (true) {
        const bool need = !dl.busy;
        const uint32_t mneed = __ballot_sync(FULL, need);
        const int avail = qn - next;
        if (need && avail > 0) {
            const int rank = __popc(mneed & ((1u << lane) - 1));
            if (rank < avail) { const int my = next + rank; dl.busy = 1; dl.vo = 0; dl.myp = {s.cqx[my], s.cqz[my]}; dl.myk = s.cqk[my]; }
        }
        next += min(__popc(mneed), avail);
        if (!flush && next >= qn) break;
        if (!__any_sync(FULL, dl.busy)) break;
        if (dl.busy) {
            bool finished = false, inside = false;
            int vidx = dl.vo + dl.vstart;
            if (vidx >= nvo) vidx -= nvo;
            if (dl.vo < nvo) inside = vo_contains(s, vidx, dl.myp);
            if (inside) { finished = true; dl.vstart = vidx; }
            else if (++dl.vo >= nvo) {
                finished = true;
                any = 1;
                const v2 curr = v2_sub(dl.myp, ent_pos);
                const float len = v2_len(v2_sub(des_v, curr));
                if (len < best || (len == best && best_idx != 0x7fffffff && dl.myk < best_idx)) { best = len; best_idx = dl.myk; best_p = curr; }
            }
            if (finished) dl.busy = 0;
        }
    }
}

// compute_all_hrvos / compute_all_vos (clearpath.c:216-247): the ray table of the velocity obstacles,
// one neighbour per lane, order-preserving compaction. Returns the number of rays (2 per obstacle).
__device__ int build_vos(VelSmem &s, const cp_ent ent, int ndyn, int nstat, uint32_t lane)
{
    // ---- compute_all_hrvos / compute_all_vos: one neighbour per lane, order-preserving compaction ----
    int n_rays = 0;
    {
        bool keep = false;
        v2 apex = {0.f, 0.f}, left = {0.f, 0.f}, right = {0.f, 0.f};
        if ((int)lane < ndyn) {
            const cp_ent nb = s.dyn[lane];
            if (!(v2_len(v2_sub(nb.pos, ent.pos)) < EPS_F)) {        // same_position (clearpath.c:123)
                keep = true;
                vo_edges(ent, nb, right, left);
                // compute_rvo / compute_hrvo (clearpath.c:161-214)
                const v2 rvo_apex = v2_add(ent.pos, v2_scale(v2_add(ent.vel, nb.vel), 0.5f));
                const v2 centerline = v2_add(left, right);
                const v2 vo_apex = v2_add(ent.pos, nb.vel);
                const float det = (centerline.x * ent.vel.z) - (centerline.z * ent.vel.x);
                apex = rvo_apex;
                if (det > EPS_F) {
                    v2 p;
                    if (line_isect(ray{rvo_apex, left}, ray{vo_apex, right}, p)) apex = p;
                } else if (det < -EPS_F) {
                    v2 p;
                    if (line_isect(ray{rvo_apex, right}, ray{vo_apex, left}, p)) apex = p;
                }
            }
        }
        const uint32_t m = __ballot_sync(FULL, keep);
        if (keep) {
            const int k = 2 * __popc(m & ((1u << lane) - 1));
            s.vo_src[k >> 1] = (uint8_t)lane;
            s.rpx[k] = apex.x; s.rpz[k] = apex.z; s.rdx[k] = left.x; s.rdz[k] = left.z; s.rsl[k] = line_slope(left);
            s.rpx[k + 1] = apex.x; s.rpz[k + 1] = apex.z; s.rdx[k + 1] = right.x; s.rdz[k + 1] = right.z; s.rsl[k + 1] = line_slope(right);
        }
        n_rays = 2 * __popc(m);
    }
    {
        bool keep = false;
        v2 apex = {0.f, 0.f}, left = {0.f, 0.f}, right = {0.f, 0.f};
        if ((int)lane < nstat) {
            const cp_ent nb = s.stat[lane];
            if (!(v2_len(v2_sub(nb.pos, ent.pos)) < EPS_F)) {
                keep = true;
                vo_edges(ent, nb, right, left);
                apex = v2_add(ent.pos, nb.vel);                       // compute_vo (clearpath.c:153)
            }
        }
        const uint32_t m = __ballot_sync(FULL, keep);
        if (keep) {
            const int k = n_rays + 2 * __popc(m & ((1u << lane) - 1));
            s.vo_src[k >> 1] = (uint8_t)(32 + lane);
            s.rpx[k] = apex.x; s.rpz[k] = apex.z; s.rdx[k] = left.x; s.rdz[k] = left.z; s.rsl[k] = line_slope(left);
            s.rpx[k + 1] = apex.x; s.rpz[k + 1] = apex.z; s.rdx[k + 1] = right.x; s.rdz[k + 1] = right.z; s.rsl[k + 1] = line_slope(right);
        }
        n_rays += 2 * __popc(m);
    }
    __syncwarp();
    return n_rays;
}

// clearpath_new_velocity (clearpath.c:552). Warp-cooperative; returns a warp-uniform status.
__device__ bool clearpath_new_velocity(VelSmem &s, const cp_ent ent, const v2 des_v, int ndyn, int nstat,
                                       uint32_t lane, v2 &out, int &n_rays_out)
{
    const int n_rays = build_vos(s, ent, ndyn, nstat, lane);
    n_rays_out = n_rays;
    const int nvo = n_rays >> 1;

    // ---- is the preferred velocity admissible? one velocity obstacle per lane ----
    const v2 des_v_ws = v2_add(ent.pos, des_v);
    bool in_any = false;
    for (int i = lane; i < nvo; i += 32) in_any |= vo_contains(s, i, des_v_ws);
    if (!__any_sync(FULL, in_any)) {
        out = des_v;
        return true;
    }

    // ---- compute_vo_xpoints + compute_vdes_proj_points + compute_vnew, fused: ray pairs are intersected
    //      32 at a time, the survivors are compacted into a small queue, and the queue is drained by
    //      drain_candidates(); the candidate list is never materialised ----
    float best = __int_as_float(0x7f800000);    // +inf ; `len < min_dist` with min_dist = INFINITY
    int best_idx = 0x7fffffff;
    v2 best_p = {0.0f, 0.0f};
    int any = 0, qn = 0;
    DrainLane dl;
    const int npairs = n_rays * n_rays;
    // Exact pruning: compute_vnew (clearpath.c:368) keeps the admissible candidate nearest to des_v (first
    // one on ties), so a candidate that is certainly farther than an admissible candidate already found
    // can neither win nor change the tie-break and need not be tested against the obstacles at all. The
    // projection points of compute_vdes_proj_points (sequence indices npairs..npairs+n_rays-1) are the
    // nearest points of each ray to des_v: they are drained FIRST to get a tight bound, then the ray-pair
    // intersections are filtered against the warp-wide bound before they enter the queue.
    for (int base = 0; base < n_rays; base += 32) {
        const int r = base + (int)lane;
        const bool ok = r < n_rays;
        if (ok) {
            const v2 d = {s.rdx[r], s.rdz[r]};
            const float len = v2_dot(d, des_v);
            const v2 p = v2_add(v2{s.rpx[r], s.rpz[r]}, v2_scale(d, len));
            s.cqx[qn + (int)lane] = p.x; s.cqz[qn + (int)lane] = p.z; s.cqk[qn + (int)lane] = npairs + r;
        }
        qn += min(32, n_rays - base);
        if (qn > CQ_CAP - 32 || base + 32 >= n_rays) {
            __syncwarp();
            drain_candidates(s, qn, nvo, ent.pos, des_v, lane, best, best_idx, best_p, any, dl, true);     // the bound below needs them all
            __syncwarp();
            qn = 0;
        }
    }
    float bound2 = __int_as_float(0x7f800000);
    auto refresh_bound = [&]() {
        float b = best;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) b = fminf(b, __shfl_xor_sync(FULL, b, off));
        bound2 = b * b * 1.00001f;              // margin >> float rounding of the two squared lengths
    };
    refresh_bound();
    int i = 0, j = (int)lane;                   // pair index of this lane: k = i * n_rays + j
    while (j >= n_rays) { j -= n_rays; i++; }
    for (int base = 0; base < npairs; base += 32) {
        const int k = base + (int)lane;
        v2 p = {0.f, 0.f};
        bool ok = false;
        if (k < npairs) {
            if (i != j) {
                // C_RayRayIntersection2D (collision.c:854)
                const v2 p1 = {s.rpx[i], s.rpz[i]}, p2 = {s.rpx[j], s.rpz[j]};
                if (line_isect_s(p1, s.rsl[i], p2, s.rsl[j], p)) {
                    const float ddx = des_v.x - (p.x - ent.pos.x), ddz = des_v.z - (p.z - ent.pos.z);
                    ok = !(ddx * ddx + ddz * ddz > bound2) &&
                         !(quot_lt0(p.x - p1.x, s.rdx[i]) || quot_lt0(p.z - p1.z, s.rdz[i]) ||
                           quot_lt0(p.x - p2.x, s.rdx[j]) || quot_lt0(p.z - p2.z, s.rdz[j]));
                }
            }
        }
        const uint32_t m = __ballot_sync(FULL, ok);
        if (ok) {
            const int q = qn + __popc(m & ((1u << lane) - 1));
            s.cqx[q] = p.x; s.cqz[q] = p.z; s.cqk[q] = k;
        }
        qn += __popc(m);
        j += 32;
        while (j >= n_rays) { j -= n_rays; i++; }
        if (qn > CQ_CAP - 32 || base + 32 >= npairs) {
            __syncwarp();
            drain_candidates(s, qn, nvo, ent.pos, des_v, lane, best, best_idx, best_p, any, dl, base + 32 >= npairs);
            __syncwarp();
            qn = 0;
            refresh_bound();
        }
    }
    any = __any_sync(FULL, any);
    if (!any) return false;
    // warp arg-min on (len, idx); lanes that never improved hold (+inf, INT_MAX)
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const float ob = __shfl_xor_sync(FULL, best, off);
        const int oi = __shfl_xor_sync(FULL, best_idx, off);
        const float ox = __shfl_xor_sync(FULL, best_p.x, off), oz = __shfl_xor_sync(FULL, best_p.z, off);
        if (ob < best || (ob == best && oi < best_idx)) { best = ob; best_idx = oi; best_p = {ox, oz}; }
    }
    out = (best_idx == 0x7fffffff) ? v2{0.0f, 0.0f} : best_p;
    return true;
}

// ------------------------------------------------------------------------------------------
// G_ClearPath_NewVelocity's retry loop (clearpath.c:702-713) in ONE pass. After a solve that finds no admissible
// velocity the reference drops the furthest neighbour (remove_furthest :390) and solves again from scratch, while both
// neighbour lists are non-empty. Which neighbour goes at which step depends on the distances and the list order only,
// never on the velocities, so the whole removal schedule is known up front: neighbour n leaves at time rank(n). The
// obstacle of a neighbour and the candidate points generated by its two rays do not depend on the other neighbours,
// hence for every candidate point c of the FIRST solve
//     adm(c)   = max rank of the obstacles that contain c   (it becomes admissible once they are all gone)
//     death(c) = min rank of the obstacles whose rays generate c
// and the solve after t removals succeeds iff the preferred velocity (adm <= t) or some candidate (adm <= t < death) is
// admissible. The first such t is T = min(adm); by minimality every candidate usable at T has adm == T exactly, and
// compute_vnew (:368) picks the one nearest to the preferred velocity, first in ITS list order on ties -- the order of
// the ray table after T swap-with-last deletions; a tie between two different points is therefore flagged and that (rare)
// entity replays the loop literally. Obstacles are tested in decreasing rank, so
// the first hit is the maximum and most points end at the nearest (widest) obstacles after one or two tests.
// Cost: one solve instead of up to 63.
// ------------------------------------------------------------------------------------------
// obstacle ranks from the neighbour ranks, and the obstacles ordered by decreasing rank (index ascending among equals)
__device__ __forceinline__ void retry_rank_vos(VelSmem &s, int nvo, uint32_t lane)
{
    for (int v = lane; v < nvo; v += 32) s.vo_rank[v] = s.nb_rank[s.vo_src[v]];
    __syncwarp();
    for (int v = lane; v < nvo; v += 32) {
        const int r = s.vo_rank[v];
        int p = 0;
        for (int u = 0; u < nvo; u++) { const int ru = s.vo_rank[u]; p += (ru > r) || (ru == r && u < v); }
        s.vo_ord[p] = (uint8_t)v;
    }
    __syncwarp();
}

// removal schedule; returns the number of removals after which the loop ends (no solve happens at that time)
__device__ int retry_schedule(VelSmem &s, const v2 pos, int ndyn, int nstat, int nvo, uint32_t lane)
{
    for (int k = lane; k < 64; k += 32) {
        const bool valid = k < 32 ? k < ndyn : (k - 32) < nstat;
        float d = -__int_as_float(0x7f800000);
        if (valid) { const cp_ent e = k < 32 ? s.dyn[k] : s.stat[k - 32]; d = v2_len(v2_sub(pos, e.pos)); }
        s.ndist[k] = d; s.nb_rank[k] = 255; s.cur[k] = (uint8_t)k;
    }
    __syncwarp();
    int nd = ndyn, ns = nstat, t = 0, t_end = 0;
    while (true) {
        float bd = -__int_as_float(0x7f800000);
        int bp = 0x7fffffff;
        for (int q = lane; q < nd + ns; q += 32) {
            const int slot = q < nd ? s.cur[q] : s.cur[32 + q - nd];
            const float d = s.ndist[slot];
            if (d > bd) { bd = d; bp = q; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const float od = __shfl_xor_sync(FULL, bd, off);
            const int op = __shfl_xor_sync(FULL, bp, off);
            if (od > bd || (od == bd && op < bp)) { bd = od; bp = op; }
        }
        if (bp == 0x7fffffff) { t_end = t + 1; break; }      // nothing left to remove: the loop condition fails next
        t++;
        if (lane == 0) {
            int slot;
            if (bp < nd) { slot = s.cur[bp]; s.cur[bp] = s.cur[nd - 1]; }
            else { const int j = bp - nd; slot = s.cur[32 + j]; s.cur[32 + j] = s.cur[32 + ns - 1]; }
            s.nb_rank[slot] = (uint8_t)t;
        }
        if (bp < nd) nd--; else ns--;
        __syncwarp();
        if (!(nd > 0 && ns > 0)) { t_end = t; break; }
    }
    retry_rank_vos(s, nvo, lane);
    return t_end;
}

// The same schedule without the serial loop, for the common case that no two neighbours are exactly equally far away:
// the loop then removes them in descending distance whatever the list order, neighbour n leaves at time
// 1 + #{m : d(m) > d(n)}, and the loop ends when the last member of either list has left. Equal distances (lattice
// crowds) fall back to the literal schedule above, whose tie-break follows the swap-with-last list order.
__device__ int retry_schedule_fast(VelSmem &s, const v2 pos, int ndyn, int nstat, int nvo, uint32_t lane)
{
    for (int k = lane; k < 64; k += 32) {
        const bool valid = k < 32 ? k < ndyn : (k - 32) < nstat;
        float d = -__int_as_float(0x7f800000);
        if (valid) { const cp_ent e = k < 32 ? s.dyn[k] : s.stat[k - 32]; d = v2_len(v2_sub(pos, e.pos)); }
        s.ndist[k] = d;
    }
    __syncwarp();
    bool tie = false;
    int rk[2] = {0, 0};
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int k = (int)lane + 32 * h;
        const bool valid = h == 0 ? (int)lane < ndyn : (int)lane < nstat;
        if (valid) {
            const float d = s.ndist[k];
            int r = 1;
            for (int j = 0; j < ndyn; j++) { const float dj = s.ndist[j]; r += dj > d; tie |= (dj == d && j != k); }
            for (int j = 0; j < nstat; j++) { const float dj = s.ndist[32 + j]; r += dj > d; tie |= (dj == d && 32 + j != k); }
            rk[h] = r;
        }
    }
    if (__any_sync(FULL, tie)) return retry_schedule(s, pos, ndyn, nstat, nvo, lane);
    int md = rk[0], ms = rk[1];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { md = max(md, __shfl_xor_sync(FULL, md, off)); ms = max(ms, __shfl_xor_sync(FULL, ms, off)); }
    const int t_end = min(md, ms);
    s.nb_rank[lane] = (uint8_t)(((int)lane < ndyn && rk[0] <= t_end) ? rk[0] : 255);
    s.nb_rank[32 + lane] = (uint8_t)(((int)lane < nstat && rk[1] <= t_end) ? rk[1] : 255);
    __syncwarp();
    retry_rank_vos(s, nvo, lane);
    return t_end;
}

struct retry_best { int T; float dist; int id; v2 p; int tie; };

// (time, distance) order. Two DIFFERENT points at exactly the same time and distance would be ordered by their position in
// the candidate list of the solve after T removals (compute_vnew keeps the first, clearpath.c:368) -- that list order
// depends on the swap-with-last deletions done so far; instead of reproducing it the tie is flagged and the caller
// replays the reference's loop literally (it practically never happens: identical points, e.g. xpoint(i, j) and
// xpoint(j, i), are no tie -- either one gives the same velocity).
__device__ __forceinline__ bool retry_better(int T, float dist, const v2 p, retry_best &b)
{
    if (T != b.T) return T < b.T;
    if (dist != b.dist) return dist < b.dist;
    if (b.id >= 0 && (p.x != b.p.x || p.z != b.p.z)) b.tie = 1;
    return false;
}

// the outcome of the retry loop from the per-lane bests: smallest time, then distance, then list position at that time
__device__ __forceinline__ v2 retry_finish(retry_best &best, int adm_des, int t_end, const v2 des_v, uint32_t lane, bool &exact)
{
    int T = best.T;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) T = min(T, __shfl_xor_sync(FULL, T, off));
    if (best.T != T) { best.dist = __int_as_float(0x7f800000); best.id = -1; best.tie = 0; }
    if (adm_des <= T && adm_des <= t_end - 1) return des_v;     // inside_pcr(des_v) is tested before any candidate (:602)
    float d = best.dist;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) d = fminf(d, __shfl_xor_sync(FULL, d, off));
    const bool mine = best.id >= 0 && best.dist == d;
    const uint32_t mm = __ballot_sync(FULL, mine);
    if (!mm) return v2{0.0f, 0.0f};                              // no solve before the loop ends finds a point
    const int src = __ffs(mm) - 1;
    v2 out;
    out.x = __shfl_sync(FULL, best.p.x, src); out.z = __shfl_sync(FULL, best.p.z, src);
    // ties between different points, inside a lane or across lanes: list order would decide
    const bool differs = mine && (best.tie || best.p.x != out.x || best.p.z != out.z);
    if (__any_sync(FULL, differs)) exact = false;
    return out;
}

// like drain_candidates, for the retry emulation: cqk holds the candidate id, cqd its death time
__device__ __forceinline__ void drain_ranked(const VelSmem &s, int qn, int nvo, const v2 ent_pos, const v2 des_v,
                                             uint32_t lane, retry_best &best)
{
    int next = 0, my = -1, k = 0, myid = 0, mydeath = 0;
    v2 myp = {0.0f, 0.0f};
    while (true) {
        const bool need = my < 0;
        const uint32_t mneed = __ballot_sync(FULL, need);
        const int avail = qn - next;
        if (need) {
            const int rank = __popc(mneed & ((1u << lane) - 1));
            if (rank < avail) { my = next + rank; k = 0; myp = {s.cqx[my], s.cqz[my]}; myid = s.cqk[my]; mydeath = s.cqd[my]; }
        }
        next += min(__popc(mneed), avail);
        if (!__any_sync(FULL, my >= 0)) break;
        if (my >= 0) {
            bool finished = false;
            int adm = -1;
            if (k < nvo) {
                const int v = s.vo_ord[k];
                const int r = s.vo_rank[v];
                // obstacles come in decreasing rank, so the first hit is the maximum rank among the containing ones
                if (vo_contains(s, v, myp)) { adm = r; finished = true; }
                else if (++k >= nvo) { adm = 0; finished = true; }
            } else { adm = 0; finished = true; }
            if (finished) {
                if (adm < mydeath && adm <= best.T) {
                    const v2 curr = v2_sub(myp, ent_pos);
                    const float len = v2_len(v2_sub(des_v, curr));
                    if (retry_better(adm, len, curr, best)) { best.T = adm; best.dist = len; best.id = myid; best.p = curr; best.tie = 0; }
                }
                my = -1;
            }
        }
    }
}

// everything G_ClearPath_NewVelocity does after its first solve found nothing. The ray table of that solve is still in
// shared memory (build_vos). Returns the velocity of the first successful later solve, or zero when the loop ends first;
// `exact` is cleared when an order-dependent tie was met (the caller then replays the loop literally).
__device__ v2 clearpath_retry(VelSmem &s, const cp_ent ent, const v2 des_v, int ndyn, int nstat, int n_rays, uint32_t lane, bool &exact)
{
    exact = true;
    const int nvo = n_rays >> 1;
    // with one of the two lists empty the loop condition fails right after the first removal (the common case in a crowd
    // where everybody moves): no second solve, the answer is zero
    if (ndyn == 0 || nstat == 0) return v2{0.0f, 0.0f};
    const int t_end = retry_schedule_fast(s, ent.pos, ndyn, nstat, nvo, lane);
    if (t_end <= 1) return v2{0.0f, 0.0f};                   // the loop ends right after the first removal
    // the preferred velocity: admissible once every obstacle that contains it is gone
    const v2 des_v_ws = v2_add(ent.pos, des_v);
    int adm_des = 0;
    for (int v = lane; v < nvo; v += 32)
        if (vo_contains(s, v, des_v_ws)) adm_des = max(adm_des, (int)s.vo_rank[v]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) adm_des = max(adm_des, __shfl_xor_sync(FULL, adm_des, off));
    retry_best best; best.T = min(adm_des, t_end - 1); best.dist = __int_as_float(0x7f800000); best.id = -1; best.p = {0.0f, 0.0f}; best.tie = 0;
    const int npairs = n_rays * n_rays;
    int qn = 0;
    auto flush = [&](bool last) {
        if (qn > CQ_CAP - 32 || (last && qn > 0)) {
            __syncwarp();
            drain_ranked(s, qn, nvo, ent.pos, des_v, lane, best);
            __syncwarp();
            qn = 0;
            int t = best.T;                                   // the warp-wide best time bounds what is still worth testing
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) t = min(t, __shfl_xor_sync(FULL, t, off));
            if (t < best.T) { best.T = t; best.dist = __int_as_float(0x7f800000); best.id = -1; best.tie = 0; }
        }
    };
    for (int base = 0; base < n_rays; base += 32) {            // projection points (compute_vdes_proj_points, :344)
        const int r = base + (int)lane;
        if (r < n_rays) {
            const v2 d = {s.rdx[r], s.rdz[r]};
            const float len = v2_dot(d, des_v);
            const v2 p = v2_add(v2{s.rpx[r], s.rpz[r]}, v2_scale(d, len));
            s.cqx[qn + (int)lane] = p.x; s.cqz[qn + (int)lane] = p.z; s.cqk[qn + (int)lane] = 0x8000 | r;
            s.cqd[qn + (int)lane] = s.vo_rank[r >> 1];
        }
        qn += min(32, n_rays - base);
        flush(base + 32 >= n_rays);
    }
    int i = 0, j = (int)lane;
    while (j >= n_rays && n_rays > 0) { j -= n_rays; i++; }
    for (int base = 0; base < npairs; base += 32) {            // ray-pair intersections (compute_vo_xpoints, :321)
        const int k = base + (int)lane;
        v2 p = {0.f, 0.f};
        bool ok = false;
        int death = 0;
        if (k < npairs && i != j) {
            death = min((int)s.vo_rank[i >> 1], (int)s.vo_rank[j >> 1]);
            if (death > 0) {           // a pair that dies at time <= 0 cannot exist (ranks start at 1); kept for symmetry
                const v2 p1 = {s.rpx[i], s.rpz[i]}, p2 = {s.rpx[j], s.rpz[j]};
                if (line_isect_s(p1, s.rsl[i], p2, s.rsl[j], p))
                    ok = !(quot_lt0(p.x - p1.x, s.rdx[i]) || quot_lt0(p.z - p1.z, s.rdz[i]) ||
                           quot_lt0(p.x - p2.x, s.rdx[j]) || quot_lt0(p.z - p2.z, s.rdz[j]));
            }
        }
        const uint32_t m = __ballot_sync(FULL, ok);
        if (ok) {
            const int q = qn + __popc(m & ((1u << lane) - 1));
            s.cqx[q] = p.x; s.cqz[q] = p.z; s.cqk[q] = (i << 7) | j; s.cqd[q] = (uint8_t)death;
        }
        qn += __popc(m);
        j += 32;
        while (j >= n_rays) { j -= n_rays; i++; }
        flush(base + 32 >= npairs);
    }
    return retry_finish(best, adm_des, t_end, des_v, lane, exact);
}

// remove_furthest (clearpath.c:390): first strict maximum over dyn then stat; swap-with-last delete
__device__ void remove_furthest(VelSmem &s, const v2 pos, int &ndyn, int &nstat, uint32_t lane)
{
    float d = -__int_as_float(0x7f800000);
    int idx = 0x7fffffff;
    const int n = ndyn + nstat;
    // n <= 64: two candidates per lane, sequence index = position in (dyn ++ stat)
    for (int k = lane; k < n; k += 32) {
        const cp_ent e = k < ndyn ? s.dyn[k] : s.stat[k - ndyn];
        const float len = v2_len(v2_sub(pos, e.pos));
        if (len > d) { d = len; idx = k; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const float od = __shfl_xor_sync(FULL, d, off);
        const int oi = __shfl_xor_sync(FULL, idx, off);
        if (od > d || (od == d && oi < idx)) { d = od; idx = oi; }
    }
    if (idx != 0x7fffffff) {
        if (lane == 0) {
            if (idx < ndyn) s.dyn[idx] = s.dyn[ndyn - 1];
            else s.stat[idx - ndyn] = s.stat[nstat - 1];
        }
        if (idx < ndyn) ndyn--; else nstat--;
    }
    __syncwarp();
}

// ------------------------------------------------------------------------------------------
// Two-phase ClearPath. Everything G_ClearPath_NewVelocity does except the final choice is independent of
// the preferred velocity: the velocity obstacles depend on positions / velocities only, and so do the
// pairwise ray intersections (compute_vo_xpoints, clearpath.c:321) and their inside-PCR tests. Phase A
// (k_agent_velocity<1>, runs while the LOS chains are still in flight) therefore collects the ADMISSIBLE
// intersection points of every agent; phase B (k_agent_velocity<2>, after the fields are joined) computes
// the preferred velocity, tests it and its projections (compute_vdes_proj_points, :344) and picks the
// nearest admissible point by (distance, sequence index) = compute_vnew's first minimum (:368).
// ------------------------------------------------------------------------------------------
struct pf_xpoint { float x, z; int k; };
#define PF_PREP_XP_CAP 64
#define PF_PREP_OVERFLOW 0xFFFFFFFFu
struct pf_prep {
    uint32_t ndyn, nstat, nx, _pad;
    float sepx, sepz;
    uint32_t dyn_id[PFNAV_MAX_NEIGHBOURS], stat_id[PFNAV_MAX_NEIGHBOURS];
    pf_xpoint xp[PF_PREP_XP_CAP];
};

// like drain_candidates, but records every candidate that lies inside no velocity obstacle
__device__ __forceinline__ void drain_collect(const VelSmem &s, int qn, int nvo, uint32_t lane, pf_xpoint *out, int &cnt,
                                              DrainLane &dl, bool flush)
{
    int next = 0;
    while (true) {
        const bool need = !dl.busy;
        const uint32_t mneed = __ballot_sync(FULL, need);
        const int avail = qn - next;
        if (need && avail > 0) {
            const int rank = __popc(mneed & ((1u << lane) - 1));
            if (rank < avail) { const int my = next + rank; dl.busy = 1; dl.vo = 0; dl.myp = {s.cqx[my], s.cqz[my]}; dl.myk = s.cqk[my]; }
        }
        next += min(__popc(mneed), avail);
        if (!flush && next >= qn) break;
        if (!__any_sync(FULL, dl.busy)) break;
        bool admissible = false;
        if (dl.busy) {
            int vidx = dl.vo + dl.vstart;
            if (vidx >= nvo) vidx -= nvo;
            bool inside = false;
            if (dl.vo < nvo) inside = vo_contains(s, vidx, dl.myp);
            if (inside) { dl.busy = 0; dl.vstart = vidx; }
            else if (++dl.vo >= nvo) { admissible = true; dl.busy = 0; }
        }
        const uint32_t ma = __ballot_sync(FULL, admissible);
        if (admissible) {
            const int q = cnt + __popc(ma & ((1u << lane) - 1));
            if (q < PF_PREP_XP_CAP) { out[q].x = dl.myp.x; out[q].z = dl.myp.z; out[q].k = dl.myk; }
        }
        cnt += __popc(ma);
    }
}

// phase A: admissible ray-pair intersections of one agent -> out[0..cnt) (cnt > cap = overflow)
__device__ int clearpath_collect(VelSmem &s, const cp_ent ent, int ndyn, int nstat, uint32_t lane, pf_xpoint *out)
{
    const int n_rays = build_vos(s, ent, ndyn, nstat, lane);
    const int nvo = n_rays >> 1, npairs = n_rays * n_rays;
    int cnt = 0, qn = 0;
    DrainLane dl;
    int i = 0, j = (int)lane;
    while (j >= n_rays && n_rays > 0) { j -= n_rays; i++; }
    for (int base = 0; base < npairs; base += 32) {
        const int k = base + (int)lane;
        v2 p = {0.f, 0.f};
        bool ok = false;
        if (k < npairs && i != j) {
            const v2 p1 = {s.rpx[i], s.rpz[i]}, p2 = {s.rpx[j], s.rpz[j]};
            if (line_isect_s(p1, s.rsl[i], p2, s.rsl[j], p)) {
                ok = !(quot_lt0(p.x - p1.x, s.rdx[i]) || quot_lt0(p.z - p1.z, s.rdz[i]) ||
                       quot_lt0(p.x - p2.x, s.rdx[j]) || quot_lt0(p.z - p2.z, s.rdz[j]));
            }
        }
        const uint32_t m = __ballot_sync(FULL, ok);
        if (ok) {
            const int q = qn + __popc(m & ((1u << lane) - 1));
            s.cqx[q] = p.x; s.cqz[q] = p.z; s.cqk[q] = k;
        }
        qn += __popc(m);
        j += 32;
        while (j >= n_rays) { j -= n_rays; i++; }
        if (qn > CQ_CAP - 32 || base + 32 >= npairs) {
            __syncwarp();
            drain_collect(s, qn, nvo, lane, out, cnt, dl, base + 32 >= npairs);
            __syncwarp();
            qn = 0;
        }
    }
    return cnt;
}

// phase B: the choice among {des_v, its projections on the rays, the stored admissible intersections}
__device__ bool clearpath_finish(VelSmem &s, const cp_ent ent, const v2 des_v, int ndyn, int nstat, uint32_t lane,
                                 const pf_xpoint *xp, int nx, v2 &out, int &n_rays_out)
{
    const int n_rays = build_vos(s, ent, ndyn, nstat, lane);
    n_rays_out = n_rays;
    const int nvo = n_rays >> 1, npairs = n_rays * n_rays;
    const v2 des_v_ws = v2_add(ent.pos, des_v);
    bool in_any = false;
    for (int i = lane; i < nvo; i += 32) in_any |= vo_contains(s, i, des_v_ws);
    if (!__any_sync(FULL, in_any)) { out = des_v; return true; }
    float best = __int_as_float(0x7f800000);
    int best_idx = 0x7fffffff;
    v2 best_p = {0.0f, 0.0f};
    int any = 0, qn = 0;
    for (int base = 0; base < n_rays; base += 32) {
        const int r = base + (int)lane;
        if (r < n_rays) {
            const v2 d = {s.rdx[r], s.rdz[r]};
            const float len = v2_dot(d, des_v);
            const v2 p = v2_add(v2{s.rpx[r], s.rpz[r]}, v2_scale(d, len));
            s.cqx[qn + (int)lane] = p.x; s.cqz[qn + (int)lane] = p.z; s.cqk[qn + (int)lane] = npairs + r;
        }
        qn += min(32, n_rays - base);
        if (qn > CQ_CAP - 32 || base + 32 >= n_rays) {
            __syncwarp();
            DrainLane dl;
            drain_candidates(s, qn, nvo, ent.pos, des_v, lane, best, best_idx, best_p, any, dl, true);
            __syncwarp();
            qn = 0;
        }
    }
    for (int q = lane; q < nx; q += 32) {       // the intersections phase A found admissible
        const pf_xpoint c = xp[q];
        const v2 curr = v2_sub(v2{c.x, c.z}, ent.pos);
        const float len = v2_len(v2_sub(des_v, curr));
        any = 1;
        if (len < best || (len == best && best_idx != 0x7fffffff && c.k < best_idx)) { best = len; best_idx = c.k; best_p = curr; }
    }
    any = __any_sync(FULL, any);
    if (!any) return false;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const float ob = __shfl_xor_sync(FULL, best, off);
        const int oi = __shfl_xor_sync(FULL, best_idx, off);
        const float ox = __shfl_xor_sync(FULL, best_p.x, off), oz = __shfl_xor_sync(FULL, best_p.z, off);
        if (ob < best || (ob == best && oi < best_idx)) { best = ob; best_idx = oi; best_p = {ox, oz}; }
    }
    out = (best_idx == 0x7fffffff) ? v2{0.0f, 0.0f} : best_p;
    return true;
}

