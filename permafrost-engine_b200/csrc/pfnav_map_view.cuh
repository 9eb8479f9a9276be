// pfnav_map_view.cuh -- the device's view of the committed map layers and the tile lookups the tick and the batched
// map queries share: the per-agent kernels (pfnav_agents.cu) and the query kernels (pfnav_query_kernel.cuh). Plain
// C++ apart from the CUDA keywords, so tests/emu can compile it on the CPU.
// Needs: <stdint.h>, <stddef.h>, fabs / min / max.
#pragma once

struct MapView {
    const uint8_t *cost; const uint16_t *blk;   // [layer][H64][W64]
    int W64, H64, chunk_w, chunk_h;
    float map_x, map_z;
};

struct tile_desc { int chunk_r, chunk_c, tile_r, tile_c; };

// M_Tile_DescForPoint2D with the nav resolution (tile.c:547; n_res nav.c:240): returns false
// outside the map box.
__device__ __forceinline__ bool desc_for_point(const MapView &m, float px, float pz, tile_desc &out)
{
    const float width = (float)(m.chunk_w * 256), height = (float)(m.chunk_h * 256);
    if (px > m.map_x || px < m.map_x - width) return false;
    if (pz < m.map_z || pz > m.map_z + height) return false;
    int chunk_r = (int)(fabs((double)(m.map_z - pz)) / 256.0);
    int chunk_c = (int)(fabs((double)(m.map_x - px)) / 256.0);
    chunk_r = min(max(chunk_r, 0), m.chunk_h - 1);
    chunk_c = min(max(chunk_c, 0), m.chunk_w - 1);
    const float base_x = m.map_x - (float)chunk_c * 256.0f;
    const float base_z = m.map_z + (float)chunk_r * 256.0f;
    int tile_r = (int)(fabs((double)(base_z - pz)) / 4);
    int tile_c = (int)(fabs((double)(base_x - px)) / 4);
    out.chunk_r = chunk_r; out.chunk_c = chunk_c;
    out.tile_r = min(max(tile_r, 0), 63);
    out.tile_c = min(max(tile_c, 0), 63);
    return true;
}

// M_NavPositionPathable / M_NavPositionBlocked (map.c:817, 831): both false outside the map box.
__device__ __forceinline__ void probe_tile(const MapView &m, int layer, float px, float pz, bool &pathable,
                                           bool &blocked)
{
    tile_desc td;
    pathable = false; blocked = false;
    if (!desc_for_point(m, px, pz, td)) return;
    const size_t off = ((size_t)layer * m.H64 + td.chunk_r * 64 + td.tile_r) * m.W64 + td.chunk_c * 64 + td.tile_c;
    pathable = m.cost[off] != 0xFF;
    blocked = m.blk[off] > 0;
}

// n_tile_blocked (nav.c:235)
__device__ __forceinline__ bool tile_blocked_abs(const MapView &m, int layer, int ar, int ac)
{
    const size_t off = ((size_t)layer * m.H64 + ar) * m.W64 + ac;
    return m.cost[off] == 0xFF || m.blk[off] > 0;
}

// N_IsAdjacentToImpassable (nav.c:4745) for the tile td: one of its 4 neighbours inside the map has cost 0xFF or a
// blocker. k_entity_update spells out the same loop: calling this function there changes that kernel's register
// allocation.
__device__ __forceinline__ bool adjacent_impassable(const MapView &m, int layer, const tile_desc &td)
{
    const int ar = td.chunk_r * 64 + td.tile_r, acol = td.chunk_c * 64 + td.tile_c;
    const int dr[4] = {-1, 0, 0, 1}, dc[4] = {0, -1, 1, 0};
    bool adj = false;
    for (int e = 0; e < 4 && !adj; e++) {
        const int nr = ar + dr[e], nc = acol + dc[e];
        if (nr < 0 || nr >= m.H64 || nc < 0 || nc >= m.W64) continue;
        adj = tile_blocked_abs(m, layer, nr, nc);
    }
    return adj;
}
