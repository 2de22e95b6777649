// xray_inpaint_plan.h — host-only planning of inpaint_xray_quadtree (xray_inpaint.inl; no CUDA: the CPU tests compile it with
// g++):
//   quad_xy / quad_index / quad_neighbor: SpatialNodeId <-> NodeId and SpatialNodeId::neighbor (quadtree/src/lib.rs:290-351)
//   xray_inpaint_adjacent:  get_adjacent_leaf_node_ids (inpaint_xray_quadtree.rs:41-71)
//   xray_inpaint_grid:      one aligned 2^j x 2^j block of leaves: its leaves, the leaves of its 1-halo (whose inpaint images
//                           its leaves need) and the visible tiles of its 2-halo that those images are stitched from
//   xray_inpaint_device_bytes / xray_inpaint_block_depth: what a block and the parents' walk hold on the device
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <functional>
#include <unordered_set>
#include <utility>
#include <vector>

#include "xray_merge_plan.h"

namespace pcv {

// NodeId -> SpatialNodeId: bit 1 of each base-4 digit is x, bit 0 is y, most significant digit first
inline void quad_xy(uint32_t level, uint64_t index, uint64_t& x, uint64_t& y) {
    x = y = 0;
    for (uint32_t l = 0; l < level; ++l) {
        x |= ((index >> (2 * l + 1)) & 1) << l;
        y |= ((index >> (2 * l)) & 1) << l;
    }
}
inline uint64_t quad_index(uint32_t level, uint64_t x, uint64_t y) {
    uint64_t index = 0;
    for (uint32_t l = 0; l < level; ++l) index |= (((x >> l) & 1) << (2 * l + 1)) | (((y >> l) & 1) << (2 * l));
    return index;
}
// SpatialNodeId::neighbor: (x + dx, y + dy), Top = y + 1; false outside [0, 2^level)
inline bool quad_neighbor(uint32_t level, uint64_t index, int dx, int dy, uint64_t& out) {
    uint64_t x, y;
    quad_xy(level, index, x, y);
    const int64_t nx = (int64_t)x + dx, ny = (int64_t)y + dy, lim = (int64_t)1 << level;
    if (nx < 0 || ny < 0 || nx >= lim || ny >= lim) return false;
    out = quad_index(level, (uint64_t)nx, (uint64_t)ny);
    return true;
}

// Left, Top, Right, Bottom, in get_adjacent_leaf_node_ids' order
constexpr int kInpaintDirs[4][2] = {{-1, 0}, {0, 1}, {1, 0}, {0, -1}};

// The deepest nodes of the neighbour pieces' metas (`nbr[d]`: the meta of R's neighbour in direction d, or null) whose
// neighbour in the opposite direction is one of `leaves` (sorted indices at level D), sorted.
inline std::vector<uint64_t> xray_inpaint_adjacent(uint32_t D, const std::vector<uint64_t>& leaves, const std::array<const XrayMetaData*, 4>& nbr) {
    std::vector<uint64_t> out;
    for (int d = 0; d < 4; ++d) {
        if (!nbr[d]) continue;
        for (const auto& n : nbr[d]->nodes) {
            uint64_t o;
            if (n.first != nbr[d]->deepest_level || n.first != D || D > 31) continue;
            if (quad_neighbor(D, n.second, -kInpaintDirs[d][0], -kInpaintDirs[d][1], o) && std::binary_search(leaves.begin(), leaves.end(), o)) out.push_back(n.second);
        }
    }
    std::sort(out.begin(), out.end());
    out.erase(std::unique(out.begin(), out.end()), out.end());
    return out;
}

// One block of leaves: B = 2^j, spatial origin (bx0, by0).  Grids are row-major with row 0 at the top (the largest y): the tile
// grid covers x in [bx0 - 2, bx0 + B + 2), y in (by0 - 3, by0 + B + 1], the image grid the same with a halo of 1.
struct XrayInpaintGrid {
    uint64_t block = 0;                 // index of the block at level D - j
    int64_t bx0 = 0, by0 = 0;
    uint32_t B = 1;
    std::vector<uint64_t> leaves;       // the block's leaves, index order
    std::vector<uint64_t> image_ids;    // the leaves of the 1-halo region (inpaint images), grid order
    std::vector<uint32_t> image_pos;    // [image] ix | iy << 16
    std::vector<int32_t> tile_slot;     // [(B + 4)^2] slot in tile_ids, or -1
    std::vector<uint64_t> tile_ids;     // the visible tiles some image is stitched from, grid order
    std::vector<std::pair<int32_t, int32_t>> hpairs, vpairs;  // (image, its Right image), (image, its Bottom image)
    std::vector<int32_t> leaf_image;    // [leaf] its image
};

// `leaves`: the sorted leaf indices at level D; `block_leaves`: those of block `block` (index order); `visible(index)`: whether
// the tile at level D is an <id>.png the stitch sees.
inline XrayInpaintGrid xray_inpaint_grid(uint32_t D, uint32_t j, uint64_t block, const std::vector<uint64_t>& block_leaves,
                                         const std::vector<uint64_t>& leaves, const std::function<bool(uint64_t)>& visible) {
    XrayInpaintGrid g;
    g.block = block;
    g.B = 1u << j;
    g.leaves = block_leaves;
    uint64_t x0, y0;
    quad_xy(D - j, block, x0, y0);
    g.bx0 = (int64_t)(x0 << j), g.by0 = (int64_t)(y0 << j);
    const int64_t lim = (int64_t)1 << D, B = g.B, GI = B + 2, GT = B + 4;
    auto is_leaf = [&](uint64_t i) { return std::binary_search(leaves.begin(), leaves.end(), i); };
    std::vector<int32_t> islot((size_t)(GI * GI), -1);
    for (int64_t iy = 0; iy < GI; ++iy)
        for (int64_t ix = 0; ix < GI; ++ix) {
            const int64_t x = g.bx0 - 1 + ix, y = g.by0 + B - iy;
            if (x < 0 || y < 0 || x >= lim || y >= lim) continue;
            const uint64_t id = quad_index(D, (uint64_t)x, (uint64_t)y);
            if (!is_leaf(id)) continue;
            islot[(size_t)(iy * GI + ix)] = (int32_t)g.image_ids.size();
            g.image_ids.push_back(id);
            g.image_pos.push_back((uint32_t)ix | ((uint32_t)iy << 16));
        }
    std::vector<char> used((size_t)(GT * GT), 0);
    for (uint32_t p : g.image_pos)
        for (int dy = 0; dy < 3; ++dy)
            for (int dx = 0; dx < 3; ++dx) used[(size_t)(((p >> 16) + dy) * GT + (p & 0xFFFFu) + dx)] = 1;
    g.tile_slot.assign((size_t)(GT * GT), -1);
    for (int64_t gy = 0; gy < GT; ++gy)
        for (int64_t gx = 0; gx < GT; ++gx) {
            const int64_t x = g.bx0 - 2 + gx, y = g.by0 + B + 1 - gy;
            if (!used[(size_t)(gy * GT + gx)] || x < 0 || y < 0 || x >= lim || y >= lim) continue;
            const uint64_t id = quad_index(D, (uint64_t)x, (uint64_t)y);
            if (!visible(id)) continue;
            g.tile_slot[(size_t)(gy * GT + gx)] = (int32_t)g.tile_ids.size();
            g.tile_ids.push_back(id);
        }
    for (int64_t iy = 0; iy < GI; ++iy)
        for (int64_t ix = 0; ix < GI; ++ix) {
            const int32_t s = islot[(size_t)(iy * GI + ix)];
            if (s < 0) continue;
            if (ix + 1 < GI && islot[(size_t)(iy * GI + ix + 1)] >= 0) g.hpairs.emplace_back(s, islot[(size_t)(iy * GI + ix + 1)]);
            if (iy + 1 < GI && islot[(size_t)((iy + 1) * GI + ix)] >= 0) g.vpairs.emplace_back(s, islot[(size_t)((iy + 1) * GI + ix)]);
        }
    for (uint64_t id : g.leaves) {
        uint64_t x, y;
        quad_xy(D, id, x, y);
        g.leaf_image.push_back(islot[(size_t)((g.by0 + B - (int64_t)y) * GI + ((int64_t)x - g.bx0 + 1))]);
    }
    return g;
}

// Device bytes of one block at depth j with T px tiles, at most: the (2^j + 4)^2 tiles and their slot grid, the (2^j + 2)^2
// inpaint images with their masks, nearest rows, envelopes (14 bytes per pixel of 2T x 2T), positions, hole counts and pairs,
// and the leaf being cropped.  k = 0 (no inpainting) holds one leaf tile.
inline uint64_t xray_inpaint_block_bytes(uint32_t j, uint32_t T, uint32_t k) {
    const uint64_t tile = (uint64_t)T * T * 4;
    if (k == 0) return tile;
    const uint64_t B = 1ull << j, tiles = (B + 4) * (B + 4), images = (B + 2) * (B + 2);
    return tiles * (tile + 4) + images * (14ull * 4 * T * T + 4 + 8 + 2 * 8) + tile;
}
// ... and the parents' walk from the leaves at level D up to the root at level L (xray_merge_device_bytes of D - L levels)
inline uint64_t xray_inpaint_device_bytes(uint32_t j, uint32_t T, uint32_t k, uint32_t D, uint32_t L) {
    return xray_inpaint_block_bytes(j, T, k) + xray_merge_device_bytes(D - L, T);
}
// The largest block depth j <= min(D - L, 5) that fits `budget`; -1 when not even j = 0 does.  Larger blocks recompute fewer
// halo images; 2^5 x 2^5 leaves bound the host's decoded tiles of one block to 36^2.
inline int xray_inpaint_block_depth(uint64_t budget, uint32_t T, uint32_t k, uint32_t D, uint32_t L) {
    int j = -1;
    for (uint32_t c = 0; c <= std::min<uint32_t>(D - L, 5); ++c)
        if (xray_inpaint_device_bytes(c, T, k, D, L) <= budget) j = (int)c;
    return k == 0 ? std::min(j, 0) : j;
}

}  // namespace pcv
