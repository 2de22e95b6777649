// xray_plan.h — host-only planning of the bounded X-ray quadtree driver (xray_api.inl; no CUDA: the CPU tests compile it with g++).
//   xray_block_depth:     how many quadtree levels one block of leaves spans, from the device-memory budget
//   xray_key_batches:     consecutive leaves of a block grouped so that their possible keys fit the key buffer
//   xray_levels_to_close: the post-order bookkeeping - which ancestors are complete when the walk moves on to the next subtree
//   xray_post_order:      every node of a subtree with the given leaves, each after all of its children
//   xray_octree_plan:     the octree sources' plan: block depth, node selection and key capacity
//   xray_clouds_fixed_bytes: what a list of resident octrees holds for the whole run besides the driver's own fixed set
//   s2_xray_plan:         the S2 cloud's leaf producer (s2_xray.inl): block depth, key capacity and attribute batch size
#pragma once
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

namespace pcv {

// Device bytes of the images at block depth g (the block root is g levels above the leaves) under `above` levels between the
// quadtree root and the block root:
//   - the block's leaf images, 4^g of them at most, and its parents up to the block root, (4^g - 1) / 3 of them (every level
//     of the block stays until the block root is built, so that the block leaves the device in one copy per level);
//   - per level above the block at most four finished children wait for their parent, plus the parent being built.
// `leaf_bytes` is everything the driver holds per leaf (image, bins, arguments); `tile_bytes` one RGBA tile.
inline uint64_t xray_block_bytes(int g, int above, uint64_t leaf_bytes, uint64_t tile_bytes) {
    const uint64_t leaves = 1ull << (2 * g), parents = (leaves - 1) / 3;
    return leaves * leaf_bytes + parents * tile_bytes + (4ull * (uint64_t)above + 1) * tile_bytes;
}

// Largest g <= min(depth, max_g) whose images take at most half of what the budget leaves after `fixed_bytes` (the other half
// holds the keys of a batch and the node selection); g = 0 when only a single leaf fits that way but fits the whole budget.
// -1: not even one leaf fits the budget.
inline int xray_block_depth(uint64_t budget, uint64_t fixed_bytes, int depth, int max_g, uint64_t leaf_bytes, uint64_t tile_bytes) {
    if (budget <= fixed_bytes || xray_block_bytes(0, depth, leaf_bytes, tile_bytes) > budget - fixed_bytes) return -1;
    const uint64_t half = (budget - fixed_bytes) / 2;
    int g = 0;
    while (g < depth && g < max_g && xray_block_bytes(g + 1, depth - g - 1, leaf_bytes, tile_bytes) <= half) ++g;
    return g;
}

// Key batches over the leaves of a block, in order: each batch is a run of consecutive leaves whose possible keys (`keys[i]`,
// one per point the leaf's location can hold) sum to at most `key_cap`.  Returns the batch starts plus an end sentinel, or an
// empty vector with `*too_big` = the first leaf that alone exceeds key_cap.
inline std::vector<uint32_t> xray_key_batches(const std::vector<uint64_t>& keys, uint64_t key_cap, int64_t* too_big) {
    std::vector<uint32_t> starts;
    *too_big = -1;
    uint64_t run = 0;
    for (size_t i = 0; i < keys.size(); ++i) {
        if (keys[i] > key_cap) {
            *too_big = (int64_t)i;
            return {};
        }
        if (starts.empty() || run + keys[i] > key_cap) {
            starts.push_back((uint32_t)i);
            run = 0;
        }
        run += keys[i];
    }
    starts.push_back((uint32_t)keys.size());
    return starts;
}

// a and b (a < b) are node indices `depth` levels below a common subtree root.  Returns how many ancestors of a are complete
// when the post-order walk moves from a's subtree to b's: those at 1, 2, ..., k levels above a (never the common root).
inline int xray_levels_to_close(uint64_t a, uint64_t b, int depth) {
    int k = 0;
    for (int up = 1; up < depth && (a >> (2 * up)) != (b >> (2 * up)); ++up) ++k;
    return k;
}

// Post-order of the subtree that holds exactly the ancestors of the given leaves: `leaves` are sorted, distinct indices
// `depth` levels below the subtree root.  Each entry is (levels above the leaves, index at that level); siblings come in
// index order, every node after its children, the subtree root last.
inline std::vector<std::pair<int, uint64_t>> xray_post_order(const std::vector<uint64_t>& leaves, int depth) {
    std::vector<std::pair<int, uint64_t>> out;
    for (size_t i = 0; i < leaves.size(); ++i) {
        out.emplace_back(0, leaves[i]);
        const int k = i + 1 < leaves.size() ? xray_levels_to_close(leaves[i], leaves[i + 1], depth) : depth;
        for (int up = 1; up <= k; ++up) out.emplace_back(up, leaves[i] >> (2 * up));
    }
    return out;
}

// What the driver runs with, from the budget: the block depth, the node selection's frontier capacity and locations per
// selection (octree sources) or candidates per pruning pass (S2), and what a block's leaves may hold besides their images.
struct XrayPlan {
    int g = -1;                // block depth (xray_block_depth); -1: not even one leaf fits
    uint32_t sel_cap = 0;      // octree sources: frontier pairs of one node selection
    uint64_t max_loc = 0;      // locations per node selection, or per pruning pass
    uint64_t key_cap = 0;      // XRay: keys of one batch
    uint64_t attr_leaves = 0;  // S2 attribute strategies: leaves whose slices one accumulation pass holds
};

// The plan of an octree source: `fixed` bytes for the whole run and `window` bytes of points (0 for a resident octree; the
// largest window of the blocks for an octree directory).  An eighth of what they leave goes to the node selection (half to
// its frontier, `sel_cap` pairs and `xray_pair_bytes(clouds)` more per pair, half to `max_loc` locations of `per_loc` bytes); g
// is the largest block depth <= max_g whose images fit besides; what remains after the block's images holds the keys of a
// batch, 4 bytes per key and its share of the work tiles.
// A pair costs 24 B of frontier and 16 B of work list.  `clouds` octrees select in turn, each frontier released before the
// next selection, but every cloud's work list stays until the batch's place passes: 24 + 16 clouds bytes per pair.
inline uint64_t xray_pair_bytes(uint32_t clouds) { return 24 + 16ull * clouds; }
inline XrayPlan xray_octree_plan(uint64_t budget, uint64_t fixed, uint64_t window, int depth, int max_g, uint64_t per_loc, uint64_t leaf_bytes,
                                 uint64_t tile_bytes, uint32_t clouds = 1) {
    XrayPlan p;
    const uint64_t pair = xray_pair_bytes(clouds);
    const uint64_t sel_bytes = budget > fixed + window ? (budget - fixed - window) / 8 : 0;
    p.sel_cap = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(sel_bytes / 2 / pair, 64), 48ull << 20);
    p.max_loc = std::max<uint64_t>(1, sel_bytes / 2 / per_loc);
    const uint64_t held = fixed + window + sel_bytes + pair * p.sel_cap;
    p.g = xray_block_depth(budget, held, depth, max_g, leaf_bytes, tile_bytes);
    if (p.g < 0) return p;
    const uint64_t used = held + xray_block_bytes(p.g, depth - p.g, leaf_bytes, tile_bytes);
    p.key_cap = budget > used ? std::min<uint64_t>((budget - used) / 5, 0xFFFFFFFEull) : 0;
    return p;
}

// The fixed bytes of resident octrees (xray_octree_plan's `fixed`): the driver's own fixed set `run_fixed`, each cloud's work
// list of every node for the pruning pass (16 B per tile and 16 B more), and the filter intervals (16 B each).  The clouds'
// frontiers and work lists of a key batch are counted per selection pair by xray_octree_plan (xray_pair_bytes).
inline uint64_t xray_clouds_fixed_bytes(uint64_t run_fixed, const std::vector<uint64_t>& cloud_tiles, uint32_t nfilt) {
    uint64_t fixed = run_fixed + 16ull * nfilt;
    for (uint64_t t : cloud_tiles) fixed += 16 * t + 16;
    return fixed;
}

// ---- the leaf producer of an S2 cloud (s2_xray.inl) --------------------------------------------------------------------------
// What it holds besides the run's fixed set (taps, mosaic, grey table, one attribute slice): the pruning pass's work list of
// every cell and the block's cell tiles, at most every tile again (16 B per tile each), the cell selection of one location (an
// 8 B pair per cell, 64 B of counters) and the filter intervals (16 B each).
inline uint64_t s2_xray_fixed_bytes(uint64_t ncells, uint64_t ntiles, uint32_t nfilt) { return 32 * ntiles + 8 * ncells + 16ull * nfilt + 4096; }

// `fixed` holds one attribute slice (`slice_bytes`, 0 for XRay); `leaf_bytes` everything a candidate leaf holds (image,
// XrayArgs, seen flag, and 4 B of count plus 4 B of offset per bin).  After the block's images, what the budget leaves goes to
// 4-byte keys or to further slices.  The pruning descent runs before any block and may use all of what `fixed` leaves, 16 B
// per candidate (8 B index + 4 B flag; no block is held meanwhile).
inline XrayPlan s2_xray_plan(uint64_t budget, uint64_t fixed, int depth, int max_g, uint64_t leaf_bytes, uint64_t tile_bytes, uint64_t slice_bytes) {
    XrayPlan p;
    p.max_loc = budget > fixed ? std::max<uint64_t>(1, (budget - fixed) / 16) : 1;
    p.g = xray_block_depth(budget, fixed, depth, max_g, leaf_bytes, tile_bytes);
    if (p.g < 0) return p;
    const uint64_t used = fixed + xray_block_bytes(p.g, depth - p.g, leaf_bytes, tile_bytes);
    const uint64_t rest = budget > used ? budget - used : 0;
    p.key_cap = std::min<uint64_t>(rest / 4, 0xFFFFFFFEull);
    p.attr_leaves = slice_bytes ? 1 + rest / slice_bytes : 0;
    return p;
}

}  // namespace pcv
