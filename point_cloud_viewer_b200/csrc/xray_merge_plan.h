// xray_merge_plan.h — host-only planning of the merge of partial X-ray quadtrees (xray_merge.inl; no CUDA: the CPU tests
// compile it with g++).  From the decoded meta files of the sub-root builds:
//   xray_merge_plan:         validate_and_merge_metadata (xray/src/bin/merge_xray_quadtrees.rs:125-176) - the checks in the
//                            reference's order, the merged rect from Node::parent (quadtree/src/lib.rs:100-120) walked from the
//                            first root up to level 0 - and the parents create_non_leaf_nodes builds (generation.rs:656-682),
//                            in the order of the depth-first walk that builds them
//   xray_merge_device_bytes: what that walk holds on the device at most
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "xray_plan.h"
#include "xray_png.hpp"
#include "xray_pyramid.h"

namespace pcv {

struct XrayMergePlan {
    int code = PCV_OK;    // PCV_OK, or the error of the first check that fails
    std::string error;    // its message
    uint32_t metas = 0, empty = 0;
    uint32_t root_level = 0, deepest_level = 0, tile_size = 0;
    QuadRect rect{};                                   // the merged quadtree's bounding rect (level 0)
    std::vector<uint64_t> roots;                       // the sub-roots' indices at root_level, sorted
    std::vector<size_t> root_meta;                     // [root] the meta it came from
    std::vector<std::pair<uint32_t, uint64_t>> walk;   // the parents, each after its children, siblings in index order
    std::vector<std::pair<uint32_t, uint64_t>> nodes;  // the merged node set: every meta's nodes and the parents, sorted
};

// Device bytes of the depth-first walk over sub-roots at level L with T px tiles: the finished children waiting for their
// parent (at most 4 on each of the levels L down to 1), one output tile, the vertically reduced mosaic and the Lanczos3 taps
// of 2T -> T (each tap array at least one element, as Scratch::upload allocates).  0 when L = 0: nothing is built.
inline uint64_t xray_merge_device_bytes(uint32_t L, uint32_t T) {
    if (L == 0) return 0;
    const uint64_t tile = (uint64_t)T * T * 4;
    const ResampleTable tb = make_lanczos3_table(2 * T, T);
    auto arr = [](size_t n, size_t sz) { return (uint64_t)std::max<size_t>(n, 1) * sz; };
    const uint64_t taps = arr(tb.left.size(), 4) + arr(tb.first.size(), 4) + arr(tb.count.size(), 4) + arr(tb.sum.size(), 4) + arr(tb.w.size(), 4);
    return (4ull * L + 1) * tile + 2ull * T * T * 4 + taps;
}

// `metas` in the order the merge reads them: input directories in argument order, each one's meta files sorted by name.
inline XrayMergePlan xray_merge_plan(const std::vector<XrayMetaData>& metas) {
    XrayMergePlan p;
    auto err = [&](int code, const std::string& msg) {
        p.code = code;
        p.error = msg;
        return p;
    };
    p.metas = (uint32_t)metas.size();
    if (metas.empty()) return err(PCV_ERR_NOT_FOUND, "No subquadtrees meta files found.");
    // Meta::get_root_node (lib.rs:139-147): the node of least level; among several at that level the least index (the
    // reference takes whichever its hash set yields first)
    std::vector<std::pair<uint32_t, uint64_t>> root_ids;
    std::vector<size_t> first_of;
    for (size_t k = 0; k < metas.size(); ++k) {
        if (metas[k].nodes.empty()) {
            p.empty++;
            continue;
        }
        root_ids.push_back(*std::min_element(metas[k].nodes.begin(), metas[k].nodes.end()));
        first_of.push_back(k);
    }
    if (root_ids.empty()) return err(PCV_ERR_INVALID, "All subquadtress are empty.");
    std::vector<std::pair<uint32_t, uint64_t>> sorted = root_ids;
    std::sort(sorted.begin(), sorted.end());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) return err(PCV_ERR_INVALID, "Not all roots are unique.");
    if (sorted.front().first != sorted.back().first) return err(PCV_ERR_INVALID, "Not all roots have the same level.");
    for (const XrayMetaData& m : metas)
        if (m.deepest_level != metas[0].deepest_level) return err(PCV_ERR_INVALID, "Not all meta files have the same deepest level.");
    for (const XrayMetaData& m : metas)
        if (m.tile_size != metas[0].tile_size) return err(PCV_ERR_INVALID, "Not all meta files have the same tile size.");
    p.root_level = sorted.front().first;
    p.deepest_level = metas[0].deepest_level;
    p.tile_size = metas[0].tile_size;
    // beyond the reference: what a quadtree NodeId and the tiles can hold
    if (p.root_level > 31 || p.deepest_level > 32)
        return err(PCV_ERR_UNSUPPORTED, "root level " + std::to_string(p.root_level) + ", deepest level " + std::to_string(p.deepest_level) +
                                            ": a quadtree NodeId holds at most 32 levels, and the roots lie above the deepest");
    for (const auto& r : sorted)
        if (r.first < 32 && (r.second >> (2 * r.first)) != 0) return err(PCV_ERR_INVALID, "root " + std::to_string(r.second) + " lies outside level " + std::to_string(r.first));
    if (p.tile_size == 0 || p.tile_size > 32768) return err(PCV_ERR_UNSUPPORTED, "tile size " + std::to_string(p.tile_size));
    // the merged rect: Node::parent from the first root up to level 0 (bit 0 of the child index: y, bit 1: x)
    const XrayMetaData& m0 = metas[first_of[0]];
    QuadRect r{m0.min_x, m0.min_y, m0.edge};
    for (uint32_t l = root_ids[0].first; l > 0; --l) {
        const uint64_t ci = (root_ids[0].second >> (2 * (root_ids[0].first - l))) & 3;
        if (ci & 1) r.min_y -= r.edge;
        if (ci & 2) r.min_x -= r.edge;
        r.edge *= 2.;
    }
    p.rect = r;
    std::vector<size_t> order(root_ids.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return root_ids[a].second < root_ids[b].second; });
    for (size_t i : order) p.roots.push_back(root_ids[i].second), p.root_meta.push_back(first_of[i]);
    for (const auto& nd : xray_post_order(p.roots, (int)p.root_level))
        if (nd.first > 0) p.walk.emplace_back(p.root_level - (uint32_t)nd.first, nd.second);
    for (const XrayMetaData& m : metas) p.nodes.insert(p.nodes.end(), m.nodes.begin(), m.nodes.end());
    p.nodes.insert(p.nodes.end(), p.walk.begin(), p.walk.end());
    std::sort(p.nodes.begin(), p.nodes.end());
    p.nodes.erase(std::unique(p.nodes.begin(), p.nodes.end()), p.nodes.end());
    return p;
}

}  // namespace pcv
