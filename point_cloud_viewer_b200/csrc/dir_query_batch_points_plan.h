// dir_query_batch_points_plan.h — host-only planning of the batched point queries that return their points straight from
// octree and S2 directories (pcv_octree_dir_query_batch_points_device and its cell-union and S2 forms,
// dir_query_batch_points.inl).  No CUDA: tests compile it with g++.
//
//   dbp_work_tiles:  the work tiles of a batch (every visited node's tiles once per visiting location), the per-tile state the
//                    call keeps on the device for all of them
//   dbp_tile_dests:  from every work tile's survivor count, the output position of its first survivor
#pragma once
#include <cstdint>
#include <functional>
#include <vector>

#include "dir_query_plan.h"

namespace pcv {

// Bytes of one work tile's destination in a chunk's tables (u64), and of its survivor count held for the whole call (u32).
constexpr uint64_t kDbpTileDest = 8;
constexpr uint64_t kDbpTileCount = 4;
// The location bits of a work tile's location field (the top bit marks a node every point of which passes the point test).
constexpr uint32_t kDbpLocMask = 0x7FFFFFFFu;

// Work tiles of the visited nodes: ceil(n / kDirTile) per node and visiting location (info(node).mult).
inline uint64_t dbp_work_tiles(const std::vector<uint32_t>& visit, const std::function<DirPlanNode(uint32_t)>& info) {
    uint64_t t = 0;
    for (uint32_t v : visit) {
        const DirPlanNode d = info(v);
        t += (d.n + kDirTile - 1) / kDirTile * d.mult;
    }
    return t;
}

// The destinations of every work tile of a batch, in call order: the chunks in order, each chunk's tiles in its table order
// (dir_chunk_tiles over the pairs sorted by node).  cnt[t]: tile t's survivors; off[l]: the first output position of location l.
// Tile t goes to its location's position after every earlier tile of that location: the chunks follow the visited nodes in
// node-index order and cut a node only at tile boundaries, and inside a chunk a piece's tiles are grouped by location in file
// order, so a location's tiles arrive in (node, point) order - the order its single-location query streams them in.
// Returns the number of tiles.
inline uint64_t dbp_tile_dests(const std::vector<DirChunk>& chunks, const std::vector<uint32_t>& pair_loc, const std::vector<uint64_t>& pair_begin,
                               const uint32_t* cnt, const uint64_t* off, uint32_t nloc, uint64_t* dest) {
    std::vector<uint64_t> run(off, off + nloc);
    uint64_t t = 0;
    for (const DirChunk& ch : chunks)
        dir_chunk_tiles(ch, &pair_loc, &pair_begin, nullptr, [&](uint32_t, uint32_t loc, uint32_t, uint32_t) {
            uint64_t& r = run[loc & kDbpLocMask];
            dest[t] = r;
            r += cnt[t];
            ++t;
        });
    return t;
}

}  // namespace pcv
