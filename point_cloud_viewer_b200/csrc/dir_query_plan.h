// dir_query_plan.h — host-only planning of queries straight from an on-disk octree (dir_query.inl; no CUDA: the CPU tests
// compile it with g++).
//   dir_chunk_bytes:  what one chunk takes in device memory (inputs, chunk-local tables, survivors)
//   plan_dir_chunks:  the visited nodes, in visit order, cut into chunks of pieces at kDirTile boundaries under a byte bound
//   dir_chunk_tiles:  the work tiles of one chunk, in the order its tile table lists them
//   nodes_blob_layout / nodes_blob_header: the /nodes_data reply of pcv_nodes_data_blob, laid out from the node table alone
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <functional>
#include <vector>

#include "../../include/pcv.h"
#include "chain.h"
#include "disk_io.hpp"

namespace pcv {

constexpr uint32_t kDirTile = 2048;    // == kQueryTile (query.cuh): pieces start at multiples of it inside their node
constexpr uint64_t kDirAlign = 256;    // every array of a chunk's device arena starts at a multiple of it
constexpr uint64_t kDirSurvivor = 24 + 3 + 4 + 8;  // one stored survivor: xyz f64, rgb, intensity, u64 slot

inline uint64_t dir_align(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

// Points [first, first + count) of node `node`.
struct DirPiece {
    uint32_t node;
    uint64_t first, count;
};
struct DirChunk {
    std::vector<DirPiece> pieces;
    uint64_t points = 0, xyz_bytes = 0, tiles = 0;  // xyz_bytes: every piece 16-byte aligned; tiles: work tiles (pairs x tiles)
};
// What the planner needs of one visited node: its points, bytes per coordinate, and how many locations visit it (1 for a
// single-location query; each visiting location gets its own work tiles).
struct DirPlanNode {
    uint64_t n;
    uint32_t bpc;
    uint32_t mult;
};

// Device bytes of one chunk: positions (+ 32 bytes of slack: the staged loads read whole 16-byte granules), colours, intensities
// when the directory has them, one QNode (64) + slot base (8) per piece, one QTile (16) + keep count (4) per work tile, the total,
// and with `store` the survivors of every point.
inline uint64_t dir_chunk_bytes(uint64_t points, uint64_t xyz_bytes, uint64_t pieces, uint64_t tiles, bool has_i, bool store) {
    const uint64_t A = kDirAlign;
    uint64_t b = dir_align(xyz_bytes + 32, A) + dir_align(3 * points, A) + (has_i ? dir_align(4 * points, A) : 0);
    b += dir_align(64 * pieces, A) + dir_align(8 * pieces, A) + dir_align(16 * tiles, A) + dir_align(4 * tiles, A) + A;
    if (store) b += dir_align(24 * points, A) + dir_align(3 * points, A) + dir_align(4 * points, A) + dir_align(8 * points, A);
    return b;
}
// The smallest chunk any query needs: one tile at the widest encoding, with its survivors.
inline uint64_t dir_min_chunk_bytes() { return dir_chunk_bytes(kDirTile, (uint64_t)kDirTile * 24, 1, 1, true, true); }

// Cuts the visited nodes (in visit order) into chunks whose dir_chunk_bytes, plus `tile_bytes` more per work tile, stays within
// `chunk_budget`.  Each piece takes as many whole tiles of its node as fit (the node's last tile may be short), so a node larger
// than a chunk is split across consecutive chunks.  False: a single tile of some node does not fit an empty chunk.
inline bool plan_dir_chunks(const std::vector<uint32_t>& visit, const std::function<DirPlanNode(uint32_t)>& info, bool has_i, bool store,
                            uint64_t chunk_budget, std::vector<DirChunk>& out, uint64_t tile_bytes = 0) {
    out.clear();
    DirChunk cur;
    auto cost_with = [&](const DirChunk& c, const DirPlanNode& d, uint64_t cnt) {
        const uint64_t tiles = (cnt + kDirTile - 1) / kDirTile * d.mult;
        return dir_chunk_bytes(c.points + cnt, c.xyz_bytes + dir_align(cnt * 3 * d.bpc, 16), c.pieces.size() + 1, c.tiles + tiles, has_i, store) +
               (tile_bytes ? dir_align(tile_bytes * (c.tiles + tiles), kDirAlign) : 0);
    };
    for (uint32_t v : visit) {
        const DirPlanNode d = info(v);
        uint64_t first = 0;
        while (first < d.n) {
            const uint64_t left = d.n - first, ntl = (left + kDirTile - 1) / kDirTile;
            uint64_t lo = 0, hi = ntl;  // the most whole tiles that fit: cost is monotone in the tile count
            while (lo < hi) {
                const uint64_t mid = (lo + hi + 1) / 2;
                if (cost_with(cur, d, std::min(left, mid * kDirTile)) <= chunk_budget)
                    lo = mid;
                else
                    hi = mid - 1;
            }
            if (lo == 0) {
                if (cur.pieces.empty()) return false;
                out.push_back(std::move(cur));
                cur = DirChunk();
                continue;
            }
            const uint64_t cnt = std::min(left, lo * kDirTile);
            cur.pieces.push_back(DirPiece{v, first, cnt});
            cur.points += cnt;
            cur.xyz_bytes += dir_align(cnt * 3 * d.bpc, 16);
            cur.tiles += (cnt + kDirTile - 1) / kDirTile * d.mult;
            first += cnt;
        }
    }
    if (!cur.pieces.empty()) out.push_back(std::move(cur));
    return true;
}

// The work tiles of chunk `ch`, in the order of its tile table: per piece k, per location that visits the piece's node - the run
// [(*pair_begin)[node], (*pair_begin)[node + 1]) of *pair_loc (batched form), or the one location (*node_flag)[node] (0 without
// flags) - the piece's tiles in file order.  f(k, location, first point of the tile inside the piece, points of the tile).
template <class F>
inline void dir_chunk_tiles(const DirChunk& ch, const std::vector<uint32_t>* pair_loc, const std::vector<uint64_t>* pair_begin,
                            const std::vector<uint32_t>* node_flag, F&& f) {
    for (size_t k = 0; k < ch.pieces.size(); ++k) {
        const DirPiece& pc = ch.pieces[k];
        const uint64_t lb = pair_begin ? (*pair_begin)[pc.node] : 0, le = pair_begin ? (*pair_begin)[pc.node + 1] : 1;
        const uint32_t loc0 = node_flag ? (*node_flag)[pc.node] : 0u;
        for (uint64_t j = lb; j < le; ++j)
            for (uint64_t t = 0; t < pc.count; t += kDirTile)
                f((uint32_t)k, pair_loc ? (*pair_loc)[j] : loc0, (uint32_t)t, (uint32_t)std::min<uint64_t>(kDirTile, pc.count - t));
    }
}

// ---- /nodes_data reply (octree_web_viewer/src/backend.rs:66-75 pad, :92-165 get_nodes_data), from the node table ----------
struct BlobPart {
    int node;
    uint64_t header_at, xyz_at, xyz_bytes, rgb_at, rgb_bytes;
};
// Per requested node, in request order: a 40-byte header, the node's position bytes, padding, its colour bytes, padding (every
// part padded with zeros to a multiple of 8).  Returns -1, or the first request whose node is unknown or has no points (no files).
inline int64_t nodes_blob_layout(const std::vector<pcv_node_meta>& nodes, const uint64_t* ids_hi_lo, uint32_t num, std::vector<BlobPart>& parts, uint64_t& size) {
    auto pad8 = [](uint64_t v) { return (v + 7) & ~(uint64_t)7; };
    parts.clear();
    size = 0;
    for (uint32_t k = 0; k < num; ++k) {
        const int i = find_node(nodes, ids_hi_lo[2 * k], ids_hi_lo[2 * k + 1]);
        if (i < 0 || nodes[i].num_points == 0) return k;
        const uint64_t n = (uint64_t)nodes[i].num_points;
        BlobPart p{i, size, 0, n * 3 * (uint64_t)enc_bytes(nodes[i].position_encoding), 0, 3 * n};
        size += pad8(8 * 4 + 4 + 1);
        p.xyz_at = size;
        size += pad8(p.xyz_bytes);
        p.rgb_at = size;
        size += pad8(p.rgb_bytes);
        parts.push_back(p);
    }
    return -1;
}
// cube min x, y, z (f64 LE), edge (f64), num_points (u32, `as u32`), bytes per coordinate (u8), 3 zero bytes
inline void nodes_blob_header(const pcv_node_meta& m, uint8_t* h) {
    std::memcpy(h, m.cube_min, 24);
    std::memcpy(h + 24, &m.cube_edge, 8);
    const uint32_t n32 = (uint32_t)m.num_points;
    std::memcpy(h + 32, &n32, 4);
    h[36] = (uint8_t)enc_bytes(m.position_encoding);
    h[37] = h[38] = h[39] = 0;
}

}  // namespace pcv
