// xray_dir_plan.h — host-only planning of the X-ray quadtree built straight from an on-disk octree (xray_dir.inl; no CUDA:
// the CPU tests compile it with g++).
//   octree_nodes_from_meta: meta.pb's nodes -> the node table pcv_octree_load_dir builds (no node file is read)
//   layout_nodes:           the point and position offsets of a node table (or a subset of it) in load_dir's layout
//   octree_children:        the 8 children of every node in that table
//   xray_window:            the nodes a block of leaves can meet: descend from the octree root while the SAT test is not Out
//   xray_window_size:       what one window takes in device memory (arrays, query tables, the attribute pass flags)
//   xray_windows_size:      what the windows of one block over several directories take together
//   xray_block_location:    a block's location, widened by the pruning margin
//   xray_occupancy_*:       the occupancy pass's work list of (directory, node) pairs, its device chunk and the chunks
//   xray_dir_block_depth:   the block depth from the budget, the images and the largest window of the occupied blocks
#pragma once
#include <algorithm>
#include <cstdint>
#include <functional>
#include <vector>

#include "chain.h"
#include "disk_io.hpp"
#include "geometry_host.hpp"
#include "xray_plan.h"
#include "xray_pyramid.h"

namespace pcv {

// pcv_octree_load_dir's layout of `nodes`, in table order: points node-contiguous, every node's positions 16-byte aligned.
inline void layout_nodes(std::vector<pcv_node_meta>& nodes, uint64_t& npoints, uint64_t& xyz_bytes) {
    uint64_t poff = 0, boff = 0;
    for (pcv_node_meta& m : nodes) {
        boff = (boff + 15) & ~15ull;
        m.point_offset = poff;
        m.xyz_byte_offset = boff;
        poff += (uint64_t)m.num_points;
        boff += (uint64_t)m.num_points * 3 * (uint64_t)enc_bytes(m.position_encoding);
    }
    npoints = poff;
    xyz_bytes = boff;
}

// The node table of an octree directory as pcv_octree_load_dir lays it out: sorted by NodeId, cubes from the bounding cube
// (node.rs:157-172), layout_nodes' offsets.  False: an invalid position encoding.
inline bool octree_nodes_from_meta(const MetaHeader& h, std::vector<ParsedNode> pn, double bmin[3], double bmax[3], std::vector<pcv_node_meta>& nodes,
                                   uint64_t& npoints, uint64_t& xyz_bytes) {
    typedef unsigned __int128 id128;
    std::sort(pn.begin(), pn.end(), [](const ParsedNode& a, const ParsedNode& b) { return a.hi != b.hi ? a.hi < b.hi : a.lo < b.lo; });
    for (int a = 0; a < 3; ++a) {
        bmin[a] = std::fmin(h.bbox_min[a], h.bbox_max[a]);
        bmax[a] = std::fmax(h.bbox_min[a], h.bbox_max[a]);
    }
    const double E = std::fmax(std::fmax(bmax[0] - bmin[0], bmax[1] - bmin[1]), bmax[2] - bmin[2]);
    nodes.clear();
    nodes.reserve(pn.size());
    for (const auto& p : pn) {
        pcv_node_meta m{};
        m.id_high = p.hi;
        m.id_low = p.lo;
        m.num_points = p.num_points;
        m.position_encoding = p.enc;
        if (p.enc < 1 || p.enc > 4) return false;
        const id128 id = ((id128)p.hi << 64) | p.lo;
        m.level = (int)(id >> 120);
        double e = E, mn[3] = {bmin[0], bmin[1], bmin[2]};
        for (int lvl = m.level - 1; lvl >= 0; --lvl) {  // node.rs:157-172
            e /= 2.;
            const unsigned ci = (unsigned)((id >> (3 * lvl)) & 7);
            mn[0] += (double)((ci >> 2) & 1) * e;
            mn[1] += (double)((ci >> 1) & 1) * e;
            mn[2] += (double)(ci & 1) * e;
        }
        for (int a = 0; a < 3; ++a) m.cube_min[a] = mn[a];
        m.cube_edge = e;
        nodes.push_back(m);
    }
    layout_nodes(nodes, npoints, xyz_bytes);
    return true;
}

// children[8 i + k]: index of child k of node i in `nodes` (sorted by NodeId), -1 if absent.
inline std::vector<int32_t> octree_children(const std::vector<pcv_node_meta>& nodes) {
    typedef unsigned __int128 id128;
    std::vector<int32_t> ch(nodes.size() * 8, -1);
    for (size_t i = 0; i < nodes.size(); ++i) {
        if (nodes[i].level == 0) continue;
        const id128 id = ((id128)nodes[i].id_high << 64) | nodes[i].id_low;
        const id128 idx = id & ((((id128)1) << 120) - 1);
        const id128 pid = ((id128)(nodes[i].level - 1) << 120) | (idx >> 3);  // node.rs:136-144
        const int p = find_node(nodes, (uint64_t)(pid >> 64), (uint64_t)pid);
        if (p >= 0) ch[(size_t)p * 8 + (size_t)(idx & 7)] = (int32_t)i;
    }
    return ch;
}

// sat() of sat.rs:174-194 with A = the location and B = the node cube (min m, edge e): sat_cube of query.cuh on the host.
inline bool sat_cube_out(const QueryGeom& g, const double m[3], double e) {
    if (g.kind == PCV_LOC_ALL) return false;
    const double mx[3] = {m[0] + e, m[1] + e, m[2] + e};
    for (int k = 0; k < g.naxes; ++k) {
        const double* ax = geom_axis(g, k);
        double alo = 1.7976931348623157e308, ahi = -1.7976931348623157e308, blo = alo, bhi = ahi;
        for (int i = 0; i < 8; ++i) {
            const double pa = g.corners[i][0] * ax[0] + g.corners[i][1] * ax[1] + g.corners[i][2] * ax[2];
            alo = std::fmin(alo, pa);
            ahi = std::fmax(ahi, pa);
            const double cx = (i & 1) ? mx[0] : m[0], cy = (i & 2) ? mx[1] : m[1], cz = (i & 4) ? mx[2] : m[2];
            const double pb = cx * ax[0] + cy * ax[1] + cz * ax[2];
            blo = std::fmin(blo, pb);
            bhi = std::fmax(bhi, pb);
        }
        if (blo > ahi || bhi < alo) return true;
    }
    return false;
}

// The window of a location: every node whose cube and whose ancestors' cubes are not Out, found by descending from the root
// (nodes_in_location's BFS semantics).  Sorted node indices, closed under ancestors: a valid octree on its own.
inline std::vector<uint32_t> xray_window(const std::vector<pcv_node_meta>& nodes, const std::vector<int32_t>& children, const QueryGeom& g) {
    std::vector<uint32_t> out, stack;
    if (nodes.empty() || nodes[0].level != 0) return out;
    stack.push_back(0);
    while (!stack.empty()) {
        const uint32_t i = stack.back();
        stack.pop_back();
        if (sat_cube_out(g, nodes[i].cube_min, nodes[i].cube_edge)) continue;
        out.push_back(i);
        for (int k = 0; k < 8; ++k)
            if (children[(size_t)i * 8 + k] >= 0) stack.push_back((uint32_t)children[(size_t)i * 8 + k]);
    }
    std::sort(out.begin(), out.end());
    return out;
}

// Device bytes per window node besides its points: the query node (64 bytes), its 8 children (32), the attribute strategies'
// relation and pass flags (2).
constexpr uint64_t kWindowNodeBytes = 64 + 32 + 2;
struct WindowSize {
    uint64_t bytes = 0, points = 0, xyz_bytes = 0;
};
// What one window takes on the device: its positions laid out as load_dir lays them (16-byte aligned, + 32 bytes of slack for
// the kernels' 16-byte staging), colours, intensities if the directory has them, and the per-node tables.
inline WindowSize xray_window_size(const std::vector<pcv_node_meta>& nodes, const std::vector<uint32_t>& win, bool has_intensity) {
    WindowSize s;
    for (uint32_t i : win) {
        s.xyz_bytes = (s.xyz_bytes + 15) & ~15ull;
        s.xyz_bytes += (uint64_t)nodes[i].num_points * 3 * (uint64_t)enc_bytes(nodes[i].position_encoding);
        s.points += (uint64_t)nodes[i].num_points;
    }
    s.bytes = s.xyz_bytes + 32 + std::max<uint64_t>(3 * s.points, 16) + (has_intensity ? 4 * s.points : 0) + kWindowNodeBytes * win.size();
    return s;
}

// The location of block `bidx` at quadtree level B: its rect (the quad_rect_of recurrence) over the z range of the box, every
// side widened by `margin`, as an Aabb or, under query_from_global, the Obb xray_location builds for a leaf.  A leaf's rect comes
// from the same recurrence, so it lies within a few ulps of its block's rect; the margin is far above that.
inline pcv_location xray_block_location(const QuadRect& rect, int B, uint64_t bidx, const double bmin[3], const double bmax[3], double margin,
                                        const double* qfg) {
    const QuadRect r = quad_rect_of(QuadId{(uint8_t)B, bidx}, rect);
    const double tmin[3] = {r.min_x - margin, r.min_y - margin, bmin[2] - margin};
    const double tmax[3] = {r.min_x + r.edge + margin, r.min_y + r.edge + margin, bmax[2] + margin};
    return xray_location(tmin, tmax, qfg);
}

// The windows of one block over several directories (windows[k]: directory k's, possibly empty), loaded together: the sum of
// xray_window_size over the non-empty ones, and the largest one's points and directory (max_dir).
struct WindowsSize {
    uint64_t bytes = 0, points = 0, max_points = 0;
    uint32_t max_dir = 0;
};
inline WindowsSize xray_windows_size(const std::vector<const std::vector<pcv_node_meta>*>& tables, const std::vector<char>& has_intensity,
                                     const std::vector<std::vector<uint32_t>>& windows) {
    WindowsSize s;
    for (size_t k = 0; k < windows.size(); ++k) {
        if (windows[k].empty()) continue;
        const WindowSize w = xray_window_size(*tables[k], windows[k], has_intensity[k] != 0);
        s.bytes += w.bytes;
        s.points += w.points;
        if (w.points > s.max_points) s.max_points = w.points, s.max_dir = (uint32_t)k;
    }
    return s;
}

// ---- the occupancy pass over the nodes with points of every directory -------------------------------------------------------
// One node of one of the directories.
struct DirNode {
    uint32_t dir, node;
};
// The pass's work list: every node with points, directory by directory in list order, each in table order; *largest: the
// largest node's position bytes.
inline std::vector<DirNode> xray_occupancy_work(const std::vector<const std::vector<pcv_node_meta>*>& tables, uint64_t* largest) {
    std::vector<DirNode> work;
    *largest = 0;
    for (uint32_t k = 0; k < (uint32_t)tables.size(); ++k)
        for (uint32_t i = 0; i < (uint32_t)tables[k]->size(); ++i) {
            const pcv_node_meta& m = (*tables[k])[i];
            if (m.num_points <= 0) continue;
            work.push_back(DirNode{k, i});
            *largest = std::max<uint64_t>(*largest, (uint64_t)m.num_points * 3 * (uint64_t)enc_bytes(m.position_encoding));
        }
    return work;
}
// Its device chunk: `chunk` position bytes (min(64 MiB, budget / 8), at least the largest node), at most `node_cap` nodes and
// `tile_cap` work tiles of `tile_points` points; `need`: those arrays (64 B per query node, 16 B per tile) besides `set_bytes`
// of occupancy set.
struct OccupancyPlan {
    uint64_t chunk = 0, node_cap = 0, tile_cap = 0, need = 0;
};
inline OccupancyPlan xray_occupancy_plan(uint64_t budget, uint64_t largest, uint32_t tile_points, uint64_t set_bytes) {
    OccupancyPlan p;
    p.chunk = std::max<uint64_t>(std::min<uint64_t>(64ull << 20, budget / 8), ((largest + 15) & ~15ull) + 16);
    p.node_cap = std::max<uint64_t>(64, p.chunk / 512);
    p.tile_cap = p.node_cap + p.chunk / (3 * (uint64_t)tile_points) + 1;
    p.need = p.chunk + p.node_cap * 64 + p.tile_cap * 16 + set_bytes;
    return p;
}
// The chunks of the work list: runs of consecutive entries, directories mixed, whose 16-byte aligned positions fit `chunk`
// and that hold at most node_cap nodes and tile_cap tiles.  The chunk starts plus an end sentinel.
inline std::vector<size_t> xray_occupancy_chunks(const std::vector<const std::vector<pcv_node_meta>*>& tables, const std::vector<DirNode>& work,
                                                 const OccupancyPlan& p, uint32_t tile_points) {
    std::vector<size_t> starts{0};
    for (size_t k = 0, bytes = 0, nt = 0; k < work.size(); ++k) {
        const pcv_node_meta& m = (*tables[work[k].dir])[work[k].node];
        const uint64_t b = ((uint64_t)m.num_points * 3 * (uint64_t)enc_bytes(m.position_encoding) + 15) & ~15ull;
        const uint64_t t = ((uint64_t)m.num_points + tile_points - 1) / tile_points;
        if (k > starts.back() && (bytes + b > p.chunk || k - starts.back() >= p.node_cap || nt + t > p.tile_cap)) starts.push_back(k), bytes = 0, nt = 0;
        bytes += b, nt += t;
    }
    starts.push_back(work.size());
    return starts;
}

// Block depth g of a directory driver: the largest g <= g_max whose plan `fits(g, w)` holds the block images, the leaf
// producer's working set and the largest window over the occupied blocks at level deepest - g (`window_max(g)`, UINT64_MAX:
// a window too large to hold).  A smaller g means a deeper block level and smaller windows.  -1: not even g = 0 fits.
inline int xray_dir_block_depth(int g_max, const std::function<uint64_t(int)>& window_max, const std::function<bool(int, uint64_t)>& fits) {
    for (int g = g_max; g >= 0; --g) {
        const uint64_t w = window_max(g);
        if (w != UINT64_MAX && fits(g, w)) return g;
    }
    return -1;
}
// ... for octree directories: the block images, the node selection and the windows fit the budget besides `fixed`; `clouds`
// directories with points keep their work lists of a key batch at once (xray_pair_bytes).
inline int xray_dir_block_depth(uint64_t budget, uint64_t fixed, int depth, int g_max, uint64_t leaf_bytes, uint64_t tile_bytes, uint64_t per_loc,
                                const std::function<uint64_t(int)>& window_max, uint32_t clouds = 1) {
    return xray_dir_block_depth(g_max, window_max, [&](int g, uint64_t w) {
        return xray_octree_plan(budget, fixed, w, depth, g, per_loc, leaf_bytes, tile_bytes, clouds).g == g;
    });
}

}  // namespace pcv
