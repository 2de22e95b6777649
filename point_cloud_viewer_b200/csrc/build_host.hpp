// build_host.hpp — host orchestration of the GPU octree build (backend agnostic).
//
// Replaces src/octree/generation.rs:289-403 (build_octree) with a different algorithm that yields the
// same tree, the same per-node point order and the same stored position codes:
//
//   split phase    the reference's recursive 8-way file split (generation.rs:58-193) becomes a
//                  top-down, level-synchronous stable multi-way partition: each pass resolves two octree
//                  levels for every point that still sits in a node with > MAX_POINTS_PER_NODE points
//                  (digit histogram per tile -> per-digit prefix over tiles -> a planner kernel decides
//                  leaf/split for the 8 + 64 descendants -> stable partition into the next pass's
//                  segments or into the leaf arena, all enqueued without a host round trip).  The
//                  per-point digits come from the re-quantising descent in chain.h, computed one pass
//                  ahead and carried with the record, so node membership is bit-identical and every
//                  level of the chain is encoded exactly once.
//   subsample      the level-by-level rewrite (generation.rs:195-253,335-387) is replaced by its closed
//                  form: a point at rank j of a node X with parent P moves up iff j % 8 == 0, to rank
//                  off(X in P) + j/8; otherwise it stays at slot j - j/8 - 1.  `place` walks each leaf
//                  point up, re-encoding through every cube it passes (same DEC/ENC chain as the
//                  reference's rewrites), and writes it to its final node-contiguous slot.
//
// The Backend interface is implemented by the CUDA kernels (kernels_build.cuh).  A second, test-only
// implementation lives under tests/ to exercise this host logic without a GPU; the shipped library
// contains only the CUDA one.
#pragma once
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "chain.h"

namespace pcv {

typedef unsigned __int128 u128;

struct PointsView {  // device pointers
    const double* x;
    const double* y;
    const double* z;
    uint64_t stride;
    const uint8_t* rgb;
    const float* intensity;
    uint64_t n;
};

// ---- structures shared with the kernels ---------------------------------------------------------
struct RecN {  // narrow partition record: codes of U8/U16/F32 levels
    uint32_t c[3];
    uint32_t idx;
};
struct RecW {  // wide record: used for the whole build when any level >= 1 is Float64 encoded
    uint64_t c[3];
    uint32_t idx;
    uint32_t pad;
};
struct TileDesc {
    uint64_t start;   // first record of the tile
    uint32_t count;   // <= kTilePoints
    uint32_t active;  // index into the pass's active-node array
};
struct ActiveDesc {
    double m[3];
    double e;
    uint64_t start, count;  // the node's segment in the pass's input records
    uint32_t chunk_begin, nchunks;
    uint32_t tile_begin;    // first tile of the node (tiles never straddle nodes)
    uint32_t node;          // index into the node table
};
struct ChunkDesc {
    uint32_t tile_begin, ntiles;
    uint32_t active;
    uint32_t first;  // 1 if first chunk of its node
};
struct BucketDesc {
    uint64_t dest;    // first record of the bucket in its destination buffer
    uint16_t b0, b1;  // digit range [b0,b1) it collects (contiguous: a whole sub-tree); b1 == 0: unused entry
    uint8_t keep;     // 1..G: which level's codes the destination stores
    uint8_t kind;     // 0 = next pass segment, 1 = leaf arena
    uint16_t owner;   // fused exchange pass only: 1 + rank whose buffers the bucket lives in (0: this context's)
};
// Fused exchange pass (sharded build): the first partition pass of a SENDER writes every bucket straight into its owner's
// buffers - as mapped in the sender's address space (own memory or CUDA-IPC peer memory).
struct RemoteBufs {
    void* rec_next;
    uint32_t* col_next;   // wide records only (narrow ones carry the colour in the record)
    uint8_t* dig_next;
    void* arena;
    uint32_t* col_arena;
    float* intensity;     // indexed by slot, or null
};
// Node table entry, appended on the device by the planner (parents before children).
struct DevNode {
    uint64_t index_hi, index_lo;  // octal path index (u128, node.rs:120-125)
    double m[3];
    uint64_t count;      // points routed into the node by the split phase
    uint64_t arena_off;  // leaves: first record in the leaf arena
    int32_t level, parent;
    int32_t leaf, pad;
};
struct DNode {
    double m[3];
    double e;
    double ry;                // RN(1/e)
    uint64_t off_in_parent;   // sum_{k'<k} ceil(n(P.k')/8)
    uint64_t out_point_off;
    uint64_t out_xyz_off;     // bytes
    uint64_t arena_off, count;  // leaves (and collectors in the top assembly): segment of the leaf arena
    int32_t parent;           // -1 for the root
    int32_t enc;
};
struct LeafTile {
    uint64_t arena_start;
    uint64_t j0;
    uint32_t node;
    uint32_t count;
};

constexpr uint32_t kTilePoints = 1792;   // partition tile: 8 warps x 7 sub-rounds of 32 (kernels_build.cuh)
constexpr uint32_t kChunkTiles = 256;    // tiles per scan chunk
constexpr uint32_t kPlaceTile = 2048;    // place tile
constexpr int kMaxPasses = kMaxLevels;   // a pass resolves at least one level

// Device-resident bookkeeping of one build: written by the planner kernel, read by every kernel of the following pass
// (grid sizes are upper bounds; blocks beyond the live counts exit), read back by the host once after the last pass.
struct PassState {
    uint32_t nactive, ntiles, nchunks, pad;
    uint64_t npoints;      // points partitioned by this pass
};
struct BuildState {
    uint32_t nnodes;
    int32_t error;         // 0, or a BuildError code raised on the device (kErr*)
    int32_t plan_error, pad0;
    uint64_t arena_used;
    uint32_t deepest_level, pad;
    // totals of the subsample plan (finish_layout): what the host needs to size the outputs and launch the placement
    uint32_t nleaves, place_tiles;
    uint64_t out_points, xyz_bytes, algo_xyz;
    PassState pass[kMaxPasses + 1];
};
enum : int32_t { kErrHistMismatch = 1, kErrTooDeep = 2, kErrCapacity = 3 };

// Multi-GPU sharding (SURVEY 8e): this context builds only the sub-trees below some level-k cells.  `counts` holds the
// GLOBAL point counts of every cell of levels 1..k (level j at offset (8^j - 8) / 7), so that nodes above level k take
// the same split decision on every rank; nodes of level k-1 ("collectors") keep the every-8th points of their local
// children (encoded in the collector's cube, in child order) for the top-of-tree assembly on one rank.
struct ShardSpec {
    int k = 0;
    const uint64_t* counts = nullptr;
    PCV_HD static size_t level_offset(int level) { return (((size_t)1 << (3 * level)) - 8) / 7; }
    uint64_t count_at(int level, uint64_t index) const { return counts[level_offset(level) + index]; }
};

// The split phase runs "one pass ahead" (DESIGN 3): a record entering the pass of a node A at level L already holds the
// point's codes at level L+1 (inside the child cube it falls into) plus the digits of levels L+1..L+G, computed while the
// previous pass (or the ingest kernel) still had the decoded position in registers.  The pass therefore ranks by digit
// without any arithmetic, and only then - in destination order - finishes the codes each destination stores and, for
// points that continue, runs the next pass's descent.  Every level of the re-quantising chain is encoded exactly once.
// Running totals of one pass of the planner (plan_active below).
struct PlanRun {
    uint32_t nodes, actives, tiles, chunks;
    uint64_t next_pts, arena_pts;
};

struct IngestArgs {
    PointsView pts;
    void* rec_out;       // codes at level 1 (RecN / RecW), idx = input position
    uint32_t* col_out;   // r | g << 8 | b << 16
    uint8_t* dig_out;    // digit of level 1 (G0 == 1) or levels 1,2 (d1 << 3 | d2)
    int G0;              // levels the first pass resolves
    bool wide;
    uint32_t ntiles;
    LevelTable lv;
    double root_min[3];
};

struct PassArgs {
    int pass, level, G, nbins;  // level L of the pass's active nodes; G = levels it resolves (1 or 2); nbins = 8^G
    int Gn;                     // levels the following pass resolves (0: there is none - every destination is a leaf)
    bool wide;
    bool rec_has_col;  // first pass over exchanged (narrow) records: a record's 4th word is the packed colour, its idx is its position
    bool holes;        // planner: leaf buckets advance the next-pass offset as well, so that a record's position in the next pass's
                       // input is its slot in cell-major order over ALL buckets (fused exchange pass: idx == position is implied)
    const RemoteBufs* remote;  // fused exchange pass (device array indexed by BucketDesc::owner - 1), else null
    const float* int_in;       // fused exchange pass: the sender's intensities by input position, or null
    // per-pass level constants as plain scalars (a dynamically indexed read of `lv` in a kernel is an indexed constant load
    // per use): levels L+1, L+2 and, for records that continue, the node level Lb = L+G and its child level
    double e1, e2, ry2, eb, eh, ryh;
    int enc1, enc2, ench, fast;
    const void* rec_in;
    void* rec_next;
    void* arena;
    // colour travels with the records (packed r | g<<8 | b<<16) so the final placement does not gather it
    const uint32_t* col_in;
    uint32_t* col_next;
    uint32_t* col_arena;
    const uint8_t* dig_in;
    uint8_t* dig_next;
    BuildState* st;
    const ActiveDesc* active;
    ActiveDesc* active_next;
    const ChunkDesc* chunks;
    ChunkDesc* chunks_next;
    uint32_t* tile_active;  // [tiles] active node of every tile (from the scan chunks)
    uint32_t* tile_counts;  // [tiles][nbins]; after scan: exclusive prefix over the node's tiles
    uint32_t* chunk_sums;   // [chunks][nbins]
    uint64_t* node_bins;    // [active][nbins]
    BucketDesc* buckets;    // [active][nbins]
    PlanRun* plan_runs;  // [active] per-node demand, then bases (device backends that plan in several kernels)
    DevNode* nodes;
    int32_t* children;  // [cap_nodes][8] index of every node's children, -1 if absent (read by the subsample plan); may be null
    uint32_t cap_active, cap_nodes, cap_tiles, cap_chunks;
    // split rule (generation.rs:128-150) + sharding
    uint64_t max_points;
    double resolution;
    int shard_k;
    const uint64_t* shard_counts;  // device copy of ShardSpec::counts
    LevelTable lv;
};

struct PlaceArgs {
    bool wide;
    PointsView pts;
    const void* arena;
    const uint32_t* col_arena;
    int fast;  // LevelTable::fast
    const DNode* d_nodes;
    const uint32_t* d_leaf_tile_begin;  // [nleaves + 1] first tile of every leaf
    const uint32_t* d_leaf_node;        // [nleaves] index into d_nodes
    uint32_t nleaves;
    uint32_t ntiles;
    uint64_t npoints, xyz_bytes;
    const LeafTile* tiles = nullptr;  // device backends: [ntiles] descriptor of every tile, written by the backend before the placement
    uint8_t* out_xyz;
    uint8_t* out_rgb;
    float* out_intensity;
    uint32_t* out_src;
};

// A tile's node by binary search over the per-node first-tile index (the active-list lookup and the CPU test backend; the
// CUDA placement materialises its tile descriptors instead, PlaceArgs::tiles).
PCV_HD uint32_t upper_index(const uint32_t* begin, size_t stride_words, uint32_t n, uint32_t b) {
    uint32_t lo = 0, hi = n;  // largest i in [0, n) with begin[i] <= b
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (begin[(size_t)mid * stride_words] <= b)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}
PCV_HD TileDesc tile_of(const ActiveDesc* active, uint32_t nactive, uint32_t b) {
    const uint32_t i = upper_index(&active[0].tile_begin, sizeof(ActiveDesc) / 4, nactive, b);
    const ActiveDesc& act = active[i];
    const uint64_t o = (uint64_t)(b - act.tile_begin) * kTilePoints;
    const uint64_t rem = act.count - o;
    return TileDesc{act.start + o, (uint32_t)(rem < kTilePoints ? rem : kTilePoints), i};
}
PCV_HD LeafTile leaf_tile_of(const PlaceArgs& a, uint32_t b) {
    const uint32_t l = upper_index(a.d_leaf_tile_begin, 1, a.nleaves, b);
    const uint32_t node = a.d_leaf_node[l];
    const DNode& nd = a.d_nodes[node];
    const uint64_t o = (uint64_t)(b - a.d_leaf_tile_begin[l]) * kPlaceTile;
    const uint64_t rem = nd.count - o;
    return LeafTile{nd.arena_off + o, o, node, (uint32_t)(rem < kPlaceTile ? rem : kPlaceTile)};
}

// ---- pass planning, on the device (one thread per active node; the CPU test backend calls the same function) -------------
// What `split` decides per batch (generation.rs:110-124) and `should_split_node` (:128-150), for the children and - in a
// two-level pass - the grandchildren of one active node: which digits form a bucket, whether the bucket is a leaf (arena)
// or a node of the next pass, where it starts, plus the node table entries, the next pass's active list and scan chunks.
// Running totals of one pass: in counting mode they start at zero and return the node's demand; in emit mode they start at
// the node's exclusive prefix (and the global bases) and every structure is written.
template <bool EMIT>
PCV_HD void plan_active(const PassArgs& a, uint32_t ai, PlanRun& run, int32_t& err, uint32_t& deepest) {
    const ActiveDesc act = a.active[ai];
    const DevNode pn = a.nodes[act.node];
    const uint64_t* nb = a.node_bins + (size_t)ai * a.nbins;
    BucketDesc* bk = a.buckets + (size_t)ai * a.nbins;
    const int w = a.nbins / 8;
    uint32_t nlocal = 0;
    if (!EMIT) {
        uint64_t total = 0;
        for (int b = 0; b < a.nbins; ++b) total += nb[b];
        if (total != act.count) err = kErrHistMismatch;
    }
    // destination of a bucket: leaf -> arena, split -> a node of the next pass
    auto route = [&](uint32_t node_index, int level, const double m[3], uint64_t cnt, bool split, int b0, int b1, int keep) {
        BucketDesc bd{};
        bd.b0 = (uint16_t)b0;
        bd.b1 = (uint16_t)b1;
        bd.keep = (uint8_t)keep;
        if (split) {
            bd.kind = 0;
            bd.dest = run.next_pts;
            const uint32_t nt = (uint32_t)((cnt + kTilePoints - 1) / kTilePoints);
            const uint32_t nc = (nt + kChunkTiles - 1) / kChunkTiles;
            if (EMIT && run.actives < a.cap_active && run.chunks + nc <= a.cap_chunks) {
                ActiveDesc& na = a.active_next[run.actives];
                na.m[0] = m[0], na.m[1] = m[1], na.m[2] = m[2];
                na.e = a.lv.edge[level];
                na.start = run.next_pts;
                na.count = cnt;
                na.chunk_begin = run.chunks;
                na.nchunks = nc;
                na.tile_begin = run.tiles;
                na.node = node_index;
                for (uint32_t o = 0, c = 0; o < nt; o += kChunkTiles, ++c)
                    a.chunks_next[run.chunks + c] = ChunkDesc{run.tiles + o, (nt - o < kChunkTiles ? nt - o : kChunkTiles), run.actives, o == 0 ? 1u : 0u};
            }
            run.actives += 1;
            run.tiles += nt;
            run.chunks += nc;
            run.next_pts += cnt;
        } else {
            bd.kind = 1;
            bd.dest = run.arena_pts;
            if (EMIT && node_index < a.cap_nodes) a.nodes[node_index].arena_off = run.arena_pts;
            run.arena_pts += cnt;
            if (a.holes) run.next_pts += cnt;
            if ((uint32_t)level > deepest) deepest = (uint32_t)level;
        }
        if (EMIT) bk[nlocal] = bd;
        ++nlocal;
    };
    auto emit_node = [&](uint32_t ni, uint32_t parent, uint64_t ihi, uint64_t ilo, int level, const double m[3], uint64_t cnt, bool leaf) {
        if (!EMIT || ni >= a.cap_nodes) return;
        DevNode& d = a.nodes[ni];
        d.index_hi = ihi;
        d.index_lo = ilo;
        d.m[0] = m[0], d.m[1] = m[1], d.m[2] = m[2];
        d.count = cnt;
        d.arena_off = 0;
        d.level = level;
        d.parent = (int32_t)parent;
        d.leaf = leaf ? 1 : 0;
        d.pad = 0;
        if (a.children) {
            for (int q = 0; q < 8; ++q) a.children[(size_t)ni * 8 + q] = -1;
            a.children[(size_t)parent * 8 + (size_t)(ilo & 7u)] = (int32_t)ni;
        }
    };
    // should_split_node (generation.rs:128-150); nodes of levels <= k of a sharded build decide on the global counts
    auto should_split = [&](int level, uint64_t ihi, uint64_t ilo, uint64_t cnt) {
        uint64_t decision = cnt;
        if (a.shard_k && level <= a.shard_k) decision = a.shard_counts[ShardSpec::level_offset(level) + ilo];
        (void)ihi;
        const bool split = decision > a.max_points && a.lv.edge[level] > a.resolution;
        if (split && level >= kMaxLevels - 1) err = kErrTooDeep;  // deeper than 40 levels is not representable in NodeId
        return split;
    };
    for (int k = 0; k < 8; ++k) {
        uint64_t cnt1 = 0;
        for (int b = k * w; b < (k + 1) * w; ++b) cnt1 += nb[b];
        if (cnt1 == 0) continue;
        const int l1 = a.level + 1;
        const uint64_t i1hi = (pn.index_hi << 3) | (pn.index_lo >> 61), i1lo = (pn.index_lo << 3) + (uint64_t)k;  // node.rs:120-125
        const double e1 = a.lv.edge[l1];
        // node.rs:165-170: x = bit2, y = bit1, z = bit0
        const double m1[3] = {(k & 4) ? pn.m[0] + e1 : pn.m[0], (k & 2) ? pn.m[1] + e1 : pn.m[1], (k & 1) ? pn.m[2] + e1 : pn.m[2]};
        const bool split1 = should_split(l1, i1hi, i1lo, cnt1);
        const uint32_t c1 = run.nodes++;
        emit_node(c1, act.node, i1hi, i1lo, l1, m1, cnt1, !split1);
        if (split1 && a.G == 2) {
            for (int k2 = 0; k2 < 8; ++k2) {
                const uint64_t cnt2 = nb[k * 8 + k2];
                if (cnt2 == 0) continue;
                const int l2 = l1 + 1;
                const uint64_t i2hi = (i1hi << 3) | (i1lo >> 61), i2lo = (i1lo << 3) + (uint64_t)k2;
                const double e2 = a.lv.edge[l2];
                const double m2[3] = {(k2 & 4) ? m1[0] + e2 : m1[0], (k2 & 2) ? m1[1] + e2 : m1[1], (k2 & 1) ? m1[2] + e2 : m1[2]};
                const bool split2 = should_split(l2, i2hi, i2lo, cnt2);
                const uint32_t c2 = run.nodes++;
                emit_node(c2, c1, i2hi, i2lo, l2, m2, cnt2, !split2);
                route(c2, l2, m2, cnt2, split2, k * 8 + k2, k * 8 + k2 + 1, 2);
            }
        } else {
            route(c1, l1, m1, cnt1, split1, k * w, (k + 1) * w, 1);
        }
    }
    if (EMIT)
        for (int lb = (int)nlocal; lb < a.nbins; ++lb) bk[lb] = BucketDesc{};
}

// ---- subsample plan, on the device (closed form of generation.rs:195-253,335-387; see the header) ---------------------------------
// Bottom-up over the levels: n(X) = size of X when it is subsampled into its parent (a leaf: its points; an inner node: the sum of
// ceil(n(child) / 8) over its children in child order, which also gives every child its offset inside the parent), then one scan
// over the nodes in creation order for the output layout and the leaf-tile index of the placement.
struct FinishArgs {
    BuildState* st;
    const DevNode* nodes;
    const int32_t* children;    // [nodes][8]
    uint64_t* nsub;             // [nodes]
    uint64_t* final_count;      // [nodes]
    DNode* dn;                  // [nodes]
    uint32_t* leaf_tile_begin;  // [nodes + 1]
    uint32_t* leaf_node;        // [nodes]
    int shard_k;
    int level;                  // finish_node sweep: the level being processed
    LevelTable lv;
};
PCV_HD void finish_node(const FinishArgs& f, uint32_t i) {
    const DevNode& nd = f.nodes[i];
    uint64_t ns;
    if (nd.leaf) {
        ns = nd.count;
    } else {
        uint64_t off = 0;
        for (int k = 0; k < 8; ++k) {
            const int32_t c = f.children[(size_t)i * 8 + k];
            if (c < 0) continue;
            f.dn[c].off_in_parent = off;
            off += (f.nsub[c] + 7) / 8;  // every 8th point by current index: ceil(n / 8)
        }
        ns = off;
        if (f.shard_k && nd.level < f.shard_k - 1) ns = 0;  // above the collectors of a sharded build: assembled elsewhere
    }
    f.nsub[i] = ns;
    const bool collector = f.shard_k && nd.level == f.shard_k - 1;
    f.final_count[i] = (nd.parent < 0 || collector) ? ns : ns - (ns + 7) / 8;
}
// One node of the layout scan: the running offsets are the exclusive prefixes over the nodes before it (creation order).
PCV_HD void finish_emit(const FinishArgs& f, uint32_t i, uint64_t point_off, uint64_t xyz_off, uint32_t leaf_ord, uint32_t tile_begin) {
    const DevNode& nd = f.nodes[i];
    DNode& d = f.dn[i];
    d.m[0] = nd.m[0], d.m[1] = nd.m[1], d.m[2] = nd.m[2];
    d.e = f.lv.edge[nd.level];
    d.ry = f.lv.ry[nd.level];  // RN(1 / e)
    if (nd.parent < 0) d.off_in_parent = 0;
    d.out_point_off = point_off;
    d.out_xyz_off = xyz_off;  // node .xyz blocks are 16-byte aligned inside the device array
    d.arena_off = nd.arena_off;
    d.count = nd.leaf ? nd.count : 0;
    const bool collector = f.shard_k && nd.level == f.shard_k - 1;
    d.parent = collector ? -1 : nd.parent;  // a collector ends the up-walk like the root does
    d.enc = f.lv.enc[nd.level];
    if (nd.leaf) {
        f.leaf_tile_begin[leaf_ord] = tile_begin;
        f.leaf_node[leaf_ord] = i;
    }
}
PCV_HD uint64_t finish_xyz_bytes(const FinishArgs& f, uint32_t i) { return f.final_count[i] * 3 * (uint64_t)enc_bytes(f.lv.enc[f.nodes[i].level]); }
// sequential form (test backend; the CUDA backend runs the same two functions from kernels)
inline void finish_plan_seq(FinishArgs f, int last_level) {
    const uint32_t n = f.st->nnodes;
    for (int L = last_level; L >= 0; --L)
        for (uint32_t i = 0; i < n; ++i)
            if (f.nodes[i].level == L) finish_node(f, i);
    uint64_t poff = 0, boff = 0, algo = 0, last_end = 0;
    uint32_t nleaves = 0, tiles = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint64_t b = finish_xyz_bytes(f, i);
        finish_emit(f, i, poff, boff, nleaves, tiles);
        if (f.nodes[i].leaf) {
            ++nleaves;
            tiles += (uint32_t)((f.nodes[i].count + kPlaceTile - 1) / kPlaceTile);
        }
        poff += f.final_count[i];
        last_end = boff + b;
        boff += (b + 15) & ~15ull;
        algo += b;
    }
    f.leaf_tile_begin[nleaves] = tiles;
    f.st->nleaves = nleaves;
    f.st->place_tiles = tiles;
    f.st->out_points = poff;
    f.st->xyz_bytes = last_end;
    f.st->algo_xyz = algo;
}

struct Backend {
    virtual ~Backend() {}
    virtual void* dmalloc(size_t bytes) = 0;
    virtual void dfree(void* p) = 0;
    virtual void h2d(void* d, const void* h, size_t bytes) = 0;
    virtual void d2h(void* h, const void* d, size_t bytes) = 0;  // synchronises
    virtual void zero(void* d, size_t bytes) = 0;
    virtual void ingest(const IngestArgs& a) = 0;   // raw points -> level-1 records + first digits
    virtual void pass(const PassArgs& a) = 0;       // digit histogram + scan + plan + partition of one pass (asynchronous)
    virtual void hist_scan(const PassArgs& a) {}    // only the digit histogram + scan of a pass (sharded build: the sender's side)
    virtual void plan(const PassArgs& a) {}         // only the planner of a pass (sharded build: the owner's side of the fused exchange pass)
    virtual void finish_plan(const FinishArgs& f, int last_level) = 0;  // the subsample plan (asynchronous)
    // asynchronous read-back into backend-owned host memory: valid after d2h_wait(); at most kReadSlots copies between two waits
    virtual const void* d2h_begin(const void* d, size_t bytes) = 0;
    virtual void d2h_wait() = 0;
    virtual void place(const PlaceArgs& a) = 0;
    virtual void mark(int what) {}  // timing hooks: 0 partition start, 1 partition end / place start, 2 place end
    virtual void pass_points(int pass, uint64_t npoints, uint64_t leaf_points) {}  // profiling: live point counts, known after the read-back
};

// ---- host-side node algebra (node.rs) -------------------------------------------------------------
struct HNode {
    u128 index;
    int level;
    int parent;
    int child[8];
    uint64_t count;  // points routed into the node by the split phase
    bool leaf;
    uint64_t arena_off;
    uint64_t n_sub;  // size when the node is subsampled into its parent
    uint64_t off_in_parent;
    uint64_t final_count;
    uint64_t out_point_off, out_xyz_off;
    double m[3];
    double e;
    int enc;
};

inline uint32_t rust_as_u32(double v) {
    if (!(v == v) || v <= 0.0) return 0u;
    if (v >= 4294967295.0) return 4294967295u;
    return (uint32_t)v;
}
// PositionEncoding::new (codec.rs:31-40)
inline int position_encoding_for(double edge, double resolution) {
    uint32_t min_bits = rust_as_u32(std::log2(edge / resolution)) + 1u;
    if (min_bits <= 8) return ENC_U8;
    if (min_bits <= 16) return ENC_U16;
    if (min_bits <= 24) return ENC_F32;
    return ENC_F64;
}

// `root_min`: min corner of the root cube.  When every coordinate inside the root cube has a magnitude in
// [2^-300, 2^300) on every axis, the numerators q - m of the whole tree are exactly 0 or in [2^-353, 2^500) (q and m are
// doubles of at least that magnitude, so a non-zero difference is at least half an ulp of 2^-300), i.e. inside
// div_known's proven range without looking at them: fast = 2 (the kernels then only check the raw inputs once).
inline LevelTable make_level_table(double root_edge, double resolution, const double* root_min = nullptr) {
    LevelTable t;
    double e = root_edge;
    t.last_level = kMaxLevels - 1;
    bool found = false;
    t.fast = 1;
    for (int L = 0; L < kMaxLevels; ++L) {
        t.edge[L] = e;
        t.ry[L] = 1.0 / e;  // RN(1/edge), for div_known
        if (!div_known_ok(e)) t.fast = 0;
        t.enc[L] = (int8_t)position_encoding_for(e, resolution);
        // should_split_node (generation.rs:128-150): a node at level L >= 1 is split only if edge > resolution.
        if (!found && L >= 1 && !(e > resolution)) {
            t.last_level = L;
            found = true;
        }
        e /= 2.;  // node.rs:161
    }
    if (t.fast && root_min && !std::getenv("PCV_CHECKED_FAST")) {  // PCV_CHECKED_FAST=1: diagnostic, keep the per-numerator checks
        const double lo = std::ldexp(1.0, -300), hi = std::ldexp(1.0, 300);
        bool ok = root_edge > 0.0 && root_edge < hi;
        for (int k = 0; k < 3 && ok; ++k) {
            const double a = root_min[k], b = root_min[k] + root_edge;
            ok = std::isfinite(a) && std::fabs(a) < hi && std::fabs(b) < hi && (a >= lo || b <= -lo);
        }
        if (ok) t.fast = 2;
    }
    // Power-of-two edges (a root edge of 2^j halves exactly down to the last level): the division by an edge is an exact
    // scaling for every operand, so the kernels multiply by 2^-j and need neither reciprocal refinement nor range checks.
    if (t.fast && !std::getenv("PCV_NO_POW2")) {
        bool pow2 = true;
        for (int L = 0; L <= std::min(t.last_level + 1, kMaxLevels - 1) && pow2; ++L) {
            int ex = 0;
            pow2 = std::isnormal(t.edge[L]) && std::frexp(t.edge[L], &ex) == 0.5 && std::isnormal(t.ry[L]) && t.ry[L] * t.edge[L] == 1.0;
        }
        if (pow2) t.fast = 3;
    }
    return t;
}

// PassArgs::e1 .. fast from the level table (pa.level and pa.G must be set)
inline void set_level_constants(PassArgs& pa, const LevelTable& lv) {
    const int L1 = pa.level + 1, L2 = std::min(pa.level + 2, kMaxLevels - 1), Lb = pa.level + pa.G, Lh = std::min(Lb + 1, kMaxLevels - 1);
    pa.e1 = lv.edge[L1], pa.e2 = lv.edge[L2], pa.ry2 = lv.ry[L2];
    pa.eb = lv.edge[Lb], pa.eh = lv.edge[Lh], pa.ryh = lv.ry[Lh];
    pa.enc1 = lv.enc[L1], pa.enc2 = lv.enc[L2], pa.ench = lv.enc[Lh];
    pa.fast = lv.fast;
}

struct BuildResult {
    std::vector<HNode> nodes;     // creation order (parents before children)
    std::vector<int> sorted;      // node indices sorted by NodeId
    uint64_t n = 0;
    uint64_t xyz_bytes = 0;
    uint8_t* d_xyz = nullptr;
    uint8_t* d_rgb = nullptr;
    float* d_intensity = nullptr;
    uint32_t* d_src = nullptr;
    uint32_t passes = 0;
    uint32_t deepest_level = 0;
    double host_ms_plan = 0, host_ms_wait = 0;
    uint64_t algorithmic_bytes = 0;
    LevelTable lv;
    double root_min[3];
    double root_edge;
};

struct BuildError : std::runtime_error {
    int code;
    BuildError(int c, const std::string& s) : std::runtime_error(s), code(c) {}
};

// Records that already went through the ingest step on another GPU (sharded build): level-1 codes + the first pass's digits
// of `n` points, in this context's memory; idx of record i must be i.  The build then starts at its first partition pass.
struct ExternalRecords {
    const void* rec = nullptr;
    const uint32_t* col = nullptr;
    const uint8_t* dig = nullptr;
    uint64_t n = 0;
    bool present = false;
    bool col_in_record = false;  // narrow records as they cross the link: {code x 3, packed colour}; idx == position is implied
    // Fused exchange pass: the senders already ran the first partition pass into this context's buffers.  `rec` / `col` / `dig`
    // then are the NEXT pass's input (n slots in cell-major order, holes where a level-2 cell is a leaf), `arena` / `col_arena`
    // (capacity n records) hold the leaf cells' records at the offsets the planner assigns, and `first_bins` (host, 64 entries)
    // is what the first pass's digit histogram would have been: the points this context owns per level-2 cell.
    bool after_first_pass = false;
    void* arena = nullptr;
    uint32_t* col_arena = nullptr;
    const uint64_t* first_bins = nullptr;
};

class BuildPlan {
   public:
    Backend& be;
    uint64_t max_points;
    ShardSpec shard;
    ExternalRecords ext;
    BuildPlan(Backend& b, uint64_t max_points_per_node, int /*levels_per_pass: the split phase resolves two levels per pass*/)
        : be(b), max_points(max_points_per_node ? max_points_per_node : 100000) {}

    template <class T>
    T* upload(const std::vector<T>& v, std::vector<void*>& owned) {
        if (v.empty()) return nullptr;
        T* d = (T*)be.dmalloc(v.size() * sizeof(T));
        owned.push_back(d);
        be.h2d(d, v.data(), v.size() * sizeof(T));
        return d;
    }

    BuildResult run(const PointsView& pts, double resolution, const double bmin[3], const double bmax[3]) {
        if (!(resolution > 0.0)) throw BuildError(-1, "resolution must be > 0");
        if (pts.n >= 0xFFFFFFFFull) throw BuildError(-6, "more than 2^32-2 points per context are not supported");
        BuildResult R;
        R.n = pts.n;
        const auto t_run0 = std::chrono::steady_clock::now();
        double ms_setup = 0;
        // Cube::bounding (aabb.rs:149-157)
        double E = std::fmax(std::fmax(bmax[0] - bmin[0], bmax[1] - bmin[1]), bmax[2] - bmin[2]);
        for (int a = 0; a < 3; ++a) R.root_min[a] = bmin[a];
        R.root_edge = E;
        R.lv = make_level_table(E, resolution, bmin);
        const LevelTable& lv = R.lv;
        if (pts.n == 0) return R;  // no leaves -> no nodes at all (generation.rs:325-397)

        bool wide = false;
        for (int L = 1; L <= lv.last_level; ++L) wide = wide || lv.enc[L] == ENC_F64;
        const size_t rec_bytes = wide ? sizeof(RecW) : sizeof(RecN);
        const uint64_t N = pts.n;

        // pass schedule: level-synchronous, two levels per pass (one when a single level is left)
        struct Sched {
            int level, G;
        };
        std::vector<Sched> sched;
        for (int L = 0; L < lv.last_level;) {
            const int G = std::min(2, lv.last_level - L);
            sched.push_back(Sched{L, G});
            L += G;
        }
        if (sched.empty()) throw BuildError(-6, "octree deeper than 40 levels is not representable in NodeId");

        // capacities (upper bounds; the planner raises kErrCapacity instead of overrunning them).  A node that is split has more
        // than max_points points - or, in a sharded build, sits at a level <= k - so a pass has at most N / (max_points + 1) (+
        // the shard's top cells) active nodes; every node but the root is a child of a split node.
        uint64_t shard_cells = 0;
        for (int j = 1; j <= shard.k; ++j) shard_cells += (uint64_t)1 << (3 * j);
        const uint64_t cap_active64 = N / (max_points + 1) + shard_cells + 2;
        const uint64_t cap_tiles64 = N / kTilePoints + cap_active64 + 1;
        const uint64_t cap_chunks64 = cap_tiles64 / kChunkTiles + cap_active64 + 1;
        const uint64_t cap_nodes64 = 2 + 8 * (uint64_t)lv.last_level * cap_active64;
        if (cap_nodes64 >= 0x7FFFFFFFull || cap_tiles64 >= 0xFFFFFFFFull) throw BuildError(-6, "node / tile tables exceed 2^31 entries");
        const uint32_t cap_active = (uint32_t)cap_active64, cap_tiles = (uint32_t)cap_tiles64, cap_chunks = (uint32_t)cap_chunks64,
                       cap_nodes = (uint32_t)cap_nodes64;

        const bool fused = ext.present && ext.after_first_pass;
        if (fused && (shard.k != 2 || sched[0].G != 2 || !ext.arena || !ext.col_arena || !ext.first_bins))
            throw BuildError(-1, "a fused exchange pass needs a level-2 sharding, a two-level first pass and the owner's arena");
        std::vector<void*> owned;
        auto dalloc = [&](size_t bytes) {
            void* p = be.dmalloc(bytes);
            owned.push_back(p);
            return p;
        };
        void* arena = nullptr;
        uint32_t* col_arena = nullptr;
        std::vector<HNode>& nodes = R.nodes;
        BuildState hs{};
        try {
            // ping-pong buffers; with external records the first of each pair is the caller's (read only, never freed here)
            // (after a fused exchange pass the caller's buffers are the SECOND of each pair: the first pass has been run into them)
            const int xb = ext.present ? (ext.after_first_pass ? 1 : 0) : -1;
            void* bufs[2];
            uint32_t* cols[2];
            uint8_t* digs[2];
            for (int b = 0; b < 2; ++b) {
                bufs[b] = b == xb ? const_cast<void*>(ext.rec) : dalloc((size_t)N * rec_bytes + 64);
                cols[b] = (b == xb && ext.col) ? const_cast<uint32_t*>(ext.col) : (uint32_t*)dalloc((size_t)N * 4 + 64);  // + slack: bulk copies read whole 16-byte granules
                digs[b] = b == xb ? const_cast<uint8_t*>(ext.dig) : (uint8_t*)dalloc((size_t)N + 64);
            }
            if (fused) {
                arena = ext.arena;
                col_arena = ext.col_arena;
            } else {
                arena = dalloc((size_t)N * rec_bytes);
                col_arena = (uint32_t*)dalloc((size_t)N * 4 + 64);
            }
            BuildState* d_st = (BuildState*)dalloc(sizeof(BuildState));
            ActiveDesc* act[2] = {(ActiveDesc*)dalloc((size_t)cap_active * sizeof(ActiveDesc)), (ActiveDesc*)dalloc((size_t)cap_active * sizeof(ActiveDesc))};
            ChunkDesc* chk[2] = {(ChunkDesc*)dalloc((size_t)cap_chunks * sizeof(ChunkDesc)), (ChunkDesc*)dalloc((size_t)cap_chunks * sizeof(ChunkDesc))};
            uint32_t* tile_counts = (uint32_t*)dalloc((size_t)cap_tiles * 64 * 4);
            uint32_t* tile_active = (uint32_t*)dalloc((size_t)cap_tiles * 4);
            uint32_t* chunk_sums = (uint32_t*)dalloc((size_t)cap_chunks * 64 * 4);
            uint64_t* node_bins = (uint64_t*)dalloc((size_t)cap_active * 64 * 8);
            BucketDesc* buckets = (BucketDesc*)dalloc((size_t)cap_active * 64 * sizeof(BucketDesc));
            PlanRun* plan_runs = (PlanRun*)dalloc((size_t)cap_active * sizeof(PlanRun));
            DevNode* d_nodes = (DevNode*)dalloc((size_t)cap_nodes * sizeof(DevNode));
            int32_t* d_children = (int32_t*)dalloc((size_t)cap_nodes * 8 * sizeof(int32_t));
            uint64_t* d_nsub = (uint64_t*)dalloc((size_t)cap_nodes * 8);
            uint64_t* d_final = (uint64_t*)dalloc((size_t)cap_nodes * 8);
            DNode* d_dn = (DNode*)dalloc((size_t)cap_nodes * sizeof(DNode));
            uint32_t* d_ltb = (uint32_t*)dalloc(((size_t)cap_nodes + 1) * 4);
            uint32_t* d_leaf_node = (uint32_t*)dalloc((size_t)cap_nodes * 4);
            uint64_t* d_shard = nullptr;
            if (shard.k) {
                const size_t ncount = ShardSpec::level_offset(shard.k + 1);
                d_shard = (uint64_t*)dalloc(ncount * 8);
                be.h2d(d_shard, shard.counts, ncount * 8);
            }

            // initial state: the root node (always split, generation.rs:312-323), one active node covering the input
            const uint32_t nt0 = (uint32_t)((N + kTilePoints - 1) / kTilePoints);
            hs.nnodes = 1;
            hs.pass[0].nactive = 1;
            hs.pass[0].ntiles = nt0;
            hs.pass[0].nchunks = (nt0 + kChunkTiles - 1) / kChunkTiles;
            hs.pass[0].npoints = N;
            be.h2d(d_st, &hs, sizeof hs);
            DevNode root{};
            for (int a = 0; a < 3; ++a) root.m[a] = bmin[a];
            root.count = N;
            root.level = 0;
            root.parent = -1;
            be.h2d(d_nodes, &root, sizeof root);
            const int32_t no_children[8] = {-1, -1, -1, -1, -1, -1, -1, -1};
            be.h2d(d_children, no_children, sizeof no_children);
            ActiveDesc a0{};
            for (int a = 0; a < 3; ++a) a0.m[a] = bmin[a];
            a0.e = E;
            a0.start = 0;
            a0.count = N;
            a0.chunk_begin = 0;
            a0.nchunks = hs.pass[0].nchunks;
            a0.tile_begin = 0;
            a0.node = 0;
            be.h2d(act[0], &a0, sizeof a0);
            std::vector<ChunkDesc> c0;
            for (uint32_t o = 0; o < nt0; o += kChunkTiles) c0.push_back(ChunkDesc{o, std::min(kChunkTiles, nt0 - o), 0u, o == 0 ? 1u : 0u});
            be.h2d(chk[0], c0.data(), c0.size() * sizeof(ChunkDesc));

            ms_setup = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_run0).count();
            be.mark(0);
            IngestArgs ia{};
            ia.pts = pts;
            ia.rec_out = bufs[0];
            ia.col_out = cols[0];
            ia.dig_out = digs[0];
            ia.G0 = sched[0].G;
            ia.wide = wide;
            ia.ntiles = nt0;
            ia.lv = lv;
            for (int a = 0; a < 3; ++a) ia.root_min[a] = bmin[a];
            if (!ext.present) be.ingest(ia);

            // Small inputs: read the state back after every pass and stop at the first pass without active nodes (a few empty
            // launches cost more than the build of a 1e5-point cloud).  Large inputs: enqueue everything, one read-back at the end.
            const bool poll = N < (4u << 20);
            size_t launched = 0;
            for (size_t p = 0; p < sched.size(); ++p) {
                PassArgs pa{};
                pa.pass = (int)p;
                pa.level = sched[p].level;
                pa.G = sched[p].G;
                pa.nbins = 1 << (3 * pa.G);
                pa.Gn = p + 1 < sched.size() ? sched[p + 1].G : 0;
                pa.wide = wide;
                pa.rec_has_col = ext.present && ext.col_in_record && p == (fused ? 1u : 0u);
                pa.holes = fused && p == 0;
                pa.rec_in = bufs[p & 1];
                pa.rec_next = bufs[(p + 1) & 1];
                pa.arena = arena;
                pa.col_in = cols[p & 1];
                pa.col_next = cols[(p + 1) & 1];
                pa.col_arena = col_arena;
                pa.dig_in = digs[p & 1];
                pa.dig_next = digs[(p + 1) & 1];
                pa.st = d_st;
                pa.active = act[p & 1];
                pa.active_next = act[(p + 1) & 1];
                pa.chunks = chk[p & 1];
                pa.chunks_next = chk[(p + 1) & 1];
                pa.tile_counts = tile_counts;
                pa.tile_active = tile_active;
                pa.chunk_sums = chunk_sums;
                pa.node_bins = node_bins;
                pa.buckets = buckets;
                pa.plan_runs = plan_runs;
                pa.nodes = d_nodes;
                pa.children = d_children;
                pa.cap_active = cap_active;
                pa.cap_nodes = cap_nodes;
                pa.cap_tiles = cap_tiles;
                pa.cap_chunks = cap_chunks;
                pa.max_points = max_points;
                pa.resolution = resolution;
                pa.shard_k = shard.k;
                pa.shard_counts = d_shard;
                pa.lv = lv;
                set_level_constants(pa, lv);
                if (fused && p == 0) {  // the senders ran this pass's partition: only its plan is made here, from the known cell counts
                    be.h2d(node_bins, ext.first_bins, 64 * sizeof(uint64_t));
                    be.plan(pa);
                } else {
                    be.pass(pa);
                }
                ++launched;
                if (poll) {
                    const auto tw0 = std::chrono::steady_clock::now();
                    be.d2h(&hs, d_st, sizeof hs);
                    R.host_ms_wait += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tw0).count();
                    if (hs.error || hs.pass[p + 1].nactive == 0) break;
                }
            }
            // ---- subsample plan on the device, enqueued behind the last pass: the host only reads totals before the placement ----
            FinishArgs fa{};
            fa.st = d_st;
            fa.nodes = d_nodes;
            fa.children = d_children;
            fa.nsub = d_nsub;
            fa.final_count = d_final;
            fa.dn = d_dn;
            fa.leaf_tile_begin = d_ltb;
            fa.leaf_node = d_leaf_node;
            fa.shard_k = shard.k;
            fa.lv = lv;
            be.finish_plan(fa, lv.last_level);
            be.mark(1);
            const auto tw0 = std::chrono::steady_clock::now();
            be.d2h(&hs, d_st, sizeof hs);
            R.host_ms_wait += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tw0).count();
            if (hs.error == kErrTooDeep) throw BuildError(-6, "octree deeper than 40 levels is not representable in NodeId");
            if (hs.error == kErrHistMismatch) throw BuildError(-2, "internal: histogram total mismatch");
            if (hs.error) throw BuildError(-2, "internal: planner capacity exceeded");
            if (hs.arena_used != N) {
                if (std::getenv("PCV_TIMING")) {
                    fprintf(stderr, "[pcv] lost points: arena %llu of %llu, nodes %u, launched %zu of %zu passes\n", (unsigned long long)hs.arena_used, (unsigned long long)N,
                            hs.nnodes, launched, sched.size());
                    for (size_t p = 0; p <= launched; ++p)
                        fprintf(stderr, "[pcv]   pass %zu: nactive %u ntiles %u nchunks %u npoints %llu\n", p, hs.pass[p].nactive, hs.pass[p].ntiles, hs.pass[p].nchunks,
                                (unsigned long long)hs.pass[p].npoints);
                }
                throw BuildError(-2, "internal: the split phase lost points");
            }
            if (hs.out_points != N) throw BuildError(-2, "internal: subsample plan does not conserve points");
            for (size_t p = 0; p < launched; ++p) {
                if (hs.pass[p].nactive) R.passes++;
                be.pass_points((int)p, hs.pass[p].npoints, hs.pass[p].npoints - hs.pass[p + 1].npoints);
            }
            R.deepest_level = hs.deepest_level;
            const auto ts0 = std::chrono::steady_clock::now();
            // the ping-pong buffers and the planner's tables are dead now; the arena and the plan's tables live until the placement is done
            auto keep = [&](void* q) {
                return q == arena || q == (void*)col_arena || q == (void*)d_nodes || q == (void*)d_dn || q == (void*)d_nsub || q == (void*)d_final || q == (void*)d_ltb ||
                       q == (void*)d_leaf_node;
            };
            for (auto& q : owned) {
                if (q && !keep(q)) {  // (a fused build's arena is the caller's and not in `owned`)
                    be.dfree(q);
                    q = nullptr;
                }
            }
            // node tables for the host-side octree object: their read-back is enqueued BEFORE the placement and consumed while it runs
            const uint32_t nn = hs.nnodes;
            const DevNode* hv = (const DevNode*)be.d2h_begin(d_nodes, (size_t)nn * sizeof(DevNode));
            const DNode* hd = (const DNode*)be.d2h_begin(d_dn, (size_t)nn * sizeof(DNode));
            const uint64_t* hns = (const uint64_t*)be.d2h_begin(d_nsub, (size_t)nn * 8);
            const uint64_t* hfc = (const uint64_t*)be.d2h_begin(d_final, (size_t)nn * 8);
            R.xyz_bytes = hs.xyz_bytes;
            R.algorithmic_bytes = 27ull * pts.n + hs.algo_xyz + 3ull * pts.n + (pts.intensity ? 8ull * pts.n : 0ull);
            R.d_xyz = (uint8_t*)be.dmalloc(hs.xyz_bytes + 32);  // + slack: the query kernels stage whole 16-byte granules
            R.d_rgb = (uint8_t*)be.dmalloc((size_t)pts.n * 3);
            R.d_src = (uint32_t*)be.dmalloc((size_t)pts.n * 4 + 64);
            R.d_intensity = pts.intensity ? (float*)be.dmalloc((size_t)pts.n * 4) : nullptr;
            PlaceArgs pl{};
            pl.wide = wide;
            pl.pts = pts;
            pl.arena = arena;
            pl.col_arena = col_arena;
            pl.fast = lv.fast;
            pl.d_nodes = d_dn;
            pl.d_leaf_tile_begin = d_ltb;
            pl.d_leaf_node = d_leaf_node;
            pl.nleaves = hs.nleaves;
            pl.ntiles = hs.place_tiles;
            pl.npoints = pts.n;
            pl.xyz_bytes = hs.algo_xyz;
            pl.out_xyz = R.d_xyz;
            pl.out_rgb = R.d_rgb;
            pl.out_intensity = R.d_intensity;
            pl.out_src = R.d_src;
            const auto ts1 = std::chrono::steady_clock::now();
            be.place(pl);
            be.mark(2);
            // ---- host-side node table (while the placement runs) ----
            be.d2h_wait();
            const auto ts2 = std::chrono::steady_clock::now();
            nodes.resize(nn);
            struct SortKey {
                uint64_t hi, lo;  // NodeId = level << 120 | index (node.rs:108-111)
                uint32_t i;
            };
            std::vector<SortKey> keys(nn);
            for (uint32_t i = 0; i < nn; ++i) {
                const DevNode& d = hv[i];
                keys[i] = SortKey{((uint64_t)d.level << 56) | d.index_hi, d.index_lo, i};
                HNode& x = nodes[i];
                x = HNode{};
                x.index = ((u128)d.index_hi << 64) | d.index_lo;
                x.level = d.level;
                x.parent = d.parent;
                for (int k = 0; k < 8; ++k) x.child[k] = -1;
                x.count = d.count;
                x.leaf = d.leaf != 0;
                x.arena_off = d.arena_off;
                for (int a = 0; a < 3; ++a) x.m[a] = d.m[a];
                x.e = lv.edge[d.level];
                x.enc = lv.enc[d.level];
                x.n_sub = hns[i];
                x.off_in_parent = hd[i].off_in_parent;
                x.final_count = hfc[i];
                x.out_point_off = hd[i].out_point_off;
                x.out_xyz_off = hd[i].out_xyz_off;
                if (d.parent >= 0) nodes[d.parent].child[(int)(d.index_lo & 7)] = (int)i;
            }
            // nodes sorted by NodeId (level << 120 | index); the device arrays are laid out in node creation order
            std::sort(keys.begin(), keys.end(), [](const SortKey& a, const SortKey& b) { return a.hi != b.hi ? a.hi < b.hi : a.lo < b.lo; });
            R.sorted.resize(nn);
            for (uint32_t i = 0; i < nn; ++i) R.sorted[i] = (int)keys[i].i;
            const auto ts3 = std::chrono::steady_clock::now();
            for (auto& q : owned) {
                if (q) {
                    be.dfree(q);
                    q = nullptr;
                }
            }
            auto tms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
            R.host_ms_plan += tms(ts0, ts1) + tms(ts2, ts3);
            if (std::getenv("PCV_TIMING"))
                fprintf(stderr, "[pcv timing] setup %.2f  passes %u  wait %.2f | frees + output allocation %.2f  table read-back %.2f  host node table %.2f (overlaps the placement)  (nodes %zu, leaf tiles %u)\n",
                        ms_setup, R.passes, R.host_ms_wait, tms(ts0, ts1), tms(ts1, ts2), tms(ts2, ts3), nodes.size(), hs.place_tiles);
        } catch (...) {
            for (void* q : owned)
                if (q) be.dfree(q);
            be.dfree(R.d_xyz), be.dfree(R.d_rgb), be.dfree(R.d_src), be.dfree(R.d_intensity);
            throw;
        }
        return R;
    }
};

// Top-of-tree assembly for the sharded build: the nodes of levels 0..k-1, whose content is what their children gave up
// (every 8th point) - children being the level-k unit roots (built on their owner ranks) or other top nodes.
//   counts      global point counts of the cells of levels 1..k (ShardSpec layout)
//   unit_nsub   n(X) of every level-k cell when it is subsampled into its parent (0 for empty cells)
//   xyz/rgb/intensity: the collectors' gathered content (level k-1 nodes in index order, inside a node child order
//               0..7, inside a child rank order), positions as node-file bytes in the COLLECTOR's encoding.
// The place kernel then walks those points up exactly as in a single-GPU build.
inline BuildResult assemble_top(Backend& be, double resolution, const double bmin[3], const double bmax[3], int k, const uint64_t* counts,
                                const uint64_t* unit_nsub, const uint8_t* xyz, const uint8_t* rgb, const float* intensity, uint64_t npoints) {
    if (k < 1 || k > 3) throw BuildError(-1, "prefix levels must be 1..3");
    if (npoints >= 0xFFFFFFFFull) throw BuildError(-6, "too many points in the top assembly");
    BuildResult R;
    R.n = npoints;
    const double E = std::fmax(std::fmax(bmax[0] - bmin[0], bmax[1] - bmin[1]), bmax[2] - bmin[2]);
    for (int a = 0; a < 3; ++a) R.root_min[a] = bmin[a];
    R.root_edge = E;
    R.lv = make_level_table(E, resolution, bmin);
    const LevelTable& lv = R.lv;
    ShardSpec sp;
    sp.k = k;
    sp.counts = counts;
    uint64_t total = 0;
    for (uint64_t c = 0; c < 8; ++c) total += sp.count_at(1, c);
    if (total == 0) return R;
    bool wide = false;
    for (int L = 1; L <= lv.last_level; ++L) wide = wide || lv.enc[L] == ENC_F64;

    std::vector<HNode>& nodes = R.nodes;
    HNode r{};
    r.parent = -1;
    for (int q = 0; q < 8; ++q) r.child[q] = -1;
    for (int a = 0; a < 3; ++a) r.m[a] = bmin[a];
    r.e = E;
    r.enc = lv.enc[0];
    r.count = total;
    nodes.push_back(r);
    for (size_t i = 0; i < nodes.size(); ++i) {  // breadth first: levels 0..k-2 get their existing children
        if (nodes[i].level >= k - 1) continue;
        for (int c = 0; c < 8; ++c) {
            const HNode p = nodes[i];
            const uint64_t cidx = ((uint64_t)p.index << 3) + (uint64_t)c;
            const uint64_t cnt = sp.count_at(p.level + 1, cidx);
            if (cnt == 0) continue;
            HNode x{};
            x.level = p.level + 1;
            x.index = cidx;
            x.parent = (int)i;
            for (int q = 0; q < 8; ++q) x.child[q] = -1;
            x.count = cnt;
            x.e = lv.edge[x.level];
            x.m[0] = (c & 4) ? p.m[0] + x.e : p.m[0];
            x.m[1] = (c & 2) ? p.m[1] + x.e : p.m[1];
            x.m[2] = (c & 1) ? p.m[2] + x.e : p.m[2];
            x.enc = lv.enc[x.level];
            nodes[i].child[c] = (int)nodes.size();
            nodes.push_back(x);
        }
    }
    // n(X) bottom-up; collectors (level k-1) sum over the level-k unit roots
    std::vector<uint64_t> unit_off(nodes.size() * 8, 0);
    for (size_t i = nodes.size(); i-- > 0;) {
        HNode& x = nodes[i];
        uint64_t off = 0;
        if (x.level == k - 1) {
            for (int c = 0; c < 8; ++c) {
                unit_off[i * 8 + c] = off;
                off += (unit_nsub[((uint64_t)x.index << 3) + (uint64_t)c] + 7) / 8;
            }
        } else {
            for (int c = 0; c < 8; ++c) {
                if (x.child[c] < 0) continue;
                nodes[x.child[c]].off_in_parent = off;
                off += (nodes[x.child[c]].n_sub + 7) / 8;
            }
        }
        x.n_sub = off;
    }
    for (auto& x : nodes) x.final_count = x.parent < 0 ? x.n_sub : x.n_sub - (x.n_sub + 7) / 8;
    R.sorted.resize(nodes.size());
    for (size_t i = 0; i < nodes.size(); ++i) R.sorted[i] = (int)i;
    std::sort(R.sorted.begin(), R.sorted.end(), [&](int a, int b) {
        if (nodes[a].level != nodes[b].level) return nodes[a].level < nodes[b].level;
        return nodes[a].index < nodes[b].index;
    });
    uint64_t poff = 0, boff = 0, arena_total = 0;
    for (int i : R.sorted) {
        HNode& x = nodes[i];
        x.out_point_off = poff;
        boff = (boff + 15) & ~15ull;
        x.out_xyz_off = boff;
        poff += x.final_count;
        boff += x.final_count * 3 * (uint64_t)enc_bytes(x.enc);
        if (x.level == k - 1) {
            x.arena_off = arena_total;
            arena_total += x.n_sub;
        }
    }
    if (arena_total != npoints || poff != npoints) throw BuildError(-1, "top assembly: gathered point count does not match the unit sizes");
    R.xyz_bytes = boff;

    // records from the gathered node-file bytes (collector encoding), in arena order == gathered order
    const int cenc = lv.enc[k - 1], bpc = enc_bytes(cenc);
    const size_t rec_bytes = wide ? sizeof(RecW) : sizeof(RecN);
    std::vector<uint8_t> recs((size_t)npoints * rec_bytes);
    std::vector<uint32_t> cols(npoints);
    for (uint64_t i = 0; i < npoints; ++i) {
        uint64_t c[3] = {0, 0, 0};
        for (int a = 0; a < 3; ++a) std::memcpy(&c[a], xyz + (i * 3 + a) * bpc, (size_t)bpc);
        if (wide) {
            RecW w{{c[0], c[1], c[2]}, (uint32_t)i, 0};
            std::memcpy(&recs[i * rec_bytes], &w, sizeof w);
        } else {
            RecN w{{(uint32_t)c[0], (uint32_t)c[1], (uint32_t)c[2]}, (uint32_t)i};
            std::memcpy(&recs[i * rec_bytes], &w, sizeof w);
        }
        cols[i] = (uint32_t)rgb[3 * i] | ((uint32_t)rgb[3 * i + 1] << 8) | ((uint32_t)rgb[3 * i + 2] << 16);
    }
    std::vector<void*> scratch;
    auto up = [&](const void* h, size_t bytes, size_t slack = 0) {
        void* d = be.dmalloc((bytes ? bytes : 16) + slack);
        scratch.push_back(d);
        if (bytes) be.h2d(d, h, bytes);
        return d;
    };
    std::vector<DNode> dn(nodes.size());
    std::vector<uint32_t> leaf_tile_begin, leaf_node;
    uint32_t nplace_tiles = 0;
    for (size_t i = 0; i < nodes.size(); ++i) {
        const HNode& x = nodes[i];
        DNode& d = dn[i];
        for (int a = 0; a < 3; ++a) d.m[a] = x.m[a];
        d.e = x.e;
        d.ry = 1.0 / x.e;
        d.off_in_parent = x.off_in_parent;
        d.out_point_off = x.out_point_off;
        d.out_xyz_off = x.out_xyz_off;
        d.arena_off = x.arena_off;
        d.count = x.level == k - 1 ? x.n_sub : 0;
        d.parent = x.parent;
        d.enc = x.enc;
        if (x.level == k - 1 && x.n_sub) {
            leaf_tile_begin.push_back(nplace_tiles);
            leaf_node.push_back((uint32_t)i);
            nplace_tiles += (uint32_t)((x.n_sub + kPlaceTile - 1) / kPlaceTile);
        }
    }
    leaf_tile_begin.push_back(nplace_tiles);
    PlaceArgs pl{};
    pl.wide = wide;
    pl.pts = PointsView{nullptr, nullptr, nullptr, 1, nullptr, intensity ? (const float*)up(intensity, (size_t)npoints * 4) : nullptr, npoints};
    pl.arena = up(recs.data(), recs.size());
    pl.col_arena = (const uint32_t*)up(cols.data(), cols.size() * 4, 64);  // + slack: the placement's bulk copies read whole 16-byte granules
    pl.fast = lv.fast;
    pl.d_nodes = (const DNode*)up(dn.data(), dn.size() * sizeof(DNode));
    pl.d_leaf_tile_begin = (const uint32_t*)up(leaf_tile_begin.data(), leaf_tile_begin.size() * 4);
    pl.d_leaf_node = (const uint32_t*)up(leaf_node.data(), leaf_node.size() * 4);
    pl.nleaves = (uint32_t)leaf_node.size();
    pl.ntiles = nplace_tiles;
    pl.npoints = npoints;
    pl.xyz_bytes = boff;
    R.d_xyz = (uint8_t*)be.dmalloc(boff + 32);  // + slack: the query kernels stage whole 16-byte granules
    R.d_rgb = (uint8_t*)be.dmalloc(std::max<uint64_t>(npoints * 3, 16));
    R.d_src = (uint32_t*)be.dmalloc(std::max<uint64_t>(npoints * 4, 16));
    R.d_intensity = intensity ? (float*)be.dmalloc(std::max<uint64_t>(npoints * 4, 16)) : nullptr;
    pl.out_xyz = R.d_xyz;
    pl.out_rgb = R.d_rgb;
    pl.out_intensity = R.d_intensity;
    pl.out_src = R.d_src;
    be.place(pl);
    for (void* p : scratch) be.dfree(p);
    return R;
}

}  // namespace pcv
