// query.cuh — sm_90a kernels of the query side.
//
//   k_sat_nodes      a11-a12  batched separating-axis test: (location, node cube) -> Relation
//   k_propagate      a11      BFS semantics of NodeIdsIterator: a node is visited iff all ancestors passed
//   k_visible_eval   a17      per node: Relation vs the view frustum + relative_size_on_screen
//   k_cull<0/1>, k_cull_chunk<0/1>  a13-a15  decode + PointCulling::contains + interval filters + order-preserving
//                                   count / write passes (FilteredIterator, iterator.rs:96-119)
//   k_cull_fused<0/1>               a13-a15  the same test in one pass: batched counts, with (1) or without (0) the survivors
//   k_s2_cell_boxes, k_s2_select_cells      the S2 cloud's point boxes and cell selection; its cells are culled by the kernels above
//   k_xray_bin<0/1>, k_xray_subtile a19  discretise + per-pixel 1024-bit z-bucket set + grey mapping
//
// All arithmetic is binary64 in the reference's operation order (compiled with -fmad=false).
#pragma once
#include <cuda_runtime.h>

#include "chain.h"
#include "geometry_host.hpp"
#include "lod_order.h"

namespace pcv {

struct QNode {
    double m[3];
    double e;
    uint64_t point_off;
    uint64_t xyz_off;
    uint32_t n;
    int32_t enc;
    int32_t parent;
    int32_t level;
};

enum : uint8_t { REL_IN = 0, REL_CROSS = 1, REL_OUT = 2 };  // sat.rs:39-47
static_assert((int)REL_IN == kS2RelIn && (int)REL_CROSS == kS2RelCross && (int)REL_OUT == kS2RelOut, "s2_cube_relation returns a Relation");

// Project the 8 corners of the cube (min m, edge e) on an axis: Aabb corners order x fastest (aabb.rs:114-125),
// max = min + edge (aabb.rs:175-181).
__device__ __forceinline__ void project_cube(const double m[3], double e, const double ax[3], double& lo, double& hi) {
    const double mx[3] = {m[0] + e, m[1] + e, m[2] + e};
    lo = 1.7976931348623157e308;
    hi = -1.7976931348623157e308;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const double cx = (i & 1) ? mx[0] : m[0], cy = (i & 2) ? mx[1] : m[1], cz = (i & 4) ? mx[2] : m[2];
        const double p = cx * ax[0] + cy * ax[1] + cz * ax[2];
        lo = fmin(lo, p);
        hi = fmax(hi, p);
    }
}

// sat() of sat.rs:174-194 with A = the location (projections precomputed: in aproj for its inline axes, in its table for a Web
// Mercator rect's further axes) and B = the node cube.  The relation does not depend on the order of the axes.
__device__ __forceinline__ uint8_t sat_cube(const QueryGeom& g, const double (*aproj)[2], const double m[3], double e) {
    uint8_t rel = REL_IN;
    const int ni = min(g.naxes, kInlineAxes);
    for (int k = 0; k < ni; ++k) {
        double bmin, bmax;
        project_cube(m, e, g.axes[k], bmin, bmax);
        const double amin = aproj[k][0], amax = aproj[k][1];
        if (bmin > amax || bmax < amin) return REL_OUT;
        if (amin > bmin || bmax > amax) rel = REL_CROSS;
    }
    for (int k = 0; k < g.naxes - kInlineAxes; ++k) {
        double bmin, bmax;
        project_cube(m, e, g.more_axes->a[k], bmin, bmax);
        const double amin = g.more_axes->proj[k][0], amax = g.more_axes->proj[k][1];
        if (bmin > amax || bmax < amin) return REL_OUT;
        if (amin > bmin || bmax > amax) rel = REL_CROSS;
    }
    return rel;
}

// The same test against an arbitrary box (an S2 cell's point box) is sat_box of geometry_host.hpp, shared with the test backend.

// The node test of one location: In for AllPoints, s2_cube_relation for a cell union, else the separating-axis test.
__device__ __forceinline__ uint8_t node_relation(const QueryGeom& g, const double (*aproj)[2], const double m[3], double e) {
    if (g.kind == PCV_LOC_ALL) return REL_IN;
    if (g.kind == kLocCellUnion) return (uint8_t)s2_cube_relation(m, e, g.squares, g.ncells);
    return sat_cube(g, aproj, m, e);
}

// The projections of the location's inline axes (sat_cube projects the others itself).
__device__ __forceinline__ void project_location(const QueryGeom& g, double (*aproj)[2]) {
    const int ni = min(g.naxes, kInlineAxes);
    for (int k = threadIdx.x; k < ni; k += blockDim.x) {
        double lo = 1.7976931348623157e308, hi = -1.7976931348623157e308;
        for (int i = 0; i < 8; ++i) {
            const double p = g.corners[i][0] * g.axes[k][0] + g.corners[i][1] * g.axes[k][1] + g.corners[i][2] * g.axes[k][2];
            lo = fmin(lo, p);
            hi = fmax(hi, p);
        }
        aproj[k][0] = lo;
        aproj[k][1] = hi;
    }
}

// grid = (ceil(nnodes/256), nloc).  rel[loc * nnodes + node]
__global__ void __launch_bounds__(256) k_sat_nodes(const QueryGeom* __restrict__ geoms, const QNode* __restrict__ nodes, uint32_t nnodes,
                                                   uint8_t* __restrict__ rel) {
    __shared__ double aproj[kInlineAxes][2];
    const QueryGeom& g = geoms[blockIdx.y];
    project_location(g, aproj);
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnodes) return;
    uint8_t r = REL_IN;
    if (g.kind != PCV_LOC_ALL) {
        const QNode nd = nodes[i];
        r = node_relation(g, aproj, nd.m, nd.e);
    }
    rel[(size_t)blockIdx.y * nnodes + i] = r;
}

// One block per location; nodes are sorted by level so parents precede children.  pass = not Out && parent passed.
__global__ void __launch_bounds__(1024) k_propagate(const QNode* __restrict__ nodes, const uint32_t* __restrict__ level_start, int nlevels,
                                                    uint32_t nnodes, uint8_t* __restrict__ rel, uint8_t* __restrict__ pass) {
    uint8_t* r = rel + (size_t)blockIdx.x * nnodes;
    uint8_t* p = pass + (size_t)blockIdx.x * nnodes;
    for (int L = 0; L < nlevels; ++L) {
        for (uint32_t i = level_start[L] + threadIdx.x; i < level_start[L + 1]; i += blockDim.x) {
            const int par = nodes[i].parent;
            p[i] = (r[i] != REL_OUT && (par < 0 || p[par])) ? 1 : 0;
        }
        __syncthreads();
    }
}

// relative_size_on_screen (octree/mod.rs:103-139): project the 8 cube corners with the 4x4 (homogeneous divide),
// clamp to [-1,1]^2 x [0,1], grow an Aabb, return diag.x * diag.y.  bad[0] is set if any w == 0 (reference panics).
__device__ __forceinline__ double num_clamp_d(double x, double lo, double hi) { return x < lo ? lo : (x > hi ? hi : x); }
__global__ void __launch_bounds__(256) k_visible_eval(const QueryGeom* __restrict__ geom, const double* __restrict__ M,
                                                      const QNode* __restrict__ nodes, uint32_t nnodes, uint8_t* __restrict__ rel,
                                                      double* __restrict__ size) {
    __shared__ double aproj[kInlineAxes][2];
    const QueryGeom& g = geom[0];
    project_location(g, aproj);
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnodes) return;
    const QNode nd = nodes[i];
    uint8_t relv = sat_cube(g, aproj, nd.m, nd.e);
    const double mn[3] = {nd.m[0], nd.m[1], nd.m[2]}, mx[3] = {nd.m[0] + nd.e, nd.m[1] + nd.e, nd.m[2] + nd.e};
    double lo[2] = {0, 0}, hi[2] = {0, 0};
    // corner order of mod.rs:122-137: min, max, then 6 mixed corners (order is irrelevant for min/max)
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const double px = (c & 1) ? mx[0] : mn[0], py = (c & 2) ? mx[1] : mn[1], pz = (c & 4) ? mx[2] : mn[2];
        double q[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            double a = M[r] * px;
            a = M[4 + r] * py + a;
            a = M[8 + r] * pz + a;
            a = M[12 + r] * 1.0 + a;
            q[r] = a;
        }
        if (q[3] == 0.0) relv |= 0x80;  // Point3::from_homogeneous(..).unwrap() panics for this node (mod.rs:103-106) - if it is ever pushed
        const double x = num_clamp_d(q[0] / q[3], -1., 1.), y = num_clamp_d(q[1] / q[3], -1., 1.);
        if (c == 0) {
            lo[0] = hi[0] = x;
            lo[1] = hi[1] = y;
        } else {
            lo[0] = fmin(lo[0], x);
            hi[0] = fmax(hi[0], x);
            lo[1] = fmin(lo[1], y);
            hi[1] = fmax(hi[1], y);
        }
    }
    size[i] = (hi[0] - lo[0]) * (hi[1] - lo[1]);
    rel[i] = relv;
}

// ---- per-point culling -----------------------------------------------------------------------------
__device__ __forceinline__ bool loc_contains(const QueryGeom& g, double x, double y, double z) {
    if (g.kind == PCV_LOC_AABB) {  // aabb.rs:46-48
        return g.aabb_min[0] <= x && g.aabb_min[1] <= y && g.aabb_min[2] <= z && x < g.aabb_max[0] && y < g.aabb_max[1] && z < g.aabb_max[2];
    }
    if (g.kind == PCV_LOC_FRUSTUM) {  // frustum.rs:120-125
        // q = clip_from_query.transform_point(p) divides by the homogeneous w, then every component must lie strictly inside
        // (-1, 1).  The three IEEE divisions dominate the point test, and they only matter within an ulp of the planes:
        // |fl(r / w)| < 1  <=>  |r / w| < 1 - 2^-54 (the midpoint below 1 rounds to 1), so with T = fl(|w| (1 - 2^-52)) <
        // |w| (1 - 2^-54):  |r| <= T is certainly inside,  |r| >= |w| certainly outside;  only the band in between (and
        // w == 0, tiny, huge or NaN) takes the divisions.  Same result as the reference's arithmetic for every input.
        const double* m = g.clip_from_query;
        double n = m[3] * x;
        n = n + m[7] * y;
        n = n + m[11] * z;
        n = n + m[15];
        double r[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            double a = m[i] * x;
            a = m[4 + i] * y + a;
            a = m[8 + i] * z + a;
            r[i] = a + m[12 + i];
        }
        const double an = fabs(n);
        if (an > 1e-290 && an < 1e300) {
            const double T = an * 0.99999999999999977795539507496869;  // 1 - 2^-52
            bool sure = true, inside = true;
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                const double ar = fabs(r[i]);
                if (ar >= an)
                    inside = false;
                else if (!(ar <= T))
                    sure = false;
            }
            if (!inside) return false;
            if (sure) return true;
        }
        double c[3] = {r[0], r[1], r[2]};
        if (n != 0.0) {
            c[0] = r[0] / n;
            c[1] = r[1] / n;
            c[2] = r[2] / n;
        }
        const double mn = fmin(fmin(c[0], c[1]), c[2]), mx = fmax(fmax(c[0], c[1]), c[2]);
        return mn > -1.0 && mx < 1.0;
    }
    if (g.kind == PCV_LOC_OBB) {  // obb.rs:83-90
        const V3 q = iso_apply(g.obb_from_query, V3{x, y, z});
        return fabs(q.x) <= g.half_extent[0] && fabs(q.y) <= g.half_extent[1] && fabs(q.z) <= g.half_extent[2];
    }
    return true;  // AllPoints, math/mod.rs:157-161
}

struct QTile {
    uint32_t loc;     // the location, | kTileIn when every point of the node passes its point test
    uint32_t node;
    uint32_t first;   // first point of the tile inside the node
    uint32_t count;
};
constexpr uint32_t kQueryTile = 2048;
// Set on the tiles of a node a cell union classifies In: its points skip the point test (the interval filters still apply).
constexpr uint32_t kTileIn = 0x80000000u;
__host__ __device__ __forceinline__ uint32_t tile_loc(const QTile& t) { return t.loc & ~kTileIn; }

// A cell union of at most kCellsShared ids is read from shared memory, staged once per tile; a larger one from global memory.
constexpr uint32_t kCellsShared = 256;
// The union's ids for the point test of one tile: staged into `sh` when they fit.  The caller synchronises the block before
// the first read.
__device__ __forceinline__ const uint64_t* stage_cells(const QueryGeom& g, uint64_t* sh) {
    if (g.kind != kLocCellUnion || g.ncells > kCellsShared) return g.cells;
    for (uint32_t k = threadIdx.x; k < g.ncells; k += blockDim.x) sh[k] = g.cells[k];
    return sh;
}

// PointCulling::contains of the cull kernels: loc_contains, for a cell union contains_cellid(from_point(p))
// (s2_cell_union.rs:27-31) on the decoded position, over the union's ids at `cells`, and for a Web Mercator rect its FP64
// ECEF -> WGS84 -> map test.  Only point queries take these two kinds, so the X-ray kernels' loc_contains does not carry them.
// Their node (cell) tests never make a tile kTileIn for a rect: its polyhedron is not its point predicate.
__device__ __forceinline__ bool cull_contains(const QueryGeom& g, const uint64_t* cells, const double p[3]) {
    if (g.kind == kLocCellUnion) return s2_union_contains(cells, g.ncells, s2_cell_id_from_point(p[0], p[1], p[2]));
    if (g.kind == PCV_LOC_WEB_MERCATOR_RECT) return web_mercator_rect_contains(g.aabb_min, g.aabb_max, p[0], p[1], p[2]);
    return loc_contains(g, p[0], p[1], p[2]);
}

struct CullArgs {
    const QueryGeom* geoms;
    const QNode* nodes;
    const QTile* tiles;
    const uint8_t* xyz;
    const uint8_t* rgb;
    const float* intensity;
    const uint32_t* src;
    const pcv_interval* filters;
    uint32_t nfilt;
    uint32_t* tile_keep;     // count pass output, then (after the scan) exclusive offsets
    double* out_xyz;         // write pass outputs (AoS)
    uint8_t* out_rgb;
    float* out_intensity;
    uint32_t* out_src;
};

__device__ __forceinline__ uint64_t load_code(const uint8_t* p, int enc) {
    if (enc == ENC_U8) return *p;
    if (enc == ENC_U16) return *reinterpret_cast<const uint16_t*>(p);
    if (enc == ENC_F32) return *reinterpret_cast<const uint32_t*>(p);
    return *reinterpret_cast<const uint64_t*>(p);
}

// Point i of node nd from the node-contiguous position codes at xyz; bpc = enc_bytes(nd.enc), computed once per node by the caller.
__device__ __forceinline__ void decode_point(const uint8_t* xyz, const QNode& nd, int bpc, uint32_t i, double p[3]) {
    const uint8_t* s = xyz + nd.xyz_off + (uint64_t)i * 3 * bpc;
#pragma unroll
    for (int k = 0; k < 3; ++k) p[k] = decode1_fast(load_code(s + k * bpc, nd.enc), nd.m[k], nd.e, nd.enc);  // == decode1, integer-built unit fraction
}

// PointCulling::contains (skipped for a tile whose node is In), then the interval filters on the intensity of the point at `slot`.
__device__ __forceinline__ bool point_passes(const CullArgs& a, const QueryGeom& g, const uint64_t* cells, bool all_in, const double p[3], uint64_t slot) {
    bool keep = all_in || cull_contains(g, cells, p);
    if (a.nfilt) {
        const double v = (double)a.intensity[slot];  // iterator.rs:82-91: attribute as f64, closed interval
        for (uint32_t f = 0; f < a.nfilt; ++f) keep = keep && (a.filters[f].lo <= v && v <= a.filters[f].hi);
    }
    return keep;
}

__device__ __forceinline__ bool eval_point(const CullArgs& a, const QueryGeom& g, const uint64_t* cells, bool all_in, const QNode& nd, uint32_t i,
                                           double p[3]) {
    decode_point(a.xyz, nd, enc_bytes(nd.enc), i, p);
    return point_passes(a, g, cells, all_in, p, nd.point_off + i);
}

// The ordered cull of one tile per block: count pass (WRITE = false), then after k_scan_u32 the write pass.  SLOT = false: the
// survivor's provenance is gathered from the resident `src` array (k_cull); SLOT = true: it is the point's slot in the node table,
// slot_base[piece] + first + i (k_cull_chunk, for pieces of nodes streamed from disk).  RGB = false: the cloud has no colour
// (an S2 cloud may have none; an octree always has it), rgb / out_rgb are not touched.
template <bool WRITE, bool SLOT, bool RGB = true>
__device__ __forceinline__ void cull_tile(const CullArgs& a, const uint64_t* slot_base, uint64_t* out_slot) {
    __shared__ uint32_t warp_cnt[8];
    __shared__ uint32_t running;
    __shared__ uint64_t scells[kCellsShared];
    const QTile t = a.tiles[blockIdx.x];
    const QueryGeom& g = a.geoms[tile_loc(t)];
    const bool all_in = (t.loc & kTileIn) != 0;
    const QNode nd = a.nodes[t.node];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t* cells = stage_cells(g, scells);
    if (threadIdx.x == 0) running = WRITE ? a.tile_keep[blockIdx.x] : 0u;
    __syncthreads();
    for (uint32_t r0 = 0; r0 < t.count; r0 += 256) {
        const uint32_t i = r0 + threadIdx.x;
        double p[3] = {0, 0, 0};
        bool keep = false;
        if (i < t.count) keep = eval_point(a, g, cells, all_in, nd, t.first + i, p);
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_cnt[warp] = __popc(bal);
        __syncthreads();
        uint32_t before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            const uint32_t c = warp_cnt[w];
            if (w < warp) before += c;
            total += c;
        }
        if (WRITE && keep) {
            const uint64_t dst = (uint64_t)running + before + __popc(bal & ((1u << lane) - 1u));
            const uint64_t sp = nd.point_off + t.first + i;
            a.out_xyz[3 * dst] = p[0];
            a.out_xyz[3 * dst + 1] = p[1];
            a.out_xyz[3 * dst + 2] = p[2];
            if (RGB) {
                a.out_rgb[3 * dst] = a.rgb[3 * sp];
                a.out_rgb[3 * dst + 1] = a.rgb[3 * sp + 1];
                a.out_rgb[3 * dst + 2] = a.rgb[3 * sp + 2];
            }
            if (a.out_intensity) a.out_intensity[dst] = a.intensity[sp];
            if (SLOT)
                out_slot[dst] = slot_base[t.node] + t.first + i;
            else
                a.out_src[dst] = a.src[sp];
        }
        __syncthreads();
        if (threadIdx.x == 0) running += total;
        __syncthreads();
    }
    if (!WRITE && threadIdx.x == 0) a.tile_keep[blockIdx.x] = running;
}
template <bool WRITE, bool RGB = true>
__global__ void __launch_bounds__(256) k_cull(const __grid_constant__ CullArgs a) {
    cull_tile<WRITE, false, RGB>(a, nullptr, nullptr);
}
// One chunk of a directory-backed query: `nodes` / `tiles` are the chunk's pieces (chunk-local offsets), `src` / `out_src` unused.
// RGB = false: an S2 directory without colour.
struct CullChunkArgs {
    CullArgs c;
    const uint64_t* slot_base;  // [piece] the slot of the piece's first point (octree: point_offset + first; S2 cell: start + first)
    uint64_t* out_slot;
};
template <bool WRITE, bool RGB = true>
__global__ void __launch_bounds__(256) k_cull_chunk(const __grid_constant__ CullChunkArgs a) {
    cull_tile<WRITE, true, RGB>(a.c, a.slot_base, a.out_slot);
}

// Exclusive scan of n u32 values in place; total (u64) to *total_out.  Single block; n is at most a few million tiles.
__global__ void __launch_bounds__(1024) k_scan_u32(uint32_t* v, uint32_t n, unsigned long long* total_out) {
    __shared__ uint32_t wsum[32];
    __shared__ unsigned long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t base = 0; base < n; base += 1024) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t x = i < n ? v[i] : 0u;
        uint32_t incl = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t s = wsum[lane], si = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, si, o);
                if (lane >= o) si += y;
            }
            wsum[lane] = si - s;  // exclusive over warps
        }
        __syncthreads();
        const unsigned long long c = carry;
        if (i < n) v[i] = (uint32_t)(c + wsum[warp] + (incl - x));
        __syncthreads();
        if (threadIdx.x == 1023) carry = c + wsum[warp] + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total_out = carry;
}

// ---- LOD draw order applied at build time (lod_order.h): gather every node's points into their shuffled order ------------------
struct LodArgs {
    const QNode* nodes;
    const QTile* tiles;  // (node, first, count) pieces of every node; loc unused
    const uint64_t* keys;  // [nnodes] permutation key of every node
    const uint8_t* xyz;
    const uint8_t* rgb;
    const float* intensity;
    const uint32_t* src;
    uint8_t* out_xyz;
    uint8_t* out_rgb;
    float* out_intensity;
    uint32_t* out_src;
};
__global__ void __launch_bounds__(256) k_lod_shuffle(const __grid_constant__ LodArgs a, uint32_t ntiles) {
    for (uint32_t ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
        const QTile t = a.tiles[ti];
        const QNode nd = a.nodes[t.node];
        const uint64_t key = a.keys[t.node];
        const int bpc = enc_bytes(nd.enc);
        for (uint32_t k = threadIdx.x; k < t.count; k += blockDim.x) {
            const uint32_t i = t.first + k, j = lod_order(key, nd.n, i);  // new[i] = old[j]
            const uint8_t* sx = a.xyz + nd.xyz_off + (uint64_t)j * 3 * bpc;
            uint8_t* dx = a.out_xyz + nd.xyz_off + (uint64_t)i * 3 * bpc;
            if (bpc == 1) {
                dx[0] = sx[0], dx[1] = sx[1], dx[2] = sx[2];
            } else if (bpc == 2) {
                const uint16_t* s16 = reinterpret_cast<const uint16_t*>(sx);
                uint16_t* d16 = reinterpret_cast<uint16_t*>(dx);
                d16[0] = s16[0], d16[1] = s16[1], d16[2] = s16[2];
            } else if (bpc == 4) {
                const uint32_t* s32 = reinterpret_cast<const uint32_t*>(sx);
                uint32_t* d32 = reinterpret_cast<uint32_t*>(dx);
                d32[0] = s32[0], d32[1] = s32[1], d32[2] = s32[2];
            } else {
                const uint64_t* s64 = reinterpret_cast<const uint64_t*>(sx);
                uint64_t* d64 = reinterpret_cast<uint64_t*>(dx);
                d64[0] = s64[0], d64[1] = s64[1], d64[2] = s64[2];
            }
            const uint64_t sp = nd.point_off + j, dp = nd.point_off + i;
            a.out_rgb[3 * dp] = a.rgb[3 * sp];
            a.out_rgb[3 * dp + 1] = a.rgb[3 * sp + 1];
            a.out_rgb[3 * dp + 2] = a.rgb[3 * sp + 2];
            a.out_src[dp] = a.src[sp];
            if (a.out_intensity) a.out_intensity[dp] = a.intensity[sp];
        }
    }
}

// ---- batched query: hierarchical node selection + single-pass culling ---------------------------------------------
// nodes_in_location for many locations at once, level by level like NodeIdsIterator (octree_iterator.rs:30-43): a frontier of
// (location, node) pairs; every pair is tested once (sat.rs:174-194), a pair that is not Out joins the work list (if the node
// holds points) and hands its existing children to the next level's frontier.  Only visited nodes are ever tested - the
// all-pairs kernel above (k_sat_nodes) stays for the single-location entry points that need the BFS order.
struct LocProj {
    double a[kInlineAxes][2];  // projections of the location's 8 corners on each of its cached axes
};
__global__ void __launch_bounds__(32) k_loc_proj(const QueryGeom* __restrict__ geoms, LocProj* __restrict__ out) {
    project_location(geoms[blockIdx.x], out[blockIdx.x].a);
}
struct BfsArgs {
    const QueryGeom* geoms;
    const LocProj* proj;
    const QNode* nodes;
    const int32_t* children;  // [nnodes][8]
    const uint2* fin;
    uint2* fout;
    const uint32_t* nin;   // size of the incoming frontier (device resident)
    uint32_t* nout;
    uint32_t cap;          // frontier / pair list capacity
    uint2* pairs;          // (location, node) pairs to cull
    uint32_t* npairs;
    unsigned long long* ntiles;
    unsigned long long* tested;  // [nloc] points of the nodes the location visits
    unsigned long long* bytes;   // sum of n * (3 bpc + 3) over the visited pairs
    int* overflow;
};
__global__ void __launch_bounds__(256) k_bfs_level(const __grid_constant__ BfsArgs a) {
    const uint32_t n = min(*a.nin, a.cap);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint2 pr = a.fin[i];
        const QueryGeom& g = a.geoms[pr.x];
        const QNode nd = a.nodes[pr.y];
        uint8_t rel = REL_IN;
        if (g.kind != PCV_LOC_ALL) rel = node_relation(g, a.proj[pr.x].a, nd.m, nd.e);
        if (rel == REL_OUT) continue;
        if (nd.n) {
            const uint32_t k = atomicAdd(a.npairs, 1u);
            if (k < a.cap)  // the pair's tiles carry kTileIn when a cell union holds the whole node
                a.pairs[k] = make_uint2(g.kind == kLocCellUnion && rel == REL_IN ? (pr.x | kTileIn) : pr.x, pr.y);
            else
                *a.overflow = 1;
            atomicAdd(a.ntiles, (unsigned long long)((nd.n + kQueryTile - 1) / kQueryTile));
            atomicAdd(&a.tested[pr.x], (unsigned long long)nd.n);
            atomicAdd(a.bytes, (unsigned long long)nd.n * (3ull * (unsigned long long)enc_bytes(nd.enc) + 3ull));
        }
        const int32_t* ch = a.children + (size_t)pr.y * 8;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int32_t cn = ch[c];
            if (cn < 0) continue;
            const uint32_t k = atomicAdd(a.nout, 1u);
            if (k < a.cap)
                a.fout[k] = make_uint2(pr.x, (uint32_t)cn);
            else
                *a.overflow = 1;
        }
    }
}
__global__ void __launch_bounds__(256) k_bfs_seed(uint2* f, uint32_t nloc, uint32_t root, uint32_t* n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nloc) f[i] = make_uint2(i, root);
    if (i == 0) *n = nloc;
}
__global__ void __launch_bounds__(256) k_pairs_to_tiles(const uint2* __restrict__ pairs, const uint32_t* __restrict__ npairs, uint32_t cap,
                                                        const QNode* __restrict__ nodes, unsigned long long* __restrict__ cursor, QTile* __restrict__ tiles) {
    const uint32_t n = min(*npairs, cap);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint2 pr = pairs[i];
        const uint32_t cnt = nodes[pr.y].n;
        const uint32_t nt = (cnt + kQueryTile - 1) / kQueryTile;
        const unsigned long long base = atomicAdd(cursor, (unsigned long long)nt);
        for (uint32_t k = 0; k < nt; ++k) tiles[base + k] = QTile{pr.x, pr.y, k * kQueryTile, min(kQueryTile, cnt - k * kQueryTile)};
    }
}

// ---- S2 cells: location queries of an S2 cloud (s2_api.inl) -------------------------------------------------------------------
// The cells of an S2 cloud go to the cull kernels as Float64 nodes (QNode m = -0.0, e = 1: fma(v, 1, -0.0) == v for every v, so
// the decoded position is the stored double, bit for bit).  A cell is selected by the separating-axis test of the location
// against its point box: the exact component-wise min and max of its stored positions.
//
// k_s2_cell_boxes: the point boxes, one block per work tile (cell, first, count) of the cell-contiguous positions.  Min and max
// are taken over order-preserving integer keys of the doubles (warp shuffles, then one atomic per warp and bound), so the box
// does not depend on the order in which tiles and lanes meet; k_s2_box_keys_to_f64 turns the keys back into doubles.
__device__ __forceinline__ unsigned long long f64_order_key(double v) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double f64_from_order_key(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFull) : ~k));
}
// kmin / kmax: [cell * 3 + axis], preset to ~0 / 0
__global__ void __launch_bounds__(256) k_s2_cell_boxes(const double* __restrict__ xyz, const QNode* __restrict__ cells, const QTile* __restrict__ tiles,
                                                      uint32_t ntiles, unsigned long long* __restrict__ kmin, unsigned long long* __restrict__ kmax) {
    for (uint32_t ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
        const QTile t = tiles[ti];
        const uint64_t first = cells[t.node].point_off + t.first;
        unsigned long long lo[3] = {~0ull, ~0ull, ~0ull}, hi[3] = {0ull, 0ull, 0ull};
        for (uint32_t i = threadIdx.x; i < t.count; i += blockDim.x) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const unsigned long long key = f64_order_key(__ldcs(xyz + 3 * (first + i) + k));
                lo[k] = min(lo[k], key);
                hi[k] = max(hi[k], key);
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
                hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
            }
        if ((threadIdx.x & 31) == 0 && threadIdx.x < t.count)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                atomicMin(&kmin[3 * (size_t)t.node + k], lo[k]);
                atomicMax(&kmax[3 * (size_t)t.node + k], hi[k]);
            }
    }
}
__global__ void __launch_bounds__(256) k_s2_box_keys_to_f64(unsigned long long* __restrict__ keys, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const double v = f64_from_order_key(keys[i]);
        reinterpret_cast<double*>(keys)[i] = v;
    }
}

// k_s2_select_cells: grid (cells / 256, locations).  Every thread tests one (location, cell): AllPoints selects every cell, a cell
// union the cells its ranges intersect (In when the union contains the whole cell: its points skip the point test), any other
// location the cells whose point box sat_box does not call Out.  A selected cell with points joins the pair list (no
// particular order); its tiles and points are added to ntiles and tested[location].  The pair list holds nloc * ncells entries:
// it cannot overflow.
struct S2SelectArgs {
    const QueryGeom* geoms;
    const LocProj* proj;
    const QNode* cells;
    const uint64_t* ids;
    const double* bmin;       // [cell * 3 + axis] point boxes
    const double* bmax;
    uint32_t ncells;
    uint2* pairs;             // (location | kTileIn, cell)
    uint32_t* npairs;
    unsigned long long* ntiles;
    unsigned long long* tested;  // [location]
};
__global__ void __launch_bounds__(256) k_s2_select_cells(const __grid_constant__ S2SelectArgs a) {
    __shared__ double aproj[kInlineAxes][2];
    const uint32_t loc = blockIdx.y;
    const QueryGeom& g = a.geoms[loc];
    for (int k = threadIdx.x; k < 2 * kInlineAxes; k += blockDim.x) aproj[k >> 1][k & 1] = a.proj[loc].a[k >> 1][k & 1];
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t n = 0, flag = 0;
    if (i < a.ncells) {
        int rel = kS2RelIn;
        if (g.kind == kLocCellUnion) {
            const uint64_t id = a.ids[i];
            rel = !s2_union_intersects(g.cells, g.ncells, id) ? kS2RelOut : s2_union_contains(g.cells, g.ncells, id) ? kS2RelIn : kS2RelCross;
            if (rel == kS2RelIn) flag = kTileIn;
        } else if (g.kind != PCV_LOC_ALL) {
            rel = sat_box(g, aproj, a.bmin + 3 * (size_t)i, a.bmax + 3 * (size_t)i);
        }
        if (rel != kS2RelOut) n = a.cells[i].n;
    }
    const unsigned sel = __ballot_sync(0xffffffffu, n != 0);
    if (sel == 0) return;
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(a.npairs, (uint32_t)__popc(sel));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (n) a.pairs[base + __popc(sel & ((1u << lane) - 1u))] = make_uint2(loc | flag, i);
    unsigned long long nt = (n + kQueryTile - 1) / kQueryTile, np = n;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        nt += __shfl_xor_sync(0xffffffffu, nt, o);
        np += __shfl_xor_sync(0xffffffffu, np, o);
    }
    if (lane == 0) {
        atomicAdd(a.ntiles, nt);
        atomicAdd(&a.tested[loc], np);
    }
}

// FilteredIterator (iterator.rs:96-119) over one tile, in ONE pass: the tile's position bytes are staged in shared memory with
// 16-byte loads (node blocks and 2048-point tiles are 16-byte aligned), every point is decoded and tested once; per round of
// 256 points the block counts its survivors with ballots, reserves their output range with one atomic, stages them in shared
// memory and copies them out as contiguous words (the order inside a round is kept; rounds land in the order they finish -
// the batched form only promises per-location totals and the compacted set).  Survivors beyond `cap` are counted, not stored.
// STORE = false only counts: the survivors of every tile are added to kept[loc] and nothing is stored (`cursor`, `cap` and the
// outputs are unused), which is how a chunk of a directory-backed batched query is culled (dir_query.inl).
struct CullFusedArgs {
    CullArgs c;
    unsigned long long* cursor;  // output slots handed out so far
    unsigned long long cap;
    unsigned long long* kept;    // [nloc]
};
constexpr uint32_t kCullStage = kQueryTile * 12 + 32;  // F32 codes: the widest staged encoding
__device__ __forceinline__ void decode_staged(const uint8_t* s, uint32_t i, const QNode& nd, double p[3]) {
    if (nd.enc == ENC_U8) {
        const uint8_t* q = s + 3 * i;
#pragma unroll
        for (int k = 0; k < 3; ++k) p[k] = decode_axis<ENC_U8>(q[k], nd.m[k], nd.e);
    } else if (nd.enc == ENC_U16) {
        const uint16_t* q = reinterpret_cast<const uint16_t*>(s) + 3 * i;
#pragma unroll
        for (int k = 0; k < 3; ++k) p[k] = decode_axis<ENC_U16>(q[k], nd.m[k], nd.e);
    } else {
        const uint32_t* q = reinterpret_cast<const uint32_t*>(s) + 3 * i;
#pragma unroll
        for (int k = 0; k < 3; ++k) p[k] = decode_axis<ENC_F32>(q[k], nd.m[k], nd.e);
    }
}
// RGB = false (STORE only): the cloud has no colour, rgb / out_rgb are not touched (as in cull_tile).
template <bool STORE, bool RGB = true>
__global__ void __launch_bounds__(256) k_cull_fused(const __grid_constant__ CullFusedArgs f, uint32_t ntiles) {
    __shared__ __align__(16) uint8_t sxyz[kCullStage];
    // survivors of one round of 256 points, staged so that the copy-out is contiguous 8 / 4 / 1-byte-per-lane stores
    __shared__ __align__(16) double st_xyz[256 * 3];
    __shared__ uint32_t st_src[256];
    __shared__ float st_int[256];
    __shared__ uint8_t st_rgb[256 * 3];
    __shared__ uint32_t wcnt[8];
    __shared__ unsigned long long sbase;
    __shared__ uint64_t scells[kCellsShared];
    const CullArgs& a = f.c;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
        const QTile t = a.tiles[ti];
        const uint32_t loc = tile_loc(t);
        const QueryGeom& g = a.geoms[loc];
        const bool all_in = (t.loc & kTileIn) != 0;
        const QNode nd = a.nodes[t.node];
        const bool staged = nd.enc != ENC_F64;
        const int bpc = enc_bytes(nd.enc);
        const uint8_t* src = a.xyz + nd.xyz_off + (uint64_t)t.first * 3 * bpc;
        if (staged) {
            const uint32_t nvec = (t.count * 3u * (uint32_t)bpc + 15u) >> 4;
            for (uint32_t v = threadIdx.x; v < nvec; v += 256) reinterpret_cast<uint4*>(sxyz)[v] = __ldcg(reinterpret_cast<const uint4*>(src) + v);
        }
        const uint64_t* cells = stage_cells(g, scells);
        __syncthreads();
        uint32_t kept_tile = 0;  // thread 0 only
        for (uint32_t r0 = 0; r0 < t.count; r0 += 256) {
            const uint32_t i = r0 + threadIdx.x;
            bool keep = false;
            double p[3] = {0, 0, 0};
            if (i < t.count) {
                if (staged) {
                    decode_staged(sxyz, i, nd, p);
                } else {  // Float64, from global memory: decode_point's addressing would cost this kernel 4 registers
#pragma unroll
                    for (int k = 0; k < 3; ++k) p[k] = decode1_fast(load_code(src + ((size_t)i * 3 + k) * bpc, nd.enc), nd.m[k], nd.e, nd.enc);
                }
                keep = point_passes(a, g, cells, all_in, p, nd.point_off + t.first + i);
            }
            const unsigned bal = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) wcnt[warp] = __popc(bal);
            __syncthreads();
            if (!STORE) {
                if (threadIdx.x == 0)
                    for (int w = 0; w < 8; ++w) kept_tile += wcnt[w];
                __syncthreads();  // wcnt is reused by the next round
                continue;
            }
            uint32_t before = 0, total = 0;
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                const uint32_t c = wcnt[w];
                if (w < warp) before += c;
                total += c;
            }
            if (total == 0) {  // uniform: nothing survived this round
                __syncthreads();
                continue;
            }
            if (threadIdx.x == 0) {
                sbase = atomicAdd(f.cursor, (unsigned long long)total);  // one reservation per round: the round's survivors stay contiguous
                kept_tile += total;
            }
            if (keep) {
                const uint32_t li = before + __popc(bal & ((1u << lane) - 1u));
                const uint64_t sp = nd.point_off + t.first + i;
                st_xyz[3 * li] = p[0];
                st_xyz[3 * li + 1] = p[1];
                st_xyz[3 * li + 2] = p[2];
                if (RGB) {
                    st_rgb[3 * li] = a.rgb[3 * sp];
                    st_rgb[3 * li + 1] = a.rgb[3 * sp + 1];
                    st_rgb[3 * li + 2] = a.rgb[3 * sp + 2];
                }
                st_src[li] = a.src[sp];
                if (a.out_intensity) st_int[li] = a.intensity[sp];
            }
            __syncthreads();
            const unsigned long long base = sbase;
            const uint32_t room = base >= f.cap ? 0u : (uint32_t)min((unsigned long long)total, f.cap - base);
            for (uint32_t k = threadIdx.x; k < 3 * room; k += 256) a.out_xyz[3 * base + k] = st_xyz[k];
            if (RGB)
                for (uint32_t k = threadIdx.x; k < 3 * room; k += 256) a.out_rgb[3 * base + k] = st_rgb[k];
            for (uint32_t k = threadIdx.x; k < room; k += 256) {
                a.out_src[base + k] = st_src[k];
                if (a.out_intensity) a.out_intensity[base + k] = st_int[k];
            }
            __syncthreads();  // the staging arrays and wcnt are reused by the next round
        }
        if (threadIdx.x == 0 && kept_tile) atomicAdd(&f.kept[loc], (unsigned long long)kept_tile);
        __syncthreads();  // sxyz is reused by the next tile
    }
}

// ---- X-ray -----------------------------------------------------------------------------------------
// Pixels no point falls into get TRANSPARENT.to_u8() = (255, 255, 255, 0) (src/color.rs:154-159, generation.rs:506-511).
constexpr uint32_t kXrayTransparent = 0x00FFFFFFu;  // r | g << 8 | b << 16 | a << 24
__global__ void __launch_bounds__(256) k_fill_u32(uint32_t* __restrict__ dst, uint32_t value, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = value;
}
struct XrayArgs {
    QueryGeom geom;
    const QNode* nodes;
    const QTile* tiles;
    const uint8_t* xyz;
    double tmin[3], tdiag[3];
    double rdiag[3];  // RN(1 / tdiag) for div_known (chain.h): the correctly rounded quotient without the division instruction
    int div_ok;       // every tdiag is admissible for div_known (host check), else the IEEE operator
    double query_from_global[7];
    int has_q;
    uint32_t w, h;
    int* any;
};

// (p - tmin) / tdiag of one axis (process_point_data, generation.rs:108-127), bit-identical to the IEEE quotient
__device__ __forceinline__ double xray_unit(const XrayArgs& a, int k, double p) {
    const double d = p - a.tmin[k];
    return a.div_ok ? div_known(d, a.tdiag[k], a.rdiag[k]) : d / a.tdiag[k];
}

// Rust `f64 as u32`: truncating, saturating, NaN -> 0.  cvt.rzi.u32.f64 saturates but returns 0x80000000 for NaN (measured).
__device__ __forceinline__ uint32_t rust_as_u32_dev(double v) {
    const uint32_t u = __double2uint_rz(v);
    return v != v ? 0u : u;
}

// The pixel of a point that passed the tile's location test: p is moved into the quadtree's frame when the tile has a
// transform (generation.rs:493-497), then process_point_data (generation.rs:108-127) gives its column x, row y and z bucket.
// The point is drawn iff x < w && y < h.
__device__ __forceinline__ void xray_pixel(const XrayArgs& a, double p[3], uint32_t& x, uint32_t& y, uint32_t& z) {
    if (a.has_q) {
        const V3 q = iso_apply(a.query_from_global, V3{p[0], p[1], p[2]});
        p[0] = q.x, p[1] = q.y, p[2] = q.z;
    }
    x = rust_as_u32_dev(xray_unit(a, 0, p[0]) * (double)a.w);
    y = rust_as_u32_dev((1. - xray_unit(a, 1, p[1])) * (double)a.h);
    z = rust_as_u32_dev(xray_unit(a, 2, p[2]) * 1024.);
}

// The XRay strategy keeps a 1024-bit z-bucket set per pixel in SHARED memory (in global memory it would take 128 B per pixel:
// 2 GiB for a 4096 x 4096 tile).  The points are first binned by 32 x 32 pixel sub-tile of the image with a counting sort of
// 4-byte keys (k_xray_bin<0>: count, k_xray_bin<1>: place; octree nodes are spatially coherent, so the lanes of a warp mostly
// share their sub-tile and the atomics are issued once per warp and sub-tile), then one block per non-empty sub-tile
// (k_xray_subtile) ORs its keys into 1024 pixels x 1024 bits of shared memory (128 KB) and resolves them to RGBA itself.
constexpr uint32_t kXraySub = 32;  // sub-tile edge in pixels
struct XrayBinArgs {
    XrayArgs x;               // geom, nodes, tiles, xyz, tile box, transform, w, h
    uint32_t ntiles;
    uint32_t sub_w;           // sub-tiles per row
    uint32_t* sub_count;      // [nsub] points per sub-tile; after the scan: exclusive offsets
    uint32_t* sub_cursor;     // [nsub] place pass: keys written so far
    uint32_t* keys;           // ly << 16 | lx << 11 | min(z, 1024)
};
// The filter intervals of the octree X-ray kernels: point `slot` takes part iff lo <= (double)intensity[slot] <= hi for every
// interval (closed, the attribute as f64: iterator.rs:82-91, as point_passes and s2_leaf_hits test it).
struct XrayFilt {
    const float* intensity;  // node-contiguous intensities
    const pcv_interval* filters;
    uint32_t nfilt;
};
__device__ __forceinline__ bool xray_filt_pass(const XrayFilt& f, uint64_t slot) {
    const double v = (double)f.intensity[slot];
    for (uint32_t k = 0; k < f.nfilt; ++k)
        if (!(f.filters[k].lo <= v && v <= f.filters[k].hi)) return false;
    return true;
}
// The count (PLACE = 0) or place (PLACE = 1) pass over work tile t of the image of `a`: every point drawn into the image goes
// to bin bin0 + its sub-tile.  Returns whether one of the thread's points passed the location test.  FILT: only points that
// pass `f` take part (a point that fails gets no key and does not count as seen).
template <int PLACE, bool FILT = false>
__device__ __forceinline__ bool xray_bin_tile(const XrayArgs& a, const QNode* nodes, const uint8_t* xyz, const QTile t, uint32_t bin0, uint32_t sub_w,
                                              uint32_t* sub_count, uint32_t* sub_cursor, uint32_t* keys, const XrayFilt& f) {
    const int lane = threadIdx.x & 31;
    const QNode nd = nodes[t.node];
    const int bpc = enc_bytes(nd.enc);
    bool seen = false;
    for (uint32_t i0 = 0; i0 < t.count; i0 += blockDim.x) {
        const uint32_t i = i0 + threadIdx.x;
        uint32_t bin = 0xFFFFFFFFu, key = 0;
        if (i < t.count) {
            double p[3];
            decode_point(xyz, nd, bpc, t.first + i, p);
            if ((!FILT || xray_filt_pass(f, nd.point_off + t.first + i)) && loc_contains(a.geom, p[0], p[1], p[2])) {
                seen = true;
                uint32_t x, y, z;
                xray_pixel(a, p, x, y, z);
                if (x < a.w && y < a.h) {
                    bin = bin0 + (y / kXraySub) * sub_w + (x / kXraySub);
                    key = ((y % kXraySub) << 16) | ((x % kXraySub) << 11) | min(z, 1024u);
                }
            }
        }
        // one atomic per warp and distinct bin
        const unsigned mask = __match_any_sync(0xffffffffu, bin);
        if (bin != 0xFFFFFFFFu) {
            const int leader = __ffs(mask) - 1;
            const uint32_t rank = __popc(mask & ((1u << lane) - 1u));
            if (PLACE) {
                uint32_t base = 0;
                if (lane == leader) base = atomicAdd(&sub_cursor[bin], (uint32_t)__popc(mask));
                base = __shfl_sync(mask, base, leader);
                keys[sub_count[bin] + base + rank] = key;
            } else if (lane == leader) {
                atomicAdd(&sub_count[bin], (uint32_t)__popc(mask));
            }
        }
    }
    return seen;
}
template <int PLACE>
__global__ void __launch_bounds__(256) k_xray_bin(const __grid_constant__ XrayBinArgs b) {
    for (uint32_t ti = blockIdx.x; ti < b.ntiles; ti += gridDim.x)
        xray_bin_tile<PLACE>(b.x, b.x.nodes, b.x.xyz, b.x.tiles[ti], 0, b.sub_w, b.sub_count, b.sub_cursor, b.keys, XrayFilt{});
}
// The same binning for a batch of leaf tiles of one quadtree (the bounded quadtree driver, xray_api.inl): every work tile
// carries its leaf in `loc`, every leaf has its own location and box (leaves[loc]; transform, w and h are shared), and the bins
// are (leaf, sub-tile) pairs, leaf-major: bin = leaf * nsub + sub.  A point on an edge shared by two leaves goes into every
// leaf whose closed box contains it (the work list holds one tile per (leaf, node) pair).  The count pass also raises
// seen[leaf] for every point that passes the leaf's location test: the leaf exists iff one does (generation.rs:489-504).
// Several octrees bin into the same bins: each runs its count pass into sub_count, then after one scan its place pass through
// the shared sub_cursor (the keys of a bin may come in any order).  FILT: only points that pass `filt` take part.
struct XrayBatchArgs {
    const XrayArgs* leaves;   // [nleaf] geom, tmin, tdiag, rdiag, div_ok, query_from_global, has_q, w, h of every leaf
    const QNode* nodes;
    const QTile* tiles;
    const uint8_t* xyz;
    uint32_t ntiles;
    uint32_t sub_w, nsub;     // sub-tiles per row and per leaf
    uint32_t* sub_count;      // [nleaf * nsub + 1]; after the scan: exclusive offsets
    uint32_t* sub_cursor;     // [nleaf * nsub]
    uint32_t* keys;
    int* seen;                // [nleaf]
    XrayFilt filt;            // FILT only
};
template <int PLACE, bool FILT>
__global__ void __launch_bounds__(256) k_xray_bin_batch(const __grid_constant__ XrayBatchArgs b) {
    for (uint32_t ti = blockIdx.x; ti < b.ntiles; ti += gridDim.x) {
        const QTile t = b.tiles[ti];
        const bool seen = xray_bin_tile<PLACE, FILT>(b.leaves[t.loc], b.nodes, b.xyz, t, t.loc * b.nsub, b.sub_w, b.sub_count, b.sub_cursor, b.keys, b.filt);
        if (!PLACE && __syncthreads_or(seen) && threadIdx.x == 0) b.seen[t.loc] = 1;
    }
}
// Which candidate quadtree nodes of one level can hold a point (the pruning of the bounded quadtree driver).  Every point of
// the octree (interior nodes hold points too, so node cubes cannot tell an empty area from a full one) is decoded, moved
// into the quadtree's frame like k_xray_bin does, and marks every candidate whose cell - the level's grid over the quadtree
// rect, widened by `margin` on each side - contains it: at most four cells, found by binary search in the sorted candidates.
struct XrayOccupyArgs {
    const QNode* nodes;
    const QTile* tiles;       // every node's points
    const uint8_t* xyz;
    uint32_t ntiles;
    double query_from_global[7];
    int has_q;
    double x0, y0, edge;      // the quadtree rect's minimum, the edge of one node of the level
    double margin;
    uint32_t level;
    const unsigned long long* cand;  // sorted node indices of the level
    uint32_t ncand;
    uint32_t* hit;            // [ncand]
};
__host__ __device__ __forceinline__ void xray_cell_range(double v, double v0, double edge, double margin, uint64_t cells, int64_t& lo, int64_t& hi) {
    const double a = floor((v - margin - v0) / edge), b = floor((v + margin - v0) / edge);
    lo = 1, hi = 0;  // empty
    if (!(a == a) || !(b == b) || b < 0.0 || a >= (double)cells) return;
    lo = a < 0.0 ? 0 : (int64_t)a;
    hi = b >= (double)cells ? (int64_t)cells - 1 : (int64_t)b;
}
// The per-point arithmetic of the pruning, shared by k_xray_occupy and k_xray_occupy_cells: the decoded point p (global frame)
// moved into the quadtree's frame like k_xray_bin moves it, then the cells [x0, x1] x [y0, y1] of the level's grid (`cells`
// per side, cell `edge`, origin (gx, gy)) whose cell widened by `margin` contains it - at most 2 x 2 of them.
__host__ __device__ __forceinline__ void xray_point_cells(const double p_in[3], const double* qfg, double gx, double gy, double edge, double margin,
                                                          uint64_t cells, int64_t& x0, int64_t& x1, int64_t& y0, int64_t& y1) {
    double p[2] = {p_in[0], p_in[1]};
    if (qfg) {
        const V3 q = iso_apply(qfg, V3{p_in[0], p_in[1], p_in[2]});
        p[0] = q.x, p[1] = q.y;
    }
    xray_cell_range(p[0], gx, edge, margin, cells, x0, x1);
    xray_cell_range(p[1], gy, edge, margin, cells, y0, y1);
}
// quadtree child k: bit 1 -> +x, bit 0 -> +y (quadtree lib.rs:84-101): the index of cell (ix, iy) of a level
__host__ __device__ __forceinline__ uint64_t xray_quad_index(uint64_t ix, uint64_t iy, uint32_t level) {
    uint64_t idx = 0;
    for (uint32_t b = 0; b < level; ++b) idx |= (((ix >> b) & 1ull) << (2 * b + 1)) | (((iy >> b) & 1ull) << (2 * b));
    return idx;
}
__global__ void __launch_bounds__(256) k_xray_occupy(const __grid_constant__ XrayOccupyArgs a) {
    const uint64_t cells = 1ull << a.level;
    for (uint32_t ti = blockIdx.x; ti < a.ntiles; ti += gridDim.x) {
        const QTile t = a.tiles[ti];
        const QNode nd = a.nodes[t.node];
        const int bpc = enc_bytes(nd.enc);
        for (uint32_t i = threadIdx.x; i < t.count; i += blockDim.x) {
            double p[3];
            decode_point(a.xyz, nd, bpc, t.first + i, p);
            int64_t x0, x1, y0, y1;
            xray_point_cells(p, a.has_q ? a.query_from_global : nullptr, a.x0, a.y0, a.edge, a.margin, cells, x0, x1, y0, y1);
            for (int64_t ix = x0; ix <= x1; ++ix)
                for (int64_t iy = y0; iy <= y1; ++iy) {
                    const uint64_t idx = xray_quad_index((uint64_t)ix, (uint64_t)iy, a.level);
                    uint32_t l = 0, h = a.ncand;
                    while (l < h) {
                        const uint32_t m = (l + h) >> 1;
                        if (a.cand[m] < idx)
                            l = m + 1;
                        else
                            h = m;
                    }
                    if (l < a.ncand && a.cand[l] == idx && !a.hit[l]) a.hit[l] = 1;
                }
        }
    }
}
// The occupancy pass of the X-ray quadtree built from an on-disk octree (xray_dir.inl): one chunk of node files streamed
// through the device, every point marking the cells of one level (the leaves) exactly as k_xray_occupy marks candidates,
// into an open-addressing set of cell indices.  Only cells in [lo, hi] (the sub-root's subtree) are kept.  Index ~0 is the
// empty slot, so that one cell raises `last` instead; a set that is full raises `overflow` (the host empties it and runs the
// chunk again: inserting is idempotent).
struct XrayOccupyCellsArgs {
    const QNode* nodes;       // the chunk's nodes: cube, encoding, point count, offset of their positions in `xyz`
    const QTile* tiles;
    const uint8_t* xyz;
    uint32_t ntiles;
    double query_from_global[7];
    int has_q;
    double x0, y0, edge, margin;
    uint32_t level;
    unsigned long long lo, hi;
    unsigned long long* set;  // [mask + 1], ~0 = empty
    uint32_t mask;
    unsigned int* count;      // slots taken
    int* overflow;
    int* last;
};
__device__ __forceinline__ void occupy_insert(const XrayOccupyCellsArgs& a, unsigned long long key) {
    if (key == ~0ull) {
        *a.last = 1;
        return;
    }
    uint32_t h = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 32) & a.mask;
    for (uint32_t probe = 0; probe <= a.mask; ++probe, h = (h + 1) & a.mask) {
        const unsigned long long cur = *(volatile unsigned long long*)(a.set + h);
        if (cur == key) return;
        if (cur == ~0ull) {
            const unsigned long long prev = atomicCAS(a.set + h, ~0ull, key);
            if (prev == ~0ull) {
                atomicAdd(a.count, 1u);
                return;
            }
            if (prev == key) return;
        }
    }
    *a.overflow = 1;
}
__global__ void __launch_bounds__(256) k_xray_occupy_cells(const __grid_constant__ XrayOccupyCellsArgs a) {
    const uint64_t cells = 1ull << a.level;
    for (uint32_t ti = blockIdx.x; ti < a.ntiles; ti += gridDim.x) {
        const QTile t = a.tiles[ti];
        const QNode nd = a.nodes[t.node];
        const int bpc = enc_bytes(nd.enc);
        for (uint32_t i = threadIdx.x; i < t.count; i += blockDim.x) {
            double p[3];
            decode_point(a.xyz, nd, bpc, t.first + i, p);
            int64_t x0, x1, y0, y1;
            xray_point_cells(p, a.has_q ? a.query_from_global : nullptr, a.x0, a.y0, a.edge, a.margin, cells, x0, x1, y0, y1);
            for (int64_t ix = x0; ix <= x1; ++ix)
                for (int64_t iy = y0; iy <= y1; ++iy) {
                    const uint64_t idx = xray_quad_index((uint64_t)ix, (uint64_t)iy, a.level);
                    if (idx >= a.lo && idx <= a.hi) occupy_insert(a, idx);
                }
        }
    }
}
// The scan pass of the X-ray quadtree built from S2 directories (s2_dir_xray.inl): one chunk of cell pieces (a cell larger
// than a chunk is cut across chunks) streamed through the device, every position read once for two things: (a) the leaves it
// falls into, marked into the set as k_xray_occupy_cells marks them, and (b) the point box of its cell, reduced over
// f64_order_key as k_s2_cell_boxes reduces it (warp shuffles, then one atomic per warp and bound) into the slot of the cell's
// index in the directory-wide table.  Min and max do not depend on how cells are cut or in which order tiles meet, so the box
// is the one s2_location_tables computes for the loaded cloud, bit for bit.  Running a chunk again is idempotent.  MARK = false
// reduces the boxes only (the S2 directory handle, s2_dir_query.inl): the set and the leaf arguments of `occ` are unused.
struct S2DirScanArgs {
    XrayOccupyCellsArgs occ;   // nodes: the chunk's pieces as Float64 nodes (m = -0.0, e = 1); tiles: their work tiles
    const uint32_t* cell;      // [piece] its cell in the directory-wide table
    unsigned long long* kmin;  // [cell * 3 + axis], preset to ~0 / 0
    unsigned long long* kmax;
};
template <bool MARK>
__global__ void __launch_bounds__(256) k_s2_dir_scan(const __grid_constant__ S2DirScanArgs s) {
    const XrayOccupyCellsArgs& a = s.occ;
    const uint64_t cells = 1ull << a.level;
    for (uint32_t ti = blockIdx.x; ti < a.ntiles; ti += gridDim.x) {
        const QTile t = a.tiles[ti];
        const QNode nd = a.nodes[t.node];
        unsigned long long lo[3] = {~0ull, ~0ull, ~0ull}, hi[3] = {0ull, 0ull, 0ull};
        for (uint32_t i = threadIdx.x; i < t.count; i += blockDim.x) {
            double p[3];
            decode_point(a.xyz, nd, 8, t.first + i, p);  // Float64 node: the stored doubles, bit for bit
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const unsigned long long key = f64_order_key(p[k]);
                lo[k] = min(lo[k], key);
                hi[k] = max(hi[k], key);
            }
            if (!MARK) continue;
            int64_t x0, x1, y0, y1;
            xray_point_cells(p, a.has_q ? a.query_from_global : nullptr, a.x0, a.y0, a.edge, a.margin, cells, x0, x1, y0, y1);
            for (int64_t ix = x0; ix <= x1; ++ix)
                for (int64_t iy = y0; iy <= y1; ++iy) {
                    const uint64_t idx = xray_quad_index((uint64_t)ix, (uint64_t)iy, a.level);
                    if (idx >= a.lo && idx <= a.hi) occupy_insert(a, idx);
                }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                lo[k] = min(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
                hi[k] = max(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
            }
        if ((threadIdx.x & 31) == 0 && threadIdx.x < t.count) {
            const size_t c = s.cell[t.node];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                atomicMin(&s.kmin[3 * c + k], lo[k]);
                atomicMax(&s.kmax[3 * c + k], hi[k]);
            }
        }
    }
}
struct XraySubArgs {
    const uint32_t* sub_off;    // [nleaf * nsub + 1] exclusive offsets into keys
    const uint32_t* keys;
    const uint8_t* grey;        // [1026]
    uint8_t* rgba;              // nleaf images of w * h * 4, one after the other, pre-filled with TRANSPARENT
    uint32_t* zbits_out;        // optional (a single leaf): w * h * 32, zero-initialised
    uint32_t sub_w, w, h;
    uint32_t nsub;              // sub-tiles per leaf image: block b resolves sub-tile b % nsub of image b / nsub
};
__global__ void __launch_bounds__(512, 1) k_xray_subtile(const __grid_constant__ XraySubArgs b) {
    extern __shared__ __align__(16) uint32_t sbits[];  // [1024 pixels][32 words]
    __shared__ uint8_t sover[kXraySub * kXraySub];
    const uint32_t k0 = b.sub_off[blockIdx.x], k1 = b.sub_off[blockIdx.x + 1];
    if (k1 == k0) return;  // no point falls into this sub-tile: its pixels stay transparent (the image is pre-filled with TRANSPARENT)
    const uint32_t sid = blockIdx.x % b.nsub;
    uint8_t* const rgba = b.rgba + (size_t)(blockIdx.x / b.nsub) * b.w * b.h * 4;
    const uint32_t px0 = (sid % b.sub_w) * kXraySub, py0 = (sid / b.sub_w) * kXraySub;
    {
        uint4* z4 = reinterpret_cast<uint4*>(sbits);
        for (uint32_t i = threadIdx.x; i < kXraySub * kXraySub * 8; i += blockDim.x) z4[i] = make_uint4(0, 0, 0, 0);
    }
    for (uint32_t i = threadIdx.x; i < kXraySub * kXraySub; i += blockDim.x) sover[i] = 0;
    __syncthreads();
    auto put = [&](uint32_t key) {
        const uint32_t lp = (key >> 16) * kXraySub + ((key >> 11) & 31u), z = key & 2047u;
        if (z < 1024)
            atomicOr(&sbits[lp * 32 + (z >> 5)], 1u << (z & 31));
        else
            sover[lp] = 1;
    };
    uint32_t k = k0 + threadIdx.x;
    for (; k + 3 * blockDim.x < k1; k += 4 * blockDim.x) {  // four independent loads in flight per thread
        const uint32_t q0 = __ldcs(b.keys + k), q1 = __ldcs(b.keys + k + blockDim.x), q2 = __ldcs(b.keys + k + 2 * blockDim.x), q3 = __ldcs(b.keys + k + 3 * blockDim.x);
        put(q0), put(q1), put(q2), put(q3);
    }
    for (; k < k1; k += blockDim.x) put(__ldcs(b.keys + k));
    __syncthreads();
    // resolve: popcount of the pixel's bucket set -> grey (generation.rs:186-197)
    for (uint32_t lp = threadIdx.x; lp < kXraySub * kXraySub; lp += blockDim.x) {
        const uint32_t x = px0 + (lp % kXraySub), y = py0 + (lp / kXraySub);
        if (x >= b.w || y >= b.h) continue;
        uint32_t cnt = sover[lp];
#pragma unroll
        for (int k = 0; k < 32; ++k) cnt += __popc(sbits[lp * 32 + ((k + lp) & 31)]);  // rotated start: no 32-way bank conflict
        if (cnt) {
            const uint8_t gv = b.grey[cnt];
            reinterpret_cast<uchar4*>(rgba)[(size_t)y * b.w + x] = make_uchar4(gv, gv, gv, 255);
        }
        if (b.zbits_out) {
            uint32_t* o = b.zbits_out + ((size_t)y * b.w + x) * 32;
            for (int k = 0; k < 32; ++k) o[k] = sbits[lp * 32 + k];
        }
    }
}

// ------------------------------------------------------------------------------------------------
// The other colouring strategies of the X-ray tiles (xray/src/generation.rs:200-405), Binning = None:
//   1 point colour mean, 2 intensity mean (log-brightened), 3 height standard deviation through a colormap.
// The reference accumulates per column in arrival order (f32 sums, Welford in f64) and its batches arrive from several
// threads in unspecified order; here the columns are accumulated with atomics (f32 sums like the reference; for the
// variance, f64 sums of d = z - pivot and d^2 around a per-column pivot, the z of whichever point claims the column
// first), so results agree up to rounding.  A pivot inside the column keeps E[d^2] - E[d]^2 free of cancellation: around
// the tile's mid height, a 1 cm spread 1e6 m away lost every digit of its variance.
// ------------------------------------------------------------------------------------------------
struct XrayAttrArgs {
    XrayArgs x;
    const uint8_t* rgb;      // node-contiguous colours
    const float* intensity;  // node-contiguous intensities (mode 2)
    float* sum;              // mode 1: npix * 4; mode 2: npix
    double* dsum;            // mode 3: npix * 2
    unsigned long long* pivot;  // mode 3: npix, the bits of the column's pivot z; kPivotEmpty until a point claims it
    uint32_t* count;
    XrayFilt filt;           // FILT only
};
constexpr unsigned long long kPivotEmpty = 0x7FF8DEADBEEF0000ull;  // a NaN payload no decoded coordinate carries
// The column's pivot: the z of the first point to claim it with one CAS; every later point reads it.
__device__ __forceinline__ double xray_pivot(unsigned long long* slot, double z) {
    unsigned long long cur = *(volatile unsigned long long*)slot;
    if (cur == kPivotEmpty) {
        const unsigned long long prev = atomicCAS(slot, kPivotEmpty, (unsigned long long)__double_as_longlong(z));
        cur = prev == kPivotEmpty ? (unsigned long long)__double_as_longlong(z) : prev;
    }
    return __longlong_as_double((long long)cur);
}

// FILT: only points that pass b.filt take part (a point that fails adds nothing and does not count as seen).
template <int MODE, bool FILT>
__global__ void __launch_bounds__(256) k_xray_accum_attr(const __grid_constant__ XrayAttrArgs b) {
    const XrayArgs& a = b.x;
    const QTile t = a.tiles[blockIdx.x];
    const QNode nd = a.nodes[t.node];
    const int bpc = enc_bytes(nd.enc);
    bool seen = false;
    for (uint32_t i = threadIdx.x; i < t.count; i += blockDim.x) {
        double p[3];
        decode_point(a.xyz, nd, bpc, t.first + i, p);
        if (FILT && !xray_filt_pass(b.filt, nd.point_off + t.first + i)) continue;
        if (!loc_contains(a.geom, p[0], p[1], p[2])) continue;
        seen = true;
        uint32_t x, y, z;
        xray_pixel(a, p, x, y, z);
        if (!(x < a.w && y < a.h)) continue;
        const size_t px = (size_t)y * a.w + x;
        const uint64_t slot = nd.point_off + t.first + i;
        if (MODE == 1) {  // Color<u8>::to_f32: f32::from(c) / 255.
            const uint8_t* c = b.rgb + 3 * slot;
            atomicAdd(&b.sum[px * 4 + 0], (float)c[0] / 255.f);
            atomicAdd(&b.sum[px * 4 + 1], (float)c[1] / 255.f);
            atomicAdd(&b.sum[px * 4 + 2], (float)c[2] / 255.f);
            atomicAdd(&b.count[px], 1u);
        } else if (MODE == 2) {
            const float v = b.intensity[slot];
            if (v < 0.f) continue;
            atomicAdd(&b.sum[px], v);
            atomicAdd(&b.count[px], 1u);
        } else {
            const double d = p[2] - xray_pivot(&b.pivot[px], p[2]);
            atomicAdd(&b.dsum[px * 2], d);
            atomicAdd(&b.dsum[px * 2 + 1], d * d);
            atomicAdd(&b.count[px], 1u);
        }
    }
    if (__syncthreads_or(seen) && threadIdx.x == 0) atomicExch(a.any, 1);
}

__device__ __forceinline__ uint8_t f32_to_u8_dev(float v) {  // Color<f32>::to_u8: (v * 255.) as u8 (saturating, NaN -> 0)
    const float s = v * 255.f;
    if (!(s == s) || s <= 0.f) return 0;
    return s >= 255.f ? (uint8_t)255 : (uint8_t)s;
}
__device__ __forceinline__ float jet_base_dev(float val) {  // xray/src/colormap.rs:30-46
    if (val <= -0.75f) return 0.f;
    if (val <= -0.25f) return (val - -0.75f) * (1.0f - 0.0f) / (-0.25f - -0.75f) + 0.0f;
    if (val <= 0.25f) return 1.0f;
    if (val <= 0.75f) return (val - 0.25f) * (0.0f - 1.0f) / (0.75f - 0.25f) + 1.0f;
    return 0.0f;
}

__global__ void __launch_bounds__(256) k_xray_resolve_attr(int mode, float p0, float p1, int colormap, const float* __restrict__ sum,
                                                           const double* __restrict__ dsum, const uint32_t* __restrict__ count, uint32_t npix,
                                                           uint8_t* __restrict__ rgba) {
    const uint32_t px = blockIdx.x * blockDim.x + threadIdx.x;
    if (px >= npix) return;
    uchar4 o = make_uchar4(255, 255, 255, 0);  // TRANSPARENT.to_u8() (color.rs:154-159; generation.rs:506-511)
    const uint32_t n = count[px];
    if (n) {
        if (mode == 1) {
            o = make_uchar4(f32_to_u8_dev(sum[px * 4] / (float)n), f32_to_u8_dev(sum[px * 4 + 1] / (float)n), f32_to_u8_dev(sum[px * 4 + 2] / (float)n), 255);
        } else if (mode == 2) {
            float m = sum[px] / (float)n;
            m = fminf(fmaxf(m, p0), p1);
            const uint8_t g = f32_to_u8_dev(logf(m - p0) / logf(p1 - p0));
            o = make_uchar4(g, g, g, 255);
        } else {
            const double mean = dsum[px * 2] / (double)n;
            double var = dsum[px * 2 + 1] / (double)n - mean * mean;
            var = var > 0.0 ? var : 0.0;
            float sd = (float)sqrt(var);
            sd = sd < 0.f ? 0.f : (sd > p0 ? p0 : sd);
            const float val = sd / p0;
            if (colormap == 0)
                o = make_uchar4(f32_to_u8_dev(jet_base_dev(val - 0.5f)), f32_to_u8_dev(jet_base_dev(val)), f32_to_u8_dev(jet_base_dev(val + 0.5f)), 255);
            else
                o = make_uchar4(f32_to_u8_dev((1.0f - val) * 0.8f), f32_to_u8_dev((1.0f - val) * 0.8f), f32_to_u8_dev((1.0f - val) * 1.0f), 255);
        }
    }
    reinterpret_cast<uchar4*>(rgba)[px] = o;
}

// ------------------------------------------------------------------------------------------------
// /nodes_data blob (octree_web_viewer/src/backend.rs:92-165): gather the position and colour bytes of the requested
// nodes from their places in the octree arrays into one contiguous, 8-byte-padded reply buffer.
// ------------------------------------------------------------------------------------------------
// One work item = up to kBlobSeg destination bytes of one node part.  Destination offsets are multiples of 8 (the
// blob's padding rule); sources start at arbitrary byte offsets (a Uint8 node has 3 n bytes), so every destination word
// is assembled from two aligned source words with a funnel shift.  HBM-bound byte copy: 2 bytes moved per byte of reply.
struct BlobItem {
    uint64_t src;   // byte offset into the source array
    uint64_t dst;   // byte offset into the blob (multiple of 8)
    uint32_t bytes;
    uint32_t from_rgb;  // 0: position bytes, 1: colour bytes
};
constexpr uint32_t kBlobSeg = 32768;

__global__ void __launch_bounds__(256) k_blob_gather(const BlobItem* __restrict__ items, const uint8_t* __restrict__ xyz, const uint8_t* __restrict__ rgb,
                                                     uint8_t* __restrict__ blob) {
    const BlobItem it = items[blockIdx.x];
    const uint8_t* src = (it.from_rgb ? rgb : xyz) + it.src;
    uint32_t* dst = reinterpret_cast<uint32_t*>(blob + it.dst);
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3), sh = mis * 8;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(src - mis);
    const uint32_t nwords = it.bytes / 4;
    for (uint32_t i = threadIdx.x; i < nwords; i += blockDim.x) {
        const uint32_t lo = __ldg(w + i);
        const uint32_t hi = mis ? __ldg(w + i + 1) : 0u;  // never read a word the source range does not touch
        dst[i] = __funnelshift_r(lo, hi, sh);
    }
    // the last 0..3 bytes; the blob's zero padding is written by the host-side memset of the reply buffer
    if (threadIdx.x < (it.bytes & 3u)) blob[it.dst + 4ull * nwords + threadIdx.x] = src[4ull * nwords + threadIdx.x];
}

}  // namespace pcv
