// kernels_build.cuh — sm_90a kernels of the octree build and the CUDA Backend that drives them.
//
//   k_bbox      a1  find_bounding_box (generation.rs:256-270): streaming min/max, warp-shuffle reduce
//   k_ingest    a3-a6  raw position -> first step of the chain (chain.h): level-1 codes + the first pass's digits
//   k_dighist   digit histogram of every tile of a pass (1 byte per point)
//   k_scan_*    per-digit exclusive prefix over the tiles of each active node (+ node totals)
//   k_plan      a4  should_split_node for all descendants of the pass, bucket tables, node table, next active list
//   k_pass      a3-a6  stable multi-way partition of a tile by the carried digits (warp match ranking), then - in
//                   destination order - the codes each destination stores and the next pass's descent
//   k_place     a7  closed-form LOD subsampling + up-chain re-encode + final node-contiguous store
//
// All of them stream SoA/record arrays once with coalesced accesses; none has a dense contraction,
// so there is no tensor-core path here.  The descent is FP64 (IEEE divide + FMA) by definition of
// the reference's codec, compiled with -fmad=false.
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <type_traits>
#include <unordered_map>

#include "build_host.hpp"
#include "chain_device.cuh"

namespace pcv {

#define PCV_CUDA_CHECK(x)                                                                            \
    do {                                                                                             \
        cudaError_t e_ = (x);                                                                        \
        if (e_ != cudaSuccess) throw ::pcv::BuildError(-2, std::string("CUDA: ") + cudaGetErrorString(e_) + " at " #x); \
    } while (0)

// ------------------------------------------------------------------------------------------------
// bbox
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// partial[block][6] = min xyz, max xyz.  Grid-stride, 4 independent loads in flight per coordinate.
__global__ void __launch_bounds__(256) k_bbox(PointsView p, double* __restrict__ partial) {
    double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t s = p.stride;
    for (; i + 3 * step < p.n; i += 4 * step) {
        double vx[4], vy[4], vz[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            vx[u] = __ldg(p.x + (i + u * step) * s);
            vy[u] = __ldg(p.y + (i + u * step) * s);
            vz[u] = __ldg(p.z + (i + u * step) * s);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            mn[0] = fmin(mn[0], vx[u]);
            mx[0] = fmax(mx[0], vx[u]);
            mn[1] = fmin(mn[1], vy[u]);
            mx[1] = fmax(mx[1], vy[u]);
            mn[2] = fmin(mn[2], vz[u]);
            mx[2] = fmax(mx[2], vz[u]);
        }
    }
    for (; i < p.n; i += step) {
        double x = __ldg(p.x + i * s), y = __ldg(p.y + i * s), z = __ldg(p.z + i * s);
        mn[0] = fmin(mn[0], x);
        mx[0] = fmax(mx[0], x);
        mn[1] = fmin(mn[1], y);
        mx[1] = fmax(mx[1], y);
        mn[2] = fmin(mn[2], z);
        mx[2] = fmax(mx[2], z);
    }
    __shared__ double sh[8][6];
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        double lo = warp_min(mn[a]), hi = warp_max(mx[a]);
        if (l == 0) {
            sh[w][a] = lo;
            sh[w][3 + a] = hi;
        }
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        double v = sh[0][threadIdx.x];
        for (int k = 1; k < 8; ++k) v = threadIdx.x < 3 ? fmin(v, sh[k][threadIdx.x]) : fmax(v, sh[k][threadIdx.x]);
        partial[blockIdx.x * 6 + threadIdx.x] = v;
    }
}

// ------------------------------------------------------------------------------------------------
// record load / store helpers
// ------------------------------------------------------------------------------------------------
template <bool WIDE>
struct RecT;
template <>
struct RecT<false> {
    typedef RecN type;
};
template <>
struct RecT<true> {
    typedef RecW type;
};

template <bool WIDE>
__device__ __forceinline__ void store_rec(void* base, uint64_t i, const uint64_t c[3], uint32_t idx) {
    if (WIDE) {
        ulonglong2 v0, v1;
        v0.x = c[0];
        v0.y = c[1];
        v1.x = c[2];
        v1.y = idx;
        ulonglong2* p = reinterpret_cast<ulonglong2*>(base) + 2 * i;
        p[0] = v0;
        p[1] = v1;
    } else {
        uint4 v;
        v.x = (uint32_t)c[0];
        v.y = (uint32_t)c[1];
        v.z = (uint32_t)c[2];
        v.w = idx;
        reinterpret_cast<uint4*>(base)[i] = v;
    }
}

// ------------------------------------------------------------------------------------------------
// shared-memory / TMA helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.release.cta.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_load(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes),
                 "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred P;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
            "selp.b32 %0, 1, 0, P;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}

template <bool WIDE>
__device__ __forceinline__ void smem_load_rec(const unsigned char* srec, uint32_t i, uint64_t c[3], uint32_t& idx) {
    if (WIDE) {
        const ulonglong2* p = reinterpret_cast<const ulonglong2*>(srec) + 2 * (size_t)i;
        const ulonglong2 v0 = p[0], v1 = p[1];
        c[0] = v0.x, c[1] = v0.y, c[2] = v1.x, idx = (uint32_t)v1.y;
    } else {
        const uint4 v = reinterpret_cast<const uint4*>(srec)[i];
        c[0] = v.x, c[1] = v.y, c[2] = v.z, idx = v.w;
    }
}

// ------------------------------------------------------------------------------------------------
// ingest: raw points -> level-1 records + the first pass's digits
// ------------------------------------------------------------------------------------------------
// One block per 4096-point tile of the input (grid-stride).  Per point: the first step of the chain from the raw position
// (child digit of the root cube, codes in the level-1 cube) and, when the first pass resolves two levels, the level-2
// digit of the re-decoded position.  The tile's rgb bytes are staged with aligned 16-byte loads and repacked four points
// at a time (3-byte-strided per-thread loads are LSU-hostile); everything is written in input order, fully coalesced.
constexpr int kIngestThreads = 256;
constexpr size_t kRgbStage = (size_t)kTilePoints * 3 + 32;

// The coordinates of kIngestBatch points per thread are requested before the first of them is processed: the kernel is a
// stream (27 B in, 21 B out per point) and lives on loads in flight, not on arithmetic.
template <bool WIDE, int FAST, int kIngestBatch>
__device__ __forceinline__ unsigned ingest_tile(const IngestArgs& a, uint64_t start, uint32_t count, const uint32_t* scol) {
    unsigned bad = 0;
    const double e0 = a.lv.edge[0], e1 = a.lv.edge[1], ry1 = a.lv.ry[1];
    for (uint32_t i0 = threadIdx.x; i0 < count; i0 += kIngestThreads * kIngestBatch) {
      double qq[kIngestBatch][3];
#pragma unroll
      for (int u = 0; u < kIngestBatch; ++u) {
          const uint32_t i = i0 + u * kIngestThreads;
          const uint64_t g = start + (i < count ? i : i0);
          // streamed once: bypass L1 (ld.global.cg)
          qq[u][0] = __ldcg(a.pts.x + g * a.pts.stride);
          qq[u][1] = __ldcg(a.pts.y + g * a.pts.stride);
          qq[u][2] = __ldcg(a.pts.z + g * a.pts.stride);
      }
#pragma unroll
      for (int u = 0; u < kIngestBatch; ++u) {
        const uint32_t i = i0 + u * kIngestThreads;
        if (i >= count) break;
        const uint64_t g = start + i;
        double q[3] = {qq[u][0], qq[u][1], qq[u][2]}, m[3] = {a.root_min[0], a.root_min[1], a.root_min[2]};
        if (FAST == 2) bad |= input_bad(q[0]) | input_bad(q[1]) | input_bad(q[2]);
        typename std::conditional<WIDE, uint64_t, uint32_t>::type code[3];
        unsigned dig = 0;
        if (a.G0 == 2) {
            PCV_ENC_SWITCH(a.lv.enc[1], dig = level_step<ENC, FAST, true>(q, m, e0, e1, ry1, code, bad);)
            dig = (dig << 3) | level_digit(q, m, e1);
        } else {
            PCV_ENC_SWITCH(a.lv.enc[1], dig = level_step<ENC, FAST, false>(q, m, e0, e1, ry1, code, bad);)
        }
        const uint64_t c64[3] = {(uint64_t)code[0], (uint64_t)code[1], (uint64_t)code[2]};
        store_rec<WIDE>(a.rec_out, g, c64, (uint32_t)g);
        a.col_out[g] = scol[i];
        a.dig_out[g] = (uint8_t)dig;
      }
    }
    return bad;
}

template <bool WIDE, int FASTMODE, int BATCH>  // FASTMODE = LevelTable::fast (a kernel per mode keeps the register budget for the loads in flight)
__global__ void __launch_bounds__(kIngestThreads, 4) k_ingest(const __grid_constant__ IngestArgs a) {
    __shared__ __align__(16) uint8_t srgb[kRgbStage];
    __shared__ __align__(16) uint32_t scol[kTilePoints];
    const int tid = threadIdx.x;
    for (uint32_t tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
        const uint64_t start = (uint64_t)tile * kTilePoints;
        const uint64_t rem = a.pts.n - start;
        const uint32_t count = (uint32_t)(rem < kTilePoints ? rem : kTilePoints);
        {
            const uint8_t* g0 = a.pts.rgb + 3 * start;
            const uint32_t nbytes = 3 * count;
            const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(g0) & 15);  // srgb[mis + k] = g0[k]
            const uint8_t* ga = g0 - mis;
            const uint32_t nvec = (mis + nbytes + 15) / 16;
            for (uint32_t v = tid; v + 1 < nvec; v += kIngestThreads) reinterpret_cast<uint4*>(srgb)[v] = __ldcg(reinterpret_cast<const uint4*>(ga) + v);
            if (tid < 16) {  // the last vector byte-wise: never read past the array's last byte
                const uint32_t k = (nvec - 1) * 16 + tid;
                if (k >= mis && k < mis + nbytes) srgb[k] = __ldg(ga + k);
            }
            __syncthreads();
            // colours of 4 consecutive points are 12 staged bytes: 4 aligned words, funnel-shifted by the misalignment, give
            // the 4 packed colours with one 16-byte store
            const uint32_t* w = reinterpret_cast<const uint32_t*>(srgb);
            for (uint32_t k = tid; 4 * k < count; k += kIngestThreads) {
                const uint32_t byte0 = mis + 12 * k, wi = byte0 >> 2, sh = (byte0 & 3) * 8;
                const uint32_t w0 = w[wi], w1 = w[wi + 1], w2 = w[wi + 2], w3 = w[wi + 3];
                const uint32_t a0 = __funnelshift_r(w0, w1, sh), a1 = __funnelshift_r(w1, w2, sh), a2 = __funnelshift_r(w2, w3, sh);
                uint4 c;  // a0 = r0 g0 b0 r1 | a1 = g1 b1 r2 g2 | a2 = b2 r3 g3 b3 (little endian)
                c.x = a0 & 0xFFFFFFu;
                c.y = (a0 >> 24) | ((a1 & 0xFFFFu) << 8);
                c.z = (a1 >> 16) | ((a2 & 0xFFu) << 16);
                c.w = a2 >> 8;
                reinterpret_cast<uint4*>(scol)[k] = c;
            }
            __syncthreads();
        }
        if (FASTMODE == 3) {
            ingest_tile<WIDE, 3, BATCH>(a, start, count, scol);  // power-of-two edges: exact for every input, nothing to repeat
        } else if (FASTMODE) {
            const unsigned bad = ingest_tile<WIDE, FASTMODE, BATCH>(a, start, count, scol);
            if (__syncthreads_or((int)bad)) ingest_tile<WIDE, 0, BATCH>(a, start, count, scol);  // a numerator outside the proven range: IEEE operator (same stores)
        } else {
            ingest_tile<WIDE, 0, BATCH>(a, start, count, scol);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// digit histogram of a pass's tiles (1 byte per point) + per-digit prefix over the tiles of every active node
// ------------------------------------------------------------------------------------------------
// tile -> active node (written once per pass from the scan chunks): a block learns its tile with two loads instead of a
// binary search of dependent loads over the active list
__global__ void k_tile_index(const __grid_constant__ PassArgs a) {
    const uint32_t nchunks = a.st->pass[a.pass].nchunks;
    for (uint32_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
        const ChunkDesc c = a.chunks[ch];
        for (uint32_t t = threadIdx.x; t < c.ntiles; t += blockDim.x) a.tile_active[c.tile_begin + t] = c.active;
    }
}
__device__ __forceinline__ TileDesc tile_lookup(const PassArgs& a, uint32_t tile) {
    const uint32_t i = a.tile_active[tile];
    const ActiveDesc& act = a.active[i];
    const uint64_t o = (uint64_t)(tile - act.tile_begin) * kTilePoints;
    const uint64_t rem = act.count - o;
    return TileDesc{act.start + o, (uint32_t)(rem < kTilePoints ? rem : kTilePoints), i};
}

// One warp per tile, no block-level synchronisation: 64 bytes of digits per lane (four independent 16-byte loads in flight),
// warp-private histogram in shared memory.
constexpr int kDigThreads = 256;
__global__ void __launch_bounds__(kDigThreads) k_dighist(const __grid_constant__ PassArgs a) {
    __shared__ uint32_t hs[kDigThreads / 32][64];
    const PassState ps = a.st->pass[a.pass];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* h = hs[warp];
    const uint32_t nwarps = gridDim.x * (kDigThreads / 32);
    for (uint32_t tile = blockIdx.x * (kDigThreads / 32) + warp; tile < ps.ntiles; tile += nwarps) {
        const TileDesc t = tile_lookup(a, tile);
        h[lane] = 0;
        h[lane + 32] = 0;
        __syncwarp();
        // aligned 16-byte loads over the covering range, bytes outside [start, start + count) masked
        const uint64_t lo = t.start, hi = t.start + t.count, base = lo & ~(uint64_t)15;
        const uint32_t nvec = (uint32_t)((hi - base + 15) >> 4);  // <= 129
        uint4 w[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const uint32_t v = lane + 32 * k;
            w[k] = make_uint4(0, 0, 0, 0);
            if (v < nvec) w[k] = __ldcg(reinterpret_cast<const uint4*>(a.dig_in + base + 16ull * v));
        }
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            const uint32_t v = lane + 32 * k;
            if (v < nvec) {
                const uint64_t p0 = base + 16ull * v;
                const uint32_t ws[4] = {w[k].x, w[k].y, w[k].z, w[k].w};
                if (p0 >= lo && p0 + 16 <= hi) {
#pragma unroll
                    for (int j = 0; j < 16; ++j) atomicAdd(&h[(ws[j >> 2] >> (8 * (j & 3))) & 63u], 1u);
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const uint64_t p = p0 + j;
                        if (p >= lo && p < hi) atomicAdd(&h[(ws[j >> 2] >> (8 * (j & 3))) & 63u], 1u);
                    }
                }
            }
        }
        __syncwarp();
        uint32_t* out = a.tile_counts + (size_t)tile * a.nbins;
        if (lane < a.nbins) out[lane] = h[lane];
        if (lane + 32 < a.nbins) out[lane + 32] = h[lane + 32];
        __syncwarp();
    }
}

__global__ void k_scan_chunk_sums(const __grid_constant__ PassArgs a) {
    const uint32_t nchunks = a.st->pass[a.pass].nchunks;
    for (uint32_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
        const ChunkDesc c = a.chunks[ch];
        for (int b = threadIdx.x; b < a.nbins; b += blockDim.x) {
            uint32_t s = 0;
            const uint32_t* p = a.tile_counts + (size_t)c.tile_begin * a.nbins + b;
#pragma unroll 8
            for (uint32_t t = 0; t < c.ntiles; ++t) s += p[(size_t)t * a.nbins];
            a.chunk_sums[(size_t)ch * a.nbins + b] = s;
        }
    }
}
__global__ void k_scan_nodes(const __grid_constant__ PassArgs a) {
    const uint32_t nactive = a.st->pass[a.pass].nactive;
    for (uint32_t n = blockIdx.x; n < nactive; n += gridDim.x) {
        const ActiveDesc act = a.active[n];
        for (int b = threadIdx.x; b < a.nbins; b += blockDim.x) {
            uint64_t run = 0;
            uint32_t* p = a.chunk_sums + (size_t)act.chunk_begin * a.nbins + b;
            uint32_t c = 0;
            for (; c + 8 <= act.nchunks; c += 8) {  // eight independent loads in flight, then the dependent prefix
                uint32_t v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) v[u] = p[(size_t)(c + u) * a.nbins];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    p[(size_t)(c + u) * a.nbins] = (uint32_t)run;
                    run += v[u];
                }
            }
            for (; c < act.nchunks; ++c) {
                uint32_t v = p[(size_t)c * a.nbins];
                p[(size_t)c * a.nbins] = (uint32_t)run;
                run += v;
            }
            a.node_bins[(size_t)n * a.nbins + b] = run;
        }
    }
}
__global__ void k_scan_tiles(const __grid_constant__ PassArgs a) {
    const uint32_t nchunks = a.st->pass[a.pass].nchunks;
    for (uint32_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
        const ChunkDesc c = a.chunks[ch];
        for (int b = threadIdx.x; b < a.nbins; b += blockDim.x) {
            uint32_t run = a.chunk_sums[(size_t)ch * a.nbins + b];
            uint32_t* p = a.tile_counts + (size_t)c.tile_begin * a.nbins + b;
            uint32_t t = 0;
            for (; t + 8 <= c.ntiles; t += 8) {
                uint32_t v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) v[u] = p[(size_t)(t + u) * a.nbins];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    p[(size_t)(t + u) * a.nbins] = run;
                    run += v[u];
                }
            }
            for (; t < c.ntiles; ++t) {
                uint32_t v = p[(size_t)t * a.nbins];
                p[(size_t)t * a.nbins] = run;
                run += v;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// plan: leaf / split decisions, bucket tables, node table, next pass's active list - one block, no host round trip
// ------------------------------------------------------------------------------------------------
// Three small kernels: per-active-node demand (many blocks: the per-node logic diverges, so it is spread over the SMs), an
// exclusive scan of the demands in one block, and the emission with every node's bases.
constexpr int kPlanThreads = 1024;
constexpr int kPlanNodeThreads = 32;
__device__ __forceinline__ uint64_t block_excl_scan(uint64_t v, uint64_t* sh /* [33] */, uint64_t& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    __syncthreads();  // sh may still be read from the previous call
    if (lane == 31) sh[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint64_t w = sh[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t u = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += u;
        }
        sh[lane] = wi - w;
        if (lane == 31) sh[32] = wi;
    }
    __syncthreads();
    total = sh[32];
    return incl - v + sh[warp];
}

__global__ void __launch_bounds__(kPlanNodeThreads) k_plan_count(const __grid_constant__ PassArgs a) {
    const PassState ps = a.st->pass[a.pass];
    for (uint32_t ai = blockIdx.x * kPlanNodeThreads + threadIdx.x; ai < ps.nactive; ai += gridDim.x * kPlanNodeThreads) {
        PlanRun t{};
        int32_t err = 0;
        uint32_t deepest = 0;
        plan_active<false>(a, ai, t, err, deepest);
        a.plan_runs[ai] = t;
        if (err) atomicMax(&a.st->plan_error, err);
        if (deepest) atomicMax(&a.st->deepest_level, deepest);
    }
}

__global__ void __launch_bounds__(kPlanThreads) k_plan_scan(const __grid_constant__ PassArgs a) {
    __shared__ uint64_t sh[33];
    BuildState* st = a.st;
    const PassState ps = st->pass[a.pass];
    PlanRun carry;  // global bases of this pass
    carry.nodes = st->nnodes;
    carry.actives = 0, carry.tiles = 0, carry.chunks = 0;
    carry.next_pts = 0;
    carry.arena_pts = st->arena_used;
    const int32_t err_in = st->plan_error;
    __syncthreads();
    for (uint32_t base = 0; base < ps.nactive; base += kPlanThreads) {
        const uint32_t ai = base + threadIdx.x;
        PlanRun t{};
        if (ai < ps.nactive) t = a.plan_runs[ai];
        uint64_t tot[6];
        PlanRun b;
        b.nodes = carry.nodes + (uint32_t)block_excl_scan(t.nodes, sh, tot[0]);
        b.actives = carry.actives + (uint32_t)block_excl_scan(t.actives, sh, tot[1]);
        b.tiles = carry.tiles + (uint32_t)block_excl_scan(t.tiles, sh, tot[2]);
        b.chunks = carry.chunks + (uint32_t)block_excl_scan(t.chunks, sh, tot[3]);
        b.next_pts = carry.next_pts + block_excl_scan(t.next_pts, sh, tot[4]);
        b.arena_pts = carry.arena_pts + block_excl_scan(t.arena_pts, sh, tot[5]);
        if (ai < ps.nactive) a.plan_runs[ai] = b;  // the node's bases
        carry.nodes += (uint32_t)tot[0];
        carry.actives += (uint32_t)tot[1];
        carry.tiles += (uint32_t)tot[2];
        carry.chunks += (uint32_t)tot[3];
        carry.next_pts += tot[4];
        carry.arena_pts += tot[5];
    }
    if (threadIdx.x == 0) {
        int32_t err = err_in;
        // capacities are checked on the totals (the emit kernel guards its own writes as well)
        if (!err && (carry.nodes > a.cap_nodes || carry.actives > a.cap_active || carry.tiles > a.cap_tiles || carry.chunks > a.cap_chunks)) err = kErrCapacity;
        const bool failed = err != 0 || st->error != 0;
        if (err && !st->error) st->error = err;
        PassState nx{};
        if (!failed) {
            nx.nactive = carry.actives;
            nx.ntiles = carry.tiles;
            nx.nchunks = carry.chunks;
            nx.npoints = carry.next_pts;
        }
        st->pass[a.pass + 1] = nx;  // an error stops the following passes: no active nodes
        st->nnodes = carry.nodes;
        st->arena_used = carry.arena_pts;
    }
}

__global__ void __launch_bounds__(kPlanNodeThreads) k_plan_emit(const __grid_constant__ PassArgs a) {
    const PassState ps = a.st->pass[a.pass];
    for (uint32_t ai = blockIdx.x * kPlanNodeThreads + threadIdx.x; ai < ps.nactive; ai += gridDim.x * kPlanNodeThreads) {
        PlanRun b = a.plan_runs[ai];
        int32_t e2 = 0;
        uint32_t d2 = 0;
        plan_active<true>(a, ai, b, e2, d2);
    }
}

// ------------------------------------------------------------------------------------------------
// subsample plan (build_host.hpp finish_node / finish_emit): one small launch per level, bottom-up, then one block that scans
// the nodes in creation order (output offsets, leaf ordinals, first placement tile of every leaf) and leaves the totals in the
// build state
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sub_level(const __grid_constant__ FinishArgs f) {
    const uint32_t n = f.st->nnodes;
    if (f.st->error) return;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (f.nodes[i].level == f.level) finish_node(f, i);
}
// exclusive block scan of K values per thread at once (one set of barriers)
template <int K>
__device__ __forceinline__ void block_excl_scan_k(uint64_t (&v)[K], uint64_t (*sh)[33], uint64_t (&total)[K]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t incl[K];
#pragma unroll
    for (int q = 0; q < K; ++q) {
        incl[q] = v[q];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t u = __shfl_up_sync(0xffffffffu, incl[q], o);
            if (lane >= o) incl[q] += u;
        }
    }
    __syncthreads();  // sh may still be read from the previous call
    if (lane == 31) {
#pragma unroll
        for (int q = 0; q < K; ++q) sh[q][warp] = incl[q];
    }
    __syncthreads();
    if (warp < K) {
        uint64_t w = sh[warp][lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t u = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += u;
        }
        sh[warp][lane] = wi - w;
        if (lane == 31) sh[warp][32] = wi;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < K; ++q) {
        total[q] = sh[q][32];
        v[q] = incl[q] - v[q] + sh[q][warp];
    }
}

__global__ void __launch_bounds__(kPlanThreads) k_sub_layout(const __grid_constant__ FinishArgs f) {
    __shared__ uint64_t sh[5][33];
    BuildState* st = f.st;
    const uint32_t n = st->error ? 0u : st->nnodes;
    uint64_t c_pts = 0, c_xyz = 0, c_leaf = 0, c_tile = 0, c_algo = 0;
    for (uint32_t base = 0; base < n; base += kPlanThreads) {
        const uint32_t i = base + threadIdx.x;
        uint64_t fc = 0, b = 0, leaf = 0, tiles = 0;
        if (i < n) {
            fc = f.final_count[i];
            b = finish_xyz_bytes(f, i);
            if (f.nodes[i].leaf) {
                leaf = 1;
                tiles = (f.nodes[i].count + kPlaceTile - 1) / kPlaceTile;
            }
        }
        uint64_t tot[5], v[5] = {fc, (b + 15) & ~15ull, leaf, tiles, b};
        block_excl_scan_k<5>(v, sh, tot);
        const uint64_t o_pts = c_pts + v[0], o_xyz = c_xyz + v[1], o_leaf = c_leaf + v[2], o_tile = c_tile + v[3];
        if (i < n) {
            finish_emit(f, i, o_pts, o_xyz, (uint32_t)o_leaf, (uint32_t)o_tile);
            if (i == n - 1) st->xyz_bytes = o_xyz + b;
        }
        c_pts += tot[0], c_xyz += tot[1], c_leaf += tot[2], c_tile += tot[3], c_algo += tot[4];
    }
    if (threadIdx.x == 0) {
        f.leaf_tile_begin[c_leaf] = (uint32_t)c_tile;
        st->nleaves = (uint32_t)c_leaf;
        st->place_tiles = (uint32_t)c_tile;
        st->out_points = c_pts;
        st->algo_xyz = c_algo;
        if (n == 0) st->xyz_bytes = 0;
    }
}

// ------------------------------------------------------------------------------------------------
// pass: stable multi-way partition of every tile + the next pass's descent, in destination order
// ------------------------------------------------------------------------------------------------
// Persistent blocks of 8 warps, four per SM (independent barrier domains that cover each other's phases), tiles of 1792
// points taken round robin.  Warp w owns the contiguous items [224 w, 224 w + 224) of the tile.
//   stage    TMA bulk copies (cp.async.bulk global -> shared, completion on mbarriers) in two groups: the small part a tile's
//            ranking needs - its digits, its row of the per-digit prefix table and its node's bucket table, 3 KB, double
//            buffered and requested a whole tile ahead - and the big part only the finish sweep needs - records and colours,
//            36 KB, requested as soon as the previous tile's finish sweep has released the buffer, so that it lands while the
//            tile is being ranked and sorted.  The node of the NEXT tile is looked up during the current one (tile index table
//            + an asynchronous copy of the active-list entry): no global-memory latency sits on the path between two tiles
//   tables   64 threads: per bucket the slot of this tile's first record (bucket start + the node's earlier tiles) and the
//            digit -> bucket map
//   rank     per item only the carried digit -> bucket look-up; lanes grouped by bucket with __match_any_sync, per-warp
//            bucket counts; no arithmetic on positions at all
//   scan     (one warp) per-bucket totals, exclusive prefix over the buckets (sorted start inside the tile) and over the warps;
//            per bucket the three store base addresses, so that a store address is base + sorted position * size
//   sort     every warp walks its items in order and writes (item, bucket) at the item's stable sorted position: the tile is
//            sorted by bucket as a permutation in shared memory
//   finish   consecutive threads take consecutive sorted positions, i.e. consecutive slots of a destination run: a leaf at
//            level L+1 stores the carried codes as they are; a destination at level L+2 gets one encode step; a record that
//            continues is decoded once more and runs the first step (and second digit) of the NEXT pass, whose codes and
//            digits travel with it.  Threads of a warp share their destination kind except at run boundaries, so the FP64
//            work is not divergent, and every store is part of a contiguous run (records 16 B, colours 4 B, digits 1 B).
// The order inside every bucket is the tile order, i.e. input order (stable).
template <bool WIDE>
struct PassCfg {
    static constexpr int threads = 256;
    static constexpr int warps = threads / 32;
    static constexpr int warp_items = kTilePoints / warps;  // 224
    static constexpr int sub_rounds = warp_items / 32;      // 7
    static constexpr int blocks_per_sm = WIDE ? 2 : 4;
    static_assert(warps * sub_rounds * 32 == (int)kTilePoints, "the tile must be a whole number of sub-rounds per warp");
};
constexpr int kPassBins = 64;
struct PassBucket {  // per bucket of the current tile (shared memory, 32 bytes)
    unsigned long long rec, col, dig;  // store address of sorted position 0 (the bucket's run starts at `start`)
    uint32_t start;                    // sorted position of the bucket's first record
    uint32_t kk;                       // keep | leaf << 8
};
struct PassBucketExt {  // fused exchange pass: what a bucket needs beyond PassBucket
    unsigned long long inten;  // store address of sorted position 0 in the owner's intensity array (indexed by slot)
    uint32_t slot0;            // slot of sorted position 0 (mod 2^32)
    uint32_t pad;
};
template <bool WIDE>
struct PassSmem {
    static constexpr size_t rec_bytes = WIDE ? 32 : 16;
    // big part of a staged tile: records + colours (single buffer)
    static constexpr size_t off_col = (size_t)kTilePoints * rec_bytes;
    static constexpr size_t big_bytes = off_col + ((size_t)kTilePoints + 4) * 4;
    // small part: digits + prefix row + bucket table (two buffers)
    static constexpr size_t sm_pfx = (size_t)kTilePoints + 32;
    static constexpr size_t sm_bk = sm_pfx + (size_t)kPassBins * 4;
    static constexpr size_t small_bytes = sm_bk + (size_t)kPassBins * sizeof(BucketDesc);
    static constexpr size_t off_small = big_bytes;
    static constexpr size_t off_perm = off_small + 2 * small_bytes;
    static constexpr size_t off_cnt = off_perm + (size_t)kTilePoints * 4;
    static constexpr size_t off_bdst = off_cnt + (size_t)PassCfg<WIDE>::warps * kPassBins * 4;
    static constexpr size_t off_lutm = off_bdst + (size_t)kPassBins * sizeof(PassBucket);
    static constexpr size_t off_first = off_lutm + (size_t)kPassBins * 4;  // [nb] slot of the bucket's first record of this tile
    static constexpr size_t off_desc = off_first + (size_t)kPassBins * 4;  // [2]
    static constexpr size_t off_nact = off_desc + 2 * 64;                  // ActiveDesc of the next tile (cp.async landing zone)
    static constexpr size_t off_bar = off_nact + 64;                       // [3]: small[0], small[1], big
    static constexpr size_t off_bext = off_bar + 32;                       // [nb] fused exchange pass only: slot / intensity bases
    static constexpr size_t bytes = off_bext + (size_t)kPassBins * sizeof(PassBucketExt);
    static_assert(big_bytes % 16 == 0 && small_bytes % 16 == 0 && sm_pfx % 16 == 0, "bulk copy destinations must be 16-byte aligned");
};
static_assert(4 * (PassSmem<false>::bytes + 1024) <= 233472, "four narrow pass blocks must fit one SM (228 KB, 1 KB reserved per block)");
static_assert(2 * (PassSmem<true>::bytes + 1024) <= 233472, "two wide pass blocks must fit one SM");

struct PassTile {  // descriptor of a staged tile (shared memory, 64 bytes)
    double m[3];  // cube min of the active node
    double e;
    uint64_t start;
    uint32_t count, active;
    uint32_t tile, valid;
    uint32_t pad[2];
};
static_assert(sizeof(PassTile) == 64 && sizeof(ActiveDesc) == 64 && sizeof(PassBucket) == 32, "descriptor layout");

// finish one record (see above).  All level constants are plain kernel parameters (PassArgs::e1 ...).
// ENCU >= 0: every level the pass touches has this one encoding (the common case), so no switch per point
#define PCV_ENC_SEL(encu, enc_value, ...)        \
    if constexpr ((encu) >= 0) {                 \
        constexpr int ENC = (encu);              \
        __VA_ARGS__                              \
    } else {                                     \
        PCV_ENC_SWITCH(enc_value, __VA_ARGS__)   \
    }
template <bool WIDE, int FAST, int ENCU>
__device__ __forceinline__ void finish_record(const PassArgs& a, const double pm[3], uint64_t c[3], unsigned dig, int keep, bool next, unsigned& dig_out,
                                              unsigned& bad) {
    typedef typename std::conditional<WIDE, uint64_t, uint32_t>::type CodeT;
    const unsigned d1 = a.G == 2 ? (dig >> 3) : dig, d2 = dig & 7u;
    const double e1 = a.e1;
    double m[3], q[3];
    // child cube min (node.rs:165-170): x = bit 2, y = bit 1, z = bit 0
    m[0] = (d1 & 4u) ? pm[0] + e1 : pm[0];
    m[1] = (d1 & 2u) ? pm[1] + e1 : pm[1];
    m[2] = (d1 & 1u) ? pm[2] + e1 : pm[2];
    PCV_ENC_SEL(ENCU, a.enc1, _Pragma("unroll") for (int k = 0; k < 3; ++k) q[k] = decode_axis<ENC>(c[k], m[k], e1);)
    if (keep == 2) {
        const double e2 = a.e2, ry2 = a.ry2;
        m[0] = (d2 & 4u) ? m[0] + e2 : m[0];
        m[1] = (d2 & 2u) ? m[1] + e2 : m[1];
        m[2] = (d2 & 1u) ? m[2] + e2 : m[2];
        if (next) {
            PCV_ENC_SEL(ENCU, a.enc2, _Pragma("unroll") for (int k = 0; k < 3; ++k) {
                c[k] = encode_axis<ENC, FAST>(q[k], m[k], e2, ry2, bad);
                q[k] = decode_axis<ENC>(c[k], m[k], e2);
            })
        } else {
            PCV_ENC_SEL(ENCU, a.enc2, _Pragma("unroll") for (int k = 0; k < 3; ++k) c[k] = encode_axis<ENC, FAST>(q[k], m[k], e2, ry2, bad);)
            return;
        }
    }
    if (!next) return;  // leaf at level L+1: the carried codes are the node's codes
    // first step of the next pass from the node at level Lb = L + G (+ the second digit when that pass resolves two levels)
    const double eb = a.eb, eh = a.eh, ryh = a.ryh;
    CodeT code[3];
    unsigned d;
    if (a.Gn == 2) {
        PCV_ENC_SEL(ENCU, a.ench, d = level_step<ENC, FAST, true>(q, m, eb, eh, ryh, code, bad);)
        d = (d << 3) | level_digit(q, m, eh);
    } else {
        PCV_ENC_SEL(ENCU, a.ench, d = level_step<ENC, FAST, false>(q, m, eb, eh, ryh, code, bad);)
    }
    c[0] = (uint64_t)code[0], c[1] = (uint64_t)code[1], c[2] = (uint64_t)code[2];
    dig_out = d;
}

template <bool WIDE, int FAST, bool REMOTE, int ENCU>
__device__ __forceinline__ unsigned pass_finish(const PassArgs& a, const PassTile& pt, const unsigned char* srec, const uint32_t* scol, const uint8_t* sdig,
                                                const uint32_t* perm, const PassBucket* bdst, const PassBucketExt* bext) {
    constexpr size_t recsz = PassSmem<WIDE>::rec_bytes;
    unsigned bad = 0;
    const double pm[3] = {pt.m[0], pt.m[1], pt.m[2]};
    const uint32_t count = pt.count;
#pragma unroll 2
    for (uint32_t p = threadIdx.x; p < count; p += PassCfg<WIDE>::threads) {
        const uint32_t e = perm[p], i = e & 2047u, lb = e >> 12;
        const PassBucket bd = bdst[lb];
        const bool next = (bd.kk >> 8) == 0;
        const int keep = (int)(bd.kk & 0xFFu);
        uint64_t c[3];
        uint32_t idx, colour;
        smem_load_rec<WIDE>(srec, i, c, idx);
        if (!WIDE && a.rec_has_col) {  // exchanged record: {codes, colour}; the record's index is its position in the slab
            colour = idx;
            idx = (uint32_t)pt.start + i;
        } else {
            colour = scol[i];
        }
        unsigned dig_out = 0;
        if (next || keep == 2) finish_record<WIDE, FAST, ENCU>(a, pm, c, sdig[i], keep, next, dig_out, bad);
        if (FAST == 1 && bad) continue;  // the block repeats the sweep with the IEEE operator
        if (REMOTE) {
            // The destination is the owner's memory.  A record that continues is stored in the wire format of the exchange
            // (narrow: {codes, colour}, its index implied by its position = its slot); a leaf record carries its slot explicitly.
            const PassBucketExt bx = bext[lb];
            const uint32_t slot = bx.slot0 + p;
            if (!WIDE && next) {
                store_rec<WIDE>(reinterpret_cast<void*>(bd.rec + (unsigned long long)p * recsz), 0, c, colour);
            } else {
                store_rec<WIDE>(reinterpret_cast<void*>(bd.rec + (unsigned long long)p * recsz), 0, c, slot);
                *reinterpret_cast<uint32_t*>(bd.col + 4ull * p) = colour;
            }
            if (next) *reinterpret_cast<uint8_t*>(bd.dig + p) = (uint8_t)dig_out;
            if (a.int_in) *reinterpret_cast<float*>(bx.inten + 4ull * p) = a.int_in[idx];
            continue;
        }
        store_rec<WIDE>(reinterpret_cast<void*>(bd.rec + (unsigned long long)p * recsz), 0, c, idx);
        *reinterpret_cast<uint32_t*>(bd.col + 4ull * p) = colour;
        if (next) *reinterpret_cast<uint8_t*>(bd.dig + p) = (uint8_t)dig_out;
    }
    return bad;
}

// The two bulk-copy groups of a tile (one thread).  Sources must be 16-byte aligned: the colour / digit copies start up to
// 3 / 15 entries early.
template <bool WIDE>
__device__ __forceinline__ void pass_stage_small(const PassArgs& a, const PassTile& d, unsigned char* sm, uint64_t* bar) {
    const uint32_t doff = (uint32_t)(d.start & 15);
    const uint32_t dig_bytes = (doff + d.count + 15u) & ~15u;
    const uint32_t pfx_bytes = (uint32_t)a.nbins * 4u, bk_bytes = (uint32_t)a.nbins * (uint32_t)sizeof(BucketDesc);
    mbar_expect_tx(bar, dig_bytes + pfx_bytes + bk_bytes);
    tma_bulk_load(sm, a.dig_in + (d.start - doff), dig_bytes, bar);
    tma_bulk_load(sm + PassSmem<WIDE>::sm_pfx, a.tile_counts + (size_t)d.tile * a.nbins, pfx_bytes, bar);
    tma_bulk_load(sm + PassSmem<WIDE>::sm_bk, a.buckets + (size_t)d.active * a.nbins, bk_bytes, bar);
}
template <bool WIDE>
__device__ __forceinline__ void pass_stage_big(const PassArgs& a, const PassTile& d, unsigned char* smem_raw, uint64_t* bar) {
    constexpr size_t recsz = PassSmem<WIDE>::rec_bytes;
    const uint32_t coff = (uint32_t)(d.start & 3);
    const uint32_t rec_bytes = d.count * (uint32_t)recsz;
    const bool with_col = WIDE || !a.rec_has_col;
    const uint32_t col_bytes = with_col ? (((coff + d.count) * 4u + 15u) & ~15u) : 0u;
    mbar_expect_tx(bar, rec_bytes + col_bytes);
    tma_bulk_load(smem_raw, reinterpret_cast<const unsigned char*>(a.rec_in) + d.start * recsz, rec_bytes, bar);
    if (with_col) tma_bulk_load(smem_raw + PassSmem<WIDE>::off_col, a.col_in + (d.start - coff), col_bytes, bar);
}
__device__ __forceinline__ void pass_make_desc(PassTile* desc, uint32_t tile, const ActiveDesc& act, uint32_t active) {
    const uint64_t o = (uint64_t)(tile - act.tile_begin) * kTilePoints;
    const uint64_t rem = act.count - o;
    desc->m[0] = act.m[0], desc->m[1] = act.m[1], desc->m[2] = act.m[2];
    desc->e = act.e;
    desc->start = act.start + o;
    desc->count = (uint32_t)(rem < kTilePoints ? rem : kTilePoints);
    desc->active = active;
    desc->tile = tile;
    desc->valid = 1;
}

// FASTMODE = PassArgs::fast, ENCU = the pass's one encoding or -1 (mixed): a kernel per combination keeps the switches out of the
// per-point code and the register budget on the work
template <bool WIDE, bool REMOTE, int FASTMODE, int ENCU>
__global__ void __launch_bounds__(PassCfg<WIDE>::threads, PassCfg<WIDE>::blocks_per_sm) k_pass(const __grid_constant__ PassArgs a) {
    constexpr int nbmax = kPassBins;
    constexpr int kThreads = PassCfg<WIDE>::threads, kWarps = PassCfg<WIDE>::warps, kWarpItems = PassCfg<WIDE>::warp_items, kSubRounds = PassCfg<WIDE>::sub_rounds;
    constexpr size_t recsz = PassSmem<WIDE>::rec_bytes;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const unsigned char* srec = smem_raw;
    uint32_t* perm = reinterpret_cast<uint32_t*>(smem_raw + PassSmem<WIDE>::off_perm);       // [tile] item | bucket << 12, sorted
    uint32_t* cnt = reinterpret_cast<uint32_t*>(smem_raw + PassSmem<WIDE>::off_cnt);         // [warps][nb]
    PassBucket* bdst = reinterpret_cast<PassBucket*>(smem_raw + PassSmem<WIDE>::off_bdst);   // [nb]
    uint32_t* lutm = reinterpret_cast<uint32_t*>(smem_raw + PassSmem<WIDE>::off_lutm);       // [nb] digit -> bucket
    uint32_t* bfirst = reinterpret_cast<uint32_t*>(smem_raw + PassSmem<WIDE>::off_first);    // [nb]
    PassTile* descs = reinterpret_cast<PassTile*>(smem_raw + PassSmem<WIDE>::off_desc);      // [2]
    ActiveDesc* snact = reinterpret_cast<ActiveDesc*>(smem_raw + PassSmem<WIDE>::off_nact);
    uint64_t* mbar = reinterpret_cast<uint64_t*>(smem_raw + PassSmem<WIDE>::off_bar);        // small[0], small[1], big
    PassBucketExt* bext = reinterpret_cast<PassBucketExt*>(smem_raw + PassSmem<WIDE>::off_bext);

    const PassState ps = a.st->pass[a.pass];
    const int nb = a.nbins;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (blockIdx.x >= ps.ntiles) return;
    if (tid == 0) {
        mbar_init(&mbar[0], 1);
        mbar_init(&mbar[1], 1);
        mbar_init(&mbar[2], 1);
        const uint32_t act0 = a.tile_active[blockIdx.x];
        pass_make_desc(&descs[0], blockIdx.x, a.active[act0], act0);
        pass_stage_small<WIDE>(a, descs[0], smem_raw + PassSmem<WIDE>::off_small, &mbar[0]);
        pass_stage_big<WIDE>(a, descs[0], smem_raw, &mbar[2]);
    }
    __syncthreads();
    uint32_t it = 0;
    for (uint32_t tile = blockIdx.x; tile < ps.ntiles; tile += gridDim.x, ++it) {
        const uint32_t s = it & 1u;
        const PassTile& pt = descs[s];  // stays in shared memory (broadcast reads)
        const unsigned char* sm = smem_raw + PassSmem<WIDE>::off_small + (size_t)s * PassSmem<WIDE>::small_bytes;
        const uint32_t* scol = reinterpret_cast<const uint32_t*>(smem_raw + PassSmem<WIDE>::off_col) + (uint32_t)(pt.start & 3);
        const uint8_t* sdig = sm + (uint32_t)(pt.start & 15);
        const uint32_t* spfx = reinterpret_cast<const uint32_t*>(sm + PassSmem<WIDE>::sm_pfx);
        const BucketDesc* sbk = reinterpret_cast<const BucketDesc*>(sm + PassSmem<WIDE>::sm_bk);
        // the next tile of this block: its node is looked up by one thread, the loads are consumed phases later
        const uint32_t ntile = tile + gridDim.x;
        const bool stage_next = tid == 0 && ntile < ps.ntiles;
        uint32_t nact = 0;
        if (stage_next) nact = a.tile_active[ntile];
        for (int i = tid; i < kWarps * nbmax; i += kThreads) cnt[i] = 0;

        mbar_wait(&mbar[s], (it >> 1) & 1u);  // digits, prefix row and bucket table of this tile (requested a tile ago)
        // (1) tables, one thread per bucket: the slot of this tile's first record = bucket start + the records of the bucket's
        // digits in the node's earlier tiles; every digit of the bucket's range learns its bucket.  (A digit without a bucket has
        // no points in the node, so its map entry is never read.)
        if (tid < nb) {
            const BucketDesc bd = sbk[tid];
            uint32_t v = 0;
            if (bd.b1 != 0) {
                v = (uint32_t)bd.dest;
                for (uint32_t d = bd.b0; d < bd.b1; ++d) {
                    v += spfx[d];
                    lutm[d] = (uint32_t)tid;
                }
            }
            bfirst[tid] = v;
        }
        __syncthreads();

        // (2) rank: bucket of every item from its carried digit; lanes of a sub-round grouped by bucket
        uint32_t info[kSubRounds];
        {
            const uint32_t count = pt.count;
            uint32_t lbv[kSubRounds];
            unsigned mask[kSubRounds];
#pragma unroll
            for (int r = 0; r < kSubRounds; ++r) {
                const uint32_t i = warp * kWarpItems + r * 32 + lane;
                lbv[r] = 0xFFFFu;
                if (i < count) lbv[r] = lutm[sdig[i] & (uint32_t)(nb - 1)];
            }
#pragma unroll
            for (int r = 0; r < kSubRounds; ++r) mask[r] = __match_any_sync(0xffffffffu, lbv[r]);  // independent: their latencies overlap
#pragma unroll
            for (int r = 0; r < kSubRounds; ++r) {
                const uint32_t leader = (uint32_t)__ffs(mask[r]) - 1u, gsize = (uint32_t)__popc(mask[r]), rank = (uint32_t)__popc(mask[r] & ((1u << lane) - 1u));
                info[r] = lbv[r] | (rank << 16) | (leader << 21) | ((gsize - 1u) << 26);
                if (lbv[r] != 0xFFFFu && lane == (int)leader) cnt[warp * nbmax + lbv[r]] += gsize;  // one leader per bucket inside the warp: no conflict
                __syncwarp();
            }
        }
        if (stage_next) {  // the next tile's node descriptor: asynchronous 16-byte copies, consumed after the sort phase
            const unsigned char* src = reinterpret_cast<const unsigned char*>(a.active + nact);
#pragma unroll
            for (int k = 0; k < 4; ++k)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(reinterpret_cast<unsigned char*>(snact) + 16 * k)), "l"(src + 16 * k) : "memory");
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        __syncthreads();
        // (3) per-bucket totals -> exclusive scan over the buckets (sorted start of every bucket) -> per-warp offsets and the
        // bucket's store bases (warp 0)
        if (warp == 0) {
            uint32_t tot[2] = {0, 0};
            for (int j = 0; j < 2; ++j) {
                const int lb = lane + 32 * j;
                if (lb < nb) {
#pragma unroll
                    for (int w = 0; w < kWarps; ++w) tot[j] += cnt[w * nbmax + lb];
                }
            }
            // buckets are numbered lane + 32 j: scan j = 0 over the lanes, then j = 1 on top of its total
            uint32_t excl[2];
            uint32_t carry = 0;
            for (int j = 0; j < 2; ++j) {
                uint32_t incl = tot[j];
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += u;
                }
                excl[j] = carry + incl - tot[j];
                carry += __shfl_sync(0xffffffffu, incl, 31);
            }
            for (int j = 0; j < 2; ++j) {
                const int lb = lane + 32 * j;
                if (lb < nb) {
                    uint32_t run = excl[j];
                    const BucketDesc bd = sbk[lb];
                    const bool leaf = bd.b1 != 0 && bd.kind;
                    const long long first = (long long)bfirst[lb] - (long long)run;  // slot of sorted position 0
                    PassBucket pb;
                    if (REMOTE) {
                        // the bucket lives in its owner's buffers; a leaf bucket's descriptor carries its slot base in the high word
                        RemoteBufs rb{};
                        if (bd.b1 != 0) rb = a.remote[bd.owner - 1u];
                        pb.rec = (unsigned long long)(leaf ? rb.arena : rb.rec_next) + (unsigned long long)(first * (long long)recsz);
                        pb.col = (unsigned long long)(leaf ? rb.col_arena : rb.col_next) + (unsigned long long)(first * 4);
                        pb.dig = (unsigned long long)rb.dig_next + (unsigned long long)first;
                        const long long slot0 = leaf ? first + (long long)(bd.dest >> 32) - (long long)(uint32_t)bd.dest : first;
                        PassBucketExt bx;
                        bx.inten = (unsigned long long)rb.intensity + (unsigned long long)(slot0 * 4);
                        bx.slot0 = (uint32_t)slot0;
                        bx.pad = 0;
                        bext[lb] = bx;
                    } else {
                    pb.rec = (unsigned long long)(leaf ? a.arena : a.rec_next) + (unsigned long long)(first * (long long)recsz);
                    pb.col = (unsigned long long)(leaf ? a.col_arena : a.col_next) + (unsigned long long)(first * 4);
                    pb.dig = (unsigned long long)a.dig_next + (unsigned long long)first;
                    }
                    pb.start = run;
                    pb.kk = (uint32_t)bd.keep | (leaf ? 0x100u : 0u);
                    bdst[lb] = pb;
#pragma unroll
                    for (int w = 0; w < kWarps; ++w) {
                        const uint32_t c = cnt[w * nbmax + lb];
                        cnt[w * nbmax + lb] = run;
                        run += c;
                    }
                }
            }
        }
        __syncthreads();
        // (4) sort: stable sorted position of every item (warp by warp, sub-round by sub-round, rank inside the group)
#pragma unroll
        for (int r = 0; r < kSubRounds; ++r) {
            const uint32_t i = warp * kWarpItems + r * 32 + lane;
            const uint32_t lbv = info[r] & 0xFFFFu, rank = (info[r] >> 16) & 31u, gsize = ((info[r] >> 26) & 31u) + 1u;
            const int leader = (int)((info[r] >> 21) & 31u);
            uint32_t old = 0;
            if (lane == leader && lbv != 0xFFFFu) {
                old = cnt[warp * nbmax + lbv];
                cnt[warp * nbmax + lbv] = old + gsize;
            }
            old = __shfl_sync(0xffffffffu, old, leader);
            if (lbv != 0xFFFFu) perm[old + rank] = i | (lbv << 12);
            __syncwarp();
        }
        // the other small buffer was last read by the previous tile: request the next tile's digits and tables now, a whole
        // tile ahead of their use
        if (stage_next) {
            asm volatile("cp.async.wait_all;" ::: "memory");
            pass_make_desc(&descs[s ^ 1u], ntile, *snact, nact);
            pass_stage_small<WIDE>(a, descs[s ^ 1u], smem_raw + PassSmem<WIDE>::off_small + (size_t)(s ^ 1u) * PassSmem<WIDE>::small_bytes, &mbar[s ^ 1u]);
        }
        __syncthreads();
        // (5) finish + store in destination order (speculatively through the reciprocal division; repeated with the IEEE
        // operator if any numerator of the block was outside the proven range - the stores are idempotent)
        mbar_wait(&mbar[2], it & 1u);  // records and colours: requested when the previous tile's sweep ended
        if (FASTMODE == 1) {
            const unsigned bad = pass_finish<WIDE, 1, REMOTE, ENCU>(a, pt, srec, scol, sdig, perm, bdst, bext);
            if (__syncthreads_or((int)bad)) pass_finish<WIDE, 0, REMOTE, ENCU>(a, pt, srec, scol, sdig, perm, bdst, bext);
        } else {
            // 3: power-of-two edges, exact scaling; 2: no per-numerator checks; 0: IEEE division - nothing to repeat in any of them
            pass_finish<WIDE, FASTMODE, REMOTE, ENCU>(a, pt, srec, scol, sdig, perm, bdst, bext);
        }
        __syncthreads();  // records, colours, perm and the tables are reused
        if (stage_next) pass_stage_big<WIDE>(a, descs[s ^ 1u], smem_raw, &mbar[2]);
    }
}

// ------------------------------------------------------------------------------------------------
// place
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_code(uint8_t* p, uint64_t c, int enc) {
    if (enc == ENC_U8)
        *p = (uint8_t)c;
    else if (enc == ENC_U16)
        *reinterpret_cast<uint16_t*>(p) = (uint16_t)c;
    else if (enc == ENC_F32)
        *reinterpret_cast<uint32_t*>(p) = (uint32_t)c;
    else
        *reinterpret_cast<uint64_t*>(p) = c;
}

__device__ __forceinline__ void place_store(const PlaceArgs& a, const DNode& nd, uint64_t slot, const uint64_t c[3], uint32_t col, uint32_t idx) {
    const uint64_t dp = nd.out_point_off + slot;
    const int bpc = enc_bytes(nd.enc);
    uint8_t* px = a.out_xyz + nd.out_xyz_off + slot * 3 * (uint64_t)bpc;
    store_code(px, c[0], nd.enc);
    store_code(px + bpc, c[1], nd.enc);
    store_code(px + 2 * bpc, c[2], nd.enc);
    uint8_t* rd = a.out_rgb + 3ull * dp;
    rd[0] = (uint8_t)col;
    rd[1] = (uint8_t)(col >> 8);
    rd[2] = (uint8_t)(col >> 16);
    a.out_src[dp] = idx;
    if (a.out_intensity) a.out_intensity[dp] = __ldg(a.pts.intensity + idx);
}

// A place tile staged in shared memory: its records, then its colours copied from the 16-byte granule that holds the first
// one (scol[coff + i] is colour i, coff = arena_start & 3), the mbarrier of the copies and the tile's node (broadcast reads
// instead of a node's worth of registers held through the whole tile).
template <bool WIDE>
struct PlaceSmem {
    static constexpr size_t rec_bytes = WIDE ? 32 : 16;
    static constexpr size_t off_col = (size_t)kPlaceTile * rec_bytes;
    static constexpr size_t off_bar = off_col + ((size_t)kPlaceTile + 4) * 4;
    static constexpr size_t off_node = off_bar + 16;
    static constexpr size_t bytes = off_node + sizeof(DNode);
    static_assert(off_col % 16 == 0 && off_bar % 16 == 0 && sizeof(DNode) % 4 == 0, "bulk copy destinations 16-byte aligned, the node copied in whole words");
};
static_assert(4 * (PlaceSmem<false>::bytes + 1024) <= 233472, "four narrow place blocks must fit one SM (228 KB, 1 KB reserved per block)");

// tile -> descriptor (one block per leaf, threads over its tiles): a k_place block finds its tile with one load instead of a
// binary search of dependent loads over the leaves' first tiles
__global__ void k_place_tiles(const __grid_constant__ PlaceArgs a, LeafTile* __restrict__ tiles) {
    const uint32_t l = blockIdx.x;
    const uint32_t t0 = a.d_leaf_tile_begin[l], nt = a.d_leaf_tile_begin[l + 1] - t0;
    const uint32_t node = a.d_leaf_node[l];
    const uint64_t arena_off = a.d_nodes[node].arena_off, count = a.d_nodes[node].count;
    for (uint32_t t = threadIdx.x; t < nt; t += blockDim.x) {
        const uint64_t o = (uint64_t)t * kPlaceTile, rem = count - o;
        tiles[t0 + t] = LeafTile{arena_off + o, o, node, (uint32_t)(rem < kPlaceTile ? rem : kPlaceTile)};
    }
}

// The 7 of 8 points of a non-root node that stay: one same-cube rewrite (child_writer, generation.rs:234-238) with the
// node's encoding hoisted out of the loop; dense lane mapping (stayer s <-> rank j = 8*(s/7) + s%7 + 1).
template <bool WIDE, int ENC, int FAST>
__device__ __forceinline__ unsigned place_stayers(const PlaceArgs& a, const LeafTile& lt, const DNode& nd, const unsigned char* srec, const uint32_t* scol) {
    unsigned bad = 0;
    const uint32_t nst = lt.count - (lt.count + 7) / 8;  // tile starts at a multiple of 8
    for (uint32_t s = threadIdx.x; s < nst; s += blockDim.x) {
        const uint32_t i = 8 * (s / 7) + (s % 7) + 1;
        uint64_t c[3];
        uint32_t idx;
        smem_load_rec<WIDE>(srec, i, c, idx);
        const uint32_t col = scol[i];
#pragma unroll
        for (int k = 0; k < 3; ++k) c[k] = encode_axis<ENC, FAST>(decode_axis<ENC>(c[k], nd.m[k], nd.e), nd.m[k], nd.e, nd.ry, bad);
        if (!FAST || !bad) {
            const uint64_t j = lt.j0 + i;
            place_store(a, nd, j - (j >> 3) - 1, c, col, idx);
        }
    }
    return bad;
}

// Points that move (every 8th by current rank, generation.rs:224-238): walk up re-encoding through every cube.
template <bool WIDE>
__device__ __forceinline__ void place_movers(const PlaceArgs& a, const LeafTile& lt, const DNode& leaf, bool all_points, const unsigned char* srec,
                                             const uint32_t* scol) {
    const uint32_t step = all_points ? 1u : 8u;
    for (uint32_t i = threadIdx.x * step; i < lt.count; i += blockDim.x * step) {
        uint64_t c[3];
        uint32_t idx;
        smem_load_rec<WIDE>(srec, i, c, idx);
        const uint32_t col = scol[i];
        uint64_t j = lt.j0 + i;
        const DNode* nd = &leaf;  // node fields are read where they are used: no node held in registers through the walk
        while (nd->parent >= 0 && (j & 7) == 0) {
            const DNode* P = a.d_nodes + nd->parent;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (a.fast) {
                    const double q = decode1_fast(c[k], nd->m[k], nd->e, nd->enc);
                    c[k] = encode1_fast(q, P->m[k], P->e, P->ry, P->enc);
                } else {
                    const double q = decode1(c[k], nd->m[k], nd->e, nd->enc);
                    c[k] = encode1(q, P->m[k], P->e, P->enc);
                }
            }
            j = nd->off_in_parent + (j >> 3);
            nd = P;
        }
        uint64_t slot = j;
        if (nd->parent >= 0) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (a.fast) {
                    const double q = decode1_fast(c[k], nd->m[k], nd->e, nd->enc);
                    c[k] = encode1_fast(q, nd->m[k], nd->e, nd->ry, nd->enc);
                } else {
                    const double q = decode1(c[k], nd->m[k], nd->e, nd->enc);
                    c[k] = encode1(q, nd->m[k], nd->e, nd->enc);
                }
            }
            slot = j - (j >> 3) - 1;
        }
        place_store(a, *nd, slot, c, col, idx);
    }
}

// One block per place tile.  Thread 0 requests the whole tile - records and colours - with bulk copies into shared memory as
// soon as the tile's descriptor is known; the node's descriptor is loaded while they are in flight, and no thread touches a
// point before the copies have landed.  The records and colours stay staged for the FAST == 1 redo.
template <bool WIDE>
__global__ void __launch_bounds__(256) k_place(const __grid_constant__ PlaceArgs a) {
    constexpr size_t recsz = PlaceSmem<WIDE>::rec_bytes;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + PlaceSmem<WIDE>::off_bar);
    const LeafTile lt = a.tiles[blockIdx.x];
    const uint32_t coff = (uint32_t)(lt.arena_start & 3);
    if (threadIdx.x == 0) {
        // records are 16 / 32 bytes, so the record range is 16-byte aligned; the colours are copied from the granule that
        // holds the first one, rounded up to whole granules (every colour arena has slack past its end for that)
        const uint32_t rec_bytes = lt.count * (uint32_t)recsz, col_bytes = ((coff + lt.count) * 4u + 15u) & ~15u;
        mbar_init(bar, 1);
        mbar_expect_tx(bar, rec_bytes + col_bytes);
        tma_bulk_load(smem_raw, reinterpret_cast<const unsigned char*>(a.arena) + lt.arena_start * recsz, rec_bytes, bar);
        tma_bulk_load(smem_raw + PlaceSmem<WIDE>::off_col, a.col_arena + (lt.arena_start - coff), col_bytes, bar);
    }
    DNode* snode = reinterpret_cast<DNode*>(smem_raw + PlaceSmem<WIDE>::off_node);
    if (threadIdx.x < sizeof(DNode) / 4) reinterpret_cast<uint32_t*>(snode)[threadIdx.x] = reinterpret_cast<const uint32_t*>(a.d_nodes + lt.node)[threadIdx.x];
    const DNode& leaf = *snode;
    const unsigned char* srec = smem_raw;
    const uint32_t* scol = reinterpret_cast<const uint32_t*>(smem_raw + PlaceSmem<WIDE>::off_col) + coff;
    __syncthreads();  // the barrier is initialised, the node is in shared memory
    mbar_wait(bar, 0);
    // A tile whose start rank is not a multiple of 8 (top assembly: a collector's points start at arbitrary ranks), or
    // whose node ends the walk (root / collector), goes through the generic per-point path.
    const bool generic = leaf.parent < 0 || (lt.j0 & 7) != 0;
    if (generic) {
        place_movers<WIDE>(a, lt, leaf, true, srec, scol);
        return;
    }
    if (a.fast == 3) {
        PCV_ENC_SWITCH(leaf.enc, place_stayers<WIDE, ENC, 3>(a, lt, leaf, srec, scol);)
    } else if (a.fast) {
        unsigned bad = 0;
        if (a.fast == 2) {
            PCV_ENC_SWITCH(leaf.enc, bad = place_stayers<WIDE, ENC, 2>(a, lt, leaf, srec, scol);)
        } else {
            PCV_ENC_SWITCH(leaf.enc, bad = place_stayers<WIDE, ENC, 1>(a, lt, leaf, srec, scol);)
        }
        if (__syncthreads_or((int)bad)) {  // rare: redo the tile's stayers with the IEEE operator (idempotent stores)
            PCV_ENC_SWITCH(leaf.enc, place_stayers<WIDE, ENC, 0>(a, lt, leaf, srec, scol);)
        }
    } else {
        PCV_ENC_SWITCH(leaf.enc, place_stayers<WIDE, ENC, 0>(a, lt, leaf, srec, scol);)
    }
    place_movers<WIDE>(a, lt, leaf, false, srec, scol);
}

// ------------------------------------------------------------------------------------------------
// CUDA backend
// ------------------------------------------------------------------------------------------------
struct CudaBackend : Backend {
    cudaStream_t stream = nullptr;
    uint64_t launches = 0;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    // optional per-kernel timing (CUDA events on the launching stream around every launch)
    enum { K_BBOX = 0, K_INGEST, K_DIGHIST, K_SCAN, K_PLAN, K_PASS, K_PLACE, K_PLY, K_COUNT };
    struct KStat {
        uint64_t launches = 0, bytes = 0;
        double ms = 0;
    };
    bool profile = false;
    KStat kstat[K_COUNT];
    struct Pending {
        int k;
        cudaEvent_t e0, e1;
        uint64_t bytes;
        int pass;  // split-phase kernels: their byte counts are filled in once the pass's live point count is known
    };
    std::vector<Pending> pending;
    void prof_begin(int k, uint64_t bytes, int pass = -1) {
        if (!profile) return;
        Pending p{k, nullptr, nullptr, bytes, pass};
        cudaEventCreate(&p.e0);
        cudaEventCreate(&p.e1);
        cudaEventRecord(p.e0, stream);
        pending.push_back(p);
    }
    void prof_end() {
        if (!profile) return;
        cudaEventRecord(pending.back().e1, stream);
    }
    void prof_collect() {  // call after a stream synchronize
        for (auto& p : pending) {
            float ms = 0;
            cudaEventElapsedTime(&ms, p.e0, p.e1);
            kstat[p.k].launches++;
            kstat[p.k].ms += ms;
            kstat[p.k].bytes += p.bytes;
            cudaEventDestroy(p.e0);
            cudaEventDestroy(p.e1);
        }
        pending.clear();
    }
    void prof_reset() {
        for (auto& k : kstat) k = KStat();
    }

    explicit CudaBackend(cudaStream_t s) : stream(s) {
        for (auto& e : ev) PCV_CUDA_CHECK(cudaEventCreate(&e));
        allow_smem_all();
    }
    ~CudaBackend() override {
        cache_release();
        if (ev_back) cudaEventDestroy(ev_back);
        for (auto& b : back_chunks) cudaFreeHost(b.p);
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        if (pin) cudaFreeHost(pin);
        if (pin_back) cudaFreeHost(pin_back);
    }
    // Large blocks are recycled by exact size inside the context before they go back to the stream-ordered pool: repeated builds
    // of the same shape (a viewer re-building, the steps of the sharded build) make no allocator calls at all in steady state.
    // Measured on the second rank of a 2-GPU sharded build, whose receive-side buffers (1.0004e9 points) are slightly larger than
    // its send-side ones (1e9): the pool cannot reuse a freed block for a larger request, and a cudaMallocAsync that has to find
    // 4 GB of new memory took 5 - 60 ms, every step.  Everything a context allocates is used on its one stream, so handing a
    // block to the next user is stream-ordered exactly like cudaFreeAsync + cudaMallocAsync.  The cache is bounded (half of the
    // device memory, oldest blocks leave first) and emptied when an allocation fails.
    static constexpr size_t kCacheMin = (size_t)1 << 20;
    struct CachedBlock {
        void* p;
        uint64_t seq;
    };
    std::unordered_map<void*, size_t> big_live;
    std::multimap<size_t, CachedBlock> big_free;
    size_t cached_bytes = 0, cache_cap = 0;
    uint64_t cache_seq = 0;
    void cache_release() {
        for (auto& kv : big_free) cudaFreeAsync(kv.second.p, stream);
        big_free.clear();
        cached_bytes = 0;
    }
    void cache_evict_oldest() {
        auto best = big_free.begin();
        for (auto it = big_free.begin(); it != big_free.end(); ++it)
            if (it->second.seq < best->second.seq) best = it;
        cudaFreeAsync(best->second.p, stream);
        cached_bytes -= best->first;
        big_free.erase(best);
    }
    bool trace_alloc = std::getenv("PCV_TRACE_ALLOC") != nullptr;
    void* dmalloc(size_t bytes) override {
        if (!trace_alloc) return dmalloc_impl(bytes);
        const auto t0 = std::chrono::steady_clock::now();
        const size_t nfree = big_free.size();
        void* p = dmalloc_impl(bytes);
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (ms > 0.2) {
            int dev = -1;
            cudaGetDevice(&dev);
            fprintf(stderr, "[pcv dmalloc dev%d] %zu bytes: %.2f ms (cached blocks before %zu, after %zu)\n", dev, bytes, ms, nfree, big_free.size());
        }
        return p;
    }
    void* dmalloc_impl(size_t bytes) {
        void* p = nullptr;
        if (bytes >= kCacheMin) {
            auto it = big_free.find(bytes);
            if (it != big_free.end()) {
                p = it->second.p;
                big_free.erase(it);
                cached_bytes -= bytes;
                big_live[p] = bytes;
                return p;
            }
        }
        cudaError_t e = cudaMallocAsync(&p, bytes ? bytes : 16, stream);
        if (e == cudaErrorMemoryAllocation && !big_free.empty()) {  // make room: everything cached goes back to the pool
            cudaGetLastError();
            cache_release();
            e = cudaMallocAsync(&p, bytes ? bytes : 16, stream);
        }
        PCV_CUDA_CHECK(e);
        if (bytes >= kCacheMin) big_live[p] = bytes;
        return p;
    }
    void dfree(void* p) override {
        if (!p) return;
        auto it = big_live.find(p);
        if (it == big_live.end()) {
            cudaFreeAsync(p, stream);
            return;
        }
        if (!cache_cap) {
            size_t fr = 0, tot = 0;
            cudaMemGetInfo(&fr, &tot);
            cache_cap = tot / 2;
        }
        const size_t bytes = it->second;
        big_live.erase(it);
        big_free.emplace(bytes, CachedBlock{p, ++cache_seq});
        cached_bytes += bytes;
        while (cached_bytes > cache_cap && !big_free.empty()) cache_evict_oldest();
    }
    // Host -> device staging through a pinned ring so that descriptor uploads are truly asynchronous (a pageable
    // source would make cudaMemcpyAsync wait for all prior work of the stream).  The ring is recycled after a
    // stream synchronize (d2h below, once per pass) or when it wraps.
    uint8_t* pin = nullptr;
    size_t pin_cap = 0, pin_off = 0;
    void h2d(void* d, const void* h, size_t bytes) override {
        if (bytes == 0) return;
        const size_t need = (bytes + 255) & ~(size_t)255;
        if (need > pin_cap / 2) {  // too big for the ring: grow it (rare) after draining the stream
            PCV_CUDA_CHECK(cudaStreamSynchronize(stream));
            if (pin) cudaFreeHost(pin);
            pin_cap = std::max<size_t>(need * 4, (size_t)64 << 20);
            PCV_CUDA_CHECK(cudaMallocHost(&pin, pin_cap));
            pin_off = 0;
        }
        if (pin_off + need > pin_cap) {
            PCV_CUDA_CHECK(cudaStreamSynchronize(stream));
            pin_off = 0;
        }
        std::memcpy(pin + pin_off, h, bytes);
        PCV_CUDA_CHECK(cudaMemcpyAsync(d, pin + pin_off, bytes, cudaMemcpyHostToDevice, stream));
        pin_off += need;
    }
    uint8_t* pin_back = nullptr;
    size_t pin_back_cap = 0;
    void d2h(void* h, const void* d, size_t bytes) override {
        if (bytes > pin_back_cap) {
            if (pin_back) cudaFreeHost(pin_back);
            pin_back_cap = std::max<size_t>(bytes * 2, (size_t)8 << 20);
            PCV_CUDA_CHECK(cudaMallocHost(&pin_back, pin_back_cap));
        }
        PCV_CUDA_CHECK(cudaMemcpyAsync(pin_back, d, bytes, cudaMemcpyDeviceToHost, stream));
        PCV_CUDA_CHECK(cudaStreamSynchronize(stream));
        std::memcpy(h, pin_back, bytes);
        pin_off = 0;  // everything staged before this point has been consumed
    }
    void mark(int what) override { cudaEventRecord(ev[what], stream); }

    void zero(void* d, size_t bytes) override {
        if (bytes) PCV_CUDA_CHECK(cudaMemsetAsync(d, 0, bytes, stream));
    }
    static void allow_smem_all() {
        for (int w = 0; w < 2; ++w)
            for (int r = 0; r < 2; ++r)
                for (int f = 0; f < 4; ++f)
                    for (int e = -1; e <= ENC_F32; ++e) {
                        const void* fn = pass_kernel(w != 0, r != 0, f, e);
                        if (fn) cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(w ? PassSmem<true>::bytes : PassSmem<false>::bytes));
                    }
        cudaFuncSetAttribute(k_place<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PlaceSmem<false>::bytes);
        cudaFuncSetAttribute(k_place<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PlaceSmem<true>::bytes);
    }
    int sms = 0;
    int sm_count() {
        if (!sms) {
            int dev = 0;
            cudaGetDevice(&dev);
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        }
        return sms;
    }

    void ingest(const IngestArgs& a) override {
        const uint32_t grid = std::min<uint32_t>(a.ntiles, (uint32_t)sm_count() * 32u);
        const uint64_t rec = a.wide ? sizeof(RecW) : sizeof(RecN);
        prof_begin(K_INGEST, a.pts.n * (27 + rec + 4 + 1));
        static const int batch = std::getenv("PCV_INGEST_BATCH") ? std::atoi(std::getenv("PCV_INGEST_BATCH")) : 2;  // 1: experiments
#define PCV_INGEST(W, F)                                                 \
    if (batch == 1)                                                      \
        k_ingest<W, F, 1><<<grid, kIngestThreads, 0, stream>>>(a);      \
    else                                                                 \
        k_ingest<W, F, 2><<<grid, kIngestThreads, 0, stream>>>(a)
        switch ((a.wide ? 4 : 0) + a.lv.fast) {
            case 0: PCV_INGEST(false, 0); break;
            case 1: PCV_INGEST(false, 1); break;
            case 2: PCV_INGEST(false, 2); break;
            case 3: PCV_INGEST(false, 3); break;
            case 4: PCV_INGEST(true, 0); break;
            case 5: PCV_INGEST(true, 1); break;
            case 6: PCV_INGEST(true, 2); break;
            default: PCV_INGEST(true, 3); break;
        }
#undef PCV_INGEST
        prof_end();
        ++launches;
        PCV_CUDA_CHECK(cudaGetLastError());
    }
    // One pass, enqueued without any host synchronisation: live sizes come from the device-resident BuildState, grids are
    // fixed (persistent / grid-stride) and blocks beyond the live counts exit.
    void pass(const PassArgs& a) override {
        hist_scan_launch(a);
        plan_launch(a);
        partition_launch(a);
        launches += 9;
        pass_wide = a.wide;
        PCV_CUDA_CHECK(cudaGetLastError());
    }
    void plan_launch(const PassArgs& a) {
        const int nsm = sm_count();
        prof_begin(K_PLAN, 0, a.pass);
        const uint32_t pg = std::min<uint32_t>((a.cap_active + kPlanNodeThreads - 1) / kPlanNodeThreads, (uint32_t)nsm * 8u);
        k_plan_count<<<pg, kPlanNodeThreads, 0, stream>>>(a);
        k_plan_scan<<<1, kPlanThreads, 0, stream>>>(a);
        k_plan_emit<<<pg, kPlanNodeThreads, 0, stream>>>(a);
        prof_end();
    }
    void finish_plan(const FinishArgs& f_in, int last_level) override {
        FinishArgs f = f_in;
        prof_begin(K_PLAN, 0);
        for (int L = last_level; L >= 0; --L) {
            f.level = L;
            k_sub_level<<<sm_count() * 2, 256, 0, stream>>>(f);
        }
        k_sub_layout<<<1, kPlanThreads, 0, stream>>>(f);
        prof_end();
        launches += (uint64_t)last_level + 2;
        PCV_CUDA_CHECK(cudaGetLastError());
    }
    // asynchronous read-backs into pinned chunks that never move (the caller keeps the returned pointers until d2h_wait)
    struct BackChunk {
        uint8_t* p;
        size_t cap, off;
    };
    std::vector<BackChunk> back_chunks;
    cudaEvent_t ev_back = nullptr;
    const void* d2h_begin(const void* d, size_t bytes) override {
        const size_t need = ((bytes ? bytes : 1) + 255) & ~(size_t)255;
        BackChunk* c = nullptr;
        for (auto& b : back_chunks)
            if (b.off + need <= b.cap) {
                c = &b;
                break;
            }
        if (!c) {
            BackChunk nb{nullptr, std::max<size_t>(need, (size_t)32 << 20), 0};
            PCV_CUDA_CHECK(cudaMallocHost(&nb.p, nb.cap));
            back_chunks.push_back(nb);
            c = &back_chunks.back();
        }
        uint8_t* dst = c->p + c->off;
        c->off += need;
        if (bytes) PCV_CUDA_CHECK(cudaMemcpyAsync(dst, d, bytes, cudaMemcpyDeviceToHost, stream));
        if (!ev_back) PCV_CUDA_CHECK(cudaEventCreateWithFlags(&ev_back, cudaEventDisableTiming));
        PCV_CUDA_CHECK(cudaEventRecord(ev_back, stream));
        return dst;
    }
    void d2h_wait() override {
        if (ev_back) PCV_CUDA_CHECK(cudaEventSynchronize(ev_back));
        for (auto& b : back_chunks) b.off = 0;
    }
    void plan(const PassArgs& a) override {
        plan_launch(a);
        launches += 3;
        PCV_CUDA_CHECK(cudaGetLastError());
    }
    // The instantiated partition kernels: wide records and the fused exchange pass only in the mixed-encoding form; narrow local
    // passes also specialised for a single encoding (U8 / U16 / F32; ENC_* values 0..2).  Null: not instantiated.
    template <bool W, bool R, int E>
    static const void* pass_kernel_f(int fast) {
        switch (fast) {
            case 0: return (const void*)k_pass<W, R, 0, E>;
            case 1: return (const void*)k_pass<W, R, 1, E>;
            case 2: return (const void*)k_pass<W, R, 2, E>;
            default: return (const void*)k_pass<W, R, 3, E>;
        }
    }
    static const void* pass_kernel(bool wide, bool remote, int fast, int encu) {
        if (wide) return encu >= 0 ? nullptr : (remote ? pass_kernel_f<true, true, -1>(fast) : pass_kernel_f<true, false, -1>(fast));
        if (remote) return encu >= 0 ? nullptr : pass_kernel_f<false, true, -1>(fast);
        switch (encu) {
            case ENC_U8: return pass_kernel_f<false, false, ENC_U8>(fast);
            case ENC_U16: return pass_kernel_f<false, false, ENC_U16>(fast);
            case ENC_F32: return pass_kernel_f<false, false, ENC_F32>(fast);
            default: return pass_kernel_f<false, false, -1>(fast);
        }
    }
    // the partition kernel of a pass; a.remote != null: the fused exchange pass of a sharded build (buckets in their owners' memory)
    void partition_launch(const PassArgs& a) {
        const int nsm = sm_count();
        prof_begin(K_PASS, 0, a.pass);
        const uint32_t gw = std::min<uint32_t>(a.cap_tiles, (uint32_t)(nsm * PassCfg<true>::blocks_per_sm));
        const uint32_t gn = std::min<uint32_t>(a.cap_tiles, (uint32_t)(nsm * PassCfg<false>::blocks_per_sm));
        // one encoding for every level this pass touches?  (level L+1, and L+2 / the next pass's first level when they are used)
        int encu = a.enc1;
        if (a.G == 2 && a.enc2 != encu) encu = -1;
        if (a.Gn > 0 && a.ench != encu) encu = -1;
        if (a.wide || a.remote || encu == ENC_F64 || std::getenv("PCV_PASS_GENERIC")) encu = -1;
        const void* fn = pass_kernel(a.wide, a.remote != nullptr, a.fast, encu);
        PassArgs arg = a;
        void* params[1] = {&arg};
        PCV_CUDA_CHECK(cudaLaunchKernel(fn, dim3(a.wide ? gw : gn), dim3(a.wide ? PassCfg<true>::threads : PassCfg<false>::threads), params,
                                        a.wide ? PassSmem<true>::bytes : PassSmem<false>::bytes, stream));
        prof_end();
    }
    void partition(const PassArgs& a) {
        partition_launch(a);
        ++launches;
        pass_wide = a.wide;
        PCV_CUDA_CHECK(cudaGetLastError());
    }
    void hist_scan_launch(const PassArgs& a) {
        const int nsm = sm_count();
        const int th = a.nbins < 32 ? 32 : a.nbins;
        prof_begin(K_DIGHIST, 0, a.pass);
        k_tile_index<<<std::min<uint32_t>(a.cap_chunks, 1024u), 256, 0, stream>>>(a);
        k_dighist<<<nsm * 8, kDigThreads, 0, stream>>>(a);
        prof_end();
        prof_begin(K_SCAN, 0, a.pass);
        k_scan_chunk_sums<<<std::min<uint32_t>(a.cap_chunks, 2048u), th, 0, stream>>>(a);
        k_scan_nodes<<<std::min<uint32_t>(a.cap_active, 2048u), th, 0, stream>>>(a);
        k_scan_tiles<<<std::min<uint32_t>(a.cap_chunks, 2048u), th, 0, stream>>>(a);
        prof_end();
    }
    void hist_scan(const PassArgs& a) override {
        hist_scan_launch(a);
        launches += 5;
        PCV_CUDA_CHECK(cudaGetLastError());
    }
    bool pass_wide = false;
    void pass_points(int pass, uint64_t npoints, uint64_t leaf_points) override {
        const uint64_t rec = pass_wide ? sizeof(RecW) : sizeof(RecN);
        for (auto& p : pending) {
            if (p.pass != pass || p.bytes != 0) continue;
            if (p.k == K_DIGHIST) p.bytes = npoints;
            if (p.k == K_SCAN) p.bytes = (npoints / kTilePoints + 1) * 64 * 12;
            if (p.k == K_PASS) p.bytes = npoints * (rec + 4 + 1) + (npoints - leaf_points) * (rec + 4 + 1) + leaf_points * (rec + 4);
        }
    }
    void place(const PlaceArgs& a_in) override {
        if (a_in.ntiles == 0) return;
        PlaceArgs a = a_in;
        LeafTile* tiles = (LeafTile*)dmalloc((size_t)a.ntiles * sizeof(LeafTile));
        a.tiles = tiles;
        prof_begin(K_PLACE, a.npoints * ((a.wide ? sizeof(RecW) : sizeof(RecN)) + 3 + 3 + 4 + (a.out_intensity ? 8 : 0)) + a.xyz_bytes);
        k_place_tiles<<<a.nleaves, 128, 0, stream>>>(a, tiles);
        if (a.wide)
            k_place<true><<<a.ntiles, 256, PlaceSmem<true>::bytes, stream>>>(a);
        else
            k_place<false><<<a.ntiles, 256, PlaceSmem<false>::bytes, stream>>>(a);
        prof_end();
        launches += 2;
        PCV_CUDA_CHECK(cudaGetLastError());
        dfree(tiles);
    }

    void bbox(const PointsView& p, double mn[3], double mx[3]) {
        if (p.n == 0) {  // generation.rs:269: unwrap_or_else(Aabb::zero)
            for (int a = 0; a < 3; ++a) mn[a] = mx[a] = 0.0;
            return;
        }
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        const int blocks = (int)std::min<uint64_t>((uint64_t)sms * 8, (p.n + 255) / 256);
        double* d = (double*)dmalloc((size_t)blocks * 6 * 8);
        prof_begin(K_BBOX, p.n * 24);
        k_bbox<<<blocks, 256, 0, stream>>>(p, d);
        prof_end();
        ++launches;
        PCV_CUDA_CHECK(cudaGetLastError());
        std::vector<double> h((size_t)blocks * 6);
        d2h(h.data(), d, h.size() * 8);
        dfree(d);
        for (int a = 0; a < 3; ++a) {
            mn[a] = h[a];
            mx[a] = h[3 + a];
        }
        for (int b = 1; b < blocks; ++b)
            for (int a = 0; a < 3; ++a) {
                mn[a] = std::fmin(mn[a], h[(size_t)b * 6 + a]);
                mx[a] = std::fmax(mx[a], h[(size_t)b * 6 + 3 + a]);
            }
    }
};

}  // namespace pcv
