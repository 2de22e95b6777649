// query_batch_points.cuh — the kernels of the batched point queries that return their points (query_batch_points.inl).
//
//   k_qbp_keys        the sort key of every selected (location, node) pair: location above node index (query_batch_points_plan.h)
//   k_qbp_pair_tiles  the tiles of every sorted pair, for the exclusive scan that gives each pair its first tile
//   k_qbp_tiles       one slab of the sorted work list: tile t belongs to the last pair whose first tile is <= t
//   k_qbp_count       every point of the slab decoded and tested once (decode_staged / point_passes, as k_cull_fused): per
//                     tile its survivor count and a 2048-bit survivor mask, per location its survivors
//   k_qbp_place       the survivors of every tile, and only those, decoded again and written at the tile's offset plus their
//                     rank in the tile: thread k of a round takes the k-th survivor, so stores are contiguous
//   k_qbp_advance     the running base: the output position of the next slab's first survivor
#pragma once

namespace pcv {

constexpr uint32_t kQbpMaskWords = kQueryTile / 32;  // one bit per point of a tile: point i of the tile is bit i & 31 of word i >> 5

__global__ void __launch_bounds__(256) k_qbp_keys(const uint2* __restrict__ pairs, uint32_t n, int node_bits, unsigned long long* __restrict__ keys) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint2 p = pairs[i];
        keys[i] = ((unsigned long long)(p.x & ~kTileIn) << node_bits) | p.y;
    }
}

__global__ void __launch_bounds__(256) k_qbp_pair_tiles(const uint2* __restrict__ pairs, uint32_t n, const QNode* __restrict__ nodes,
                                                        unsigned long long* __restrict__ ntiles) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        ntiles[i] = (nodes[pairs[i].y].n + kQueryTile - 1) / kQueryTile;
}

// tiles[j] = tile first + j of the work list; first_tile[i] = the first tile of sorted pair i (exclusive scan, non-decreasing).
__global__ void __launch_bounds__(256) k_qbp_tiles(const uint2* __restrict__ pairs, const unsigned long long* __restrict__ first_tile, uint32_t npairs,
                                                   const QNode* __restrict__ nodes, unsigned long long first, uint32_t n, QTile* __restrict__ tiles) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const unsigned long long t = first + j;
        uint32_t lo = 0, hi = npairs;  // the last pair with first_tile <= t: first_tile[0] = 0 <= t
        while (hi - lo > 1) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (first_tile[mid] <= t)
                lo = mid;
            else
                hi = mid;
        }
        const uint2 p = pairs[lo];
        const uint32_t k = (uint32_t)(t - first_tile[lo]), cnt = nodes[p.y].n;
        tiles[j] = QTile{p.x, p.y, k * kQueryTile, min(kQueryTile, cnt - k * kQueryTile)};
    }
}

struct QbpArgs {
    CullArgs c;                      // geoms, nodes, tiles (the slab), point arrays, filters; out_xyz / out_rgb / out_intensity
    uint32_t* tile_cnt;              // [slab tile] survivors
    uint32_t* mask;                  // [slab tile][kQbpMaskWords]; nullptr: count only
    unsigned long long* kept;        // [location] survivors
    unsigned long long* pos_bytes;   // position bytes of the survivors (3 bpc each), for the statistics
    const uint32_t* tile_off;        // [slab tile] exclusive scan of tile_cnt
    const unsigned long long* base;  // output position of the slab's first survivor
    unsigned long long cap;          // output capacity: survivors at or past it are not stored
    uint64_t* out_src;               // may be nullptr
};

__global__ void __launch_bounds__(256) k_qbp_count(const __grid_constant__ QbpArgs f, uint32_t ntiles) {
    __shared__ __align__(16) uint8_t sxyz[kCullStage];
    __shared__ uint32_t smask[kQbpMaskWords];
    __shared__ uint64_t scells[kCellsShared];
    const CullArgs& a = f.c;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long pos_bytes = 0;  // warp 0, lane 0 only
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
        for (uint32_t r0 = 0; r0 < t.count; r0 += 256) {
            const uint32_t i = r0 + threadIdx.x;
            bool keep = false;
            if (i < t.count) {
                double p[3];
                if (staged) {
                    decode_staged(sxyz, i, nd, p);
                } else {
#pragma unroll
                    for (int k = 0; k < 3; ++k) p[k] = decode1_fast(load_code(src + ((size_t)i * 3 + k) * bpc, nd.enc), nd.m[k], nd.e, nd.enc);
                }
                keep = point_passes(a, g, cells, all_in, p, nd.point_off + t.first + i);
            }
            const unsigned bal = __ballot_sync(0xffffffffu, keep);
            if (lane == 0) smask[(r0 >> 5) + warp] = bal;
        }
        __syncthreads();
        if (warp == 0) {
            const uint32_t used = ((t.count + 255u) >> 8) * 8u;  // words of the rounds that ran; the rest of the mask is zero
            const uint32_t w0 = (uint32_t)lane < used ? smask[lane] : 0u, w1 = (uint32_t)lane + 32u < used ? smask[lane + 32] : 0u;
            if (f.mask) {
                f.mask[(size_t)ti * kQbpMaskWords + lane] = w0;
                f.mask[(size_t)ti * kQbpMaskWords + 32 + lane] = w1;
            }
            uint32_t n = __popc(w0) + __popc(w1);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
            if (lane == 0) {
                f.tile_cnt[ti] = n;
                if (n) atomicAdd(&f.kept[loc], (unsigned long long)n);
                pos_bytes += (unsigned long long)n * 3ull * (unsigned long long)bpc;
            }
        }
        __syncthreads();  // sxyz and smask are reused by the next tile
    }
    if (threadIdx.x == 0 && pos_bytes) atomicAdd(f.pos_bytes, pos_bytes);
}

// The position of the r-th set bit (r < popc(w)) of w.
__device__ __forceinline__ uint32_t qbp_select_bit(uint32_t w, uint32_t r) {
    uint32_t pos = 0;
#pragma unroll
    for (uint32_t s = 16; s > 0; s >>= 1) {
        const uint32_t lo = __popc(w & ((1u << s) - 1u));
        if (r >= lo) {
            r -= lo;
            w >>= s;
            pos += s;
        }
    }
    return pos;
}

__global__ void __launch_bounds__(256) k_qbp_place(const __grid_constant__ QbpArgs f, uint32_t ntiles) {
    __shared__ uint32_t smask[kQbpMaskWords];
    __shared__ uint32_t spre[kQbpMaskWords];  // survivors in the words before each word
    __shared__ __align__(16) double st_xyz[256 * 3];
    __shared__ uint8_t st_rgb[256 * 3];
    const CullArgs& a = f.c;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned long long base = *f.base;
    for (uint32_t ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
        const uint32_t n = f.tile_cnt[ti];
        if (n == 0) continue;  // uniform over the block
        const QTile t = a.tiles[ti];
        const QNode nd = a.nodes[t.node];
        const int bpc = enc_bytes(nd.enc);
        if (warp == 0) {
            const uint32_t w0 = f.mask[(size_t)ti * kQbpMaskWords + lane], w1 = f.mask[(size_t)ti * kQbpMaskWords + 32 + lane];
            uint32_t i0 = __popc(w0), i1 = __popc(w1);
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y0 = __shfl_up_sync(0xffffffffu, i0, o), y1 = __shfl_up_sync(0xffffffffu, i1, o);
                if (lane >= o) i0 += y0, i1 += y1;
            }
            const uint32_t half = __shfl_sync(0xffffffffu, i0, 31);
            smask[lane] = w0;
            smask[lane + 32] = w1;
            spre[lane] = i0 - __popc(w0);
            spre[lane + 32] = half + i1 - __popc(w1);
        }
        __syncthreads();
        const unsigned long long d0 = base + f.tile_off[ti];
        for (uint32_t k0 = 0; k0 < n; k0 += 256) {
            const uint32_t k = k0 + threadIdx.x;
            if (k < n) {
                uint32_t w = 0;  // the last word with spre[w] <= k: it holds survivor k
#pragma unroll
                for (uint32_t s = kQbpMaskWords / 2; s > 0; s >>= 1)
                    if (spre[w + s] <= k) w += s;
                const uint32_t i = t.first + w * 32 + qbp_select_bit(smask[w], k - spre[w]);
                double p[3];
                decode_point(a.xyz, nd, bpc, i, p);
                st_xyz[3 * threadIdx.x] = p[0];
                st_xyz[3 * threadIdx.x + 1] = p[1];
                st_xyz[3 * threadIdx.x + 2] = p[2];
                const uint64_t sp = nd.point_off + i;
                if (a.out_rgb) {
                    st_rgb[3 * threadIdx.x] = a.rgb[3 * sp];
                    st_rgb[3 * threadIdx.x + 1] = a.rgb[3 * sp + 1];
                    st_rgb[3 * threadIdx.x + 2] = a.rgb[3 * sp + 2];
                }
                const unsigned long long dst = d0 + k;
                if (dst < f.cap) {
                    if (a.out_intensity) a.out_intensity[dst] = a.intensity[sp];
                    if (f.out_src) f.out_src[dst] = a.src[sp];
                }
            }
            __syncthreads();
            const unsigned long long b = d0 + k0;
            const uint32_t room = b >= f.cap ? 0u : (uint32_t)min((unsigned long long)min(256u, n - k0), f.cap - b);
            for (uint32_t q = threadIdx.x; q < 3 * room; q += 256) a.out_xyz[3 * b + q] = st_xyz[q];
            if (a.out_rgb)
                for (uint32_t q = threadIdx.x; q < 3 * room; q += 256) a.out_rgb[3 * b + q] = st_rgb[q];
            __syncthreads();  // the staging arrays are reused by the next round
        }
    }
}

// *base += the survivors of the slab just placed (its last tile's offset plus count)
__global__ void k_qbp_advance(unsigned long long* base, const uint32_t* tile_off, const uint32_t* tile_cnt, uint32_t n) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *base += (unsigned long long)tile_off[n - 1] + tile_cnt[n - 1];
}

}  // namespace pcv
