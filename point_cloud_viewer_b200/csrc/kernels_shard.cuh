// kernels_shard.cuh — multi-GPU sharding helpers (SURVEY 8e): level-k prefix cell of every point (the first k steps
// of the re-quantising descent on the raw positions, i.e. exactly the cell the single-GPU build would route the
// point to), its 8^k histogram, and a stable pack of the points by destination rank into contiguous send buffers.
#pragma once
#include <cuda_runtime.h>

#include "kernels_build.cuh"

namespace pcv {

struct PrefixArgs {
    PointsView pts;
    LevelTable lv;
    double root_min[3];
    int k;
    int nbins;  // 8^k
};

__device__ __forceinline__ unsigned prefix_cell_of(const PrefixArgs& a, const double p[3]) {
    double q[3] = {p[0], p[1], p[2]};
    double m[3] = {a.root_min[0], a.root_min[1], a.root_min[2]};
    if (a.lv.fast) {  // the kernels' straight-line descent (chain_device.cuh); a flagged numerator falls through to the generic path
        double e = a.lv.edge[0];
        unsigned cell = 0, bad = 0;
        for (int j = 1; j <= a.k; ++j) {
            const double eh = a.lv.edge[j], ry = a.lv.ry[j];
            uint64_t code[3];
            PCV_ENC_SWITCH(a.lv.enc[j], cell = (cell << 3) | level_step<ENC, 1, true>(q, m, e, eh, ry, code, bad);)
            e = eh;
        }
        if (!bad) return cell;
        q[0] = p[0], q[1] = p[1], q[2] = p[2];
        m[0] = a.root_min[0], m[1] = a.root_min[1], m[2] = a.root_min[2];
    }
    double e = a.lv.edge[0];
    unsigned cell = 0;
    for (int j = 1; j <= a.k; ++j) {
        Step s = descend(q, m, e, a.lv.edge[j], a.lv.enc[j]);
        cell = (cell << 3) | s.digit;
        e = a.lv.edge[j];
    }
    return cell;
}

__device__ __forceinline__ unsigned prefix_cell(const PrefixArgs& a, uint64_t i) {
    double q[3] = {__ldg(a.pts.x + i * a.pts.stride), __ldg(a.pts.y + i * a.pts.stride), __ldg(a.pts.z + i * a.pts.stride)};
    return prefix_cell_of(a, q);
}

// `cells` (optional): the cell of every point, kept for the pack that follows so that it does not repeat the descent.
// `bbox_partial` (optional, [gridDim.x][6]): min / max of the block's points - find_bounding_box folded into the same read.
__global__ void __launch_bounds__(256) k_prefix_hist(const __grid_constant__ PrefixArgs a, unsigned long long* __restrict__ counts, uint16_t* __restrict__ cells,
                                                     double* __restrict__ bbox_partial) {
    extern __shared__ uint32_t sh_cnt[];
    for (int b = threadIdx.x; b < a.nbins; b += blockDim.x) sh_cnt[b] = 0;
    __syncthreads();
    double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.pts.n; i += step) {
        const double p[3] = {__ldg(a.pts.x + i * a.pts.stride), __ldg(a.pts.y + i * a.pts.stride), __ldg(a.pts.z + i * a.pts.stride)};
#pragma unroll
        for (int k = 0; k < 3; ++k) mn[k] = fmin(mn[k], p[k]), mx[k] = fmax(mx[k], p[k]);
        const unsigned cell = prefix_cell_of(a, p);
        if (cells) cells[i] = (uint16_t)cell;
        atomicAdd(&sh_cnt[cell], 1u);
    }
    __syncthreads();
    for (int b = threadIdx.x; b < a.nbins; b += blockDim.x)
        if (sh_cnt[b]) atomicAdd(&counts[b], (unsigned long long)sh_cnt[b]);
    if (bbox_partial) {
        __shared__ double sh[8][6];
        const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double lo = warp_min(mn[k]), hi = warp_max(mx[k]);
            if (l == 0) sh[w][k] = lo, sh[w][3 + k] = hi;
        }
        __syncthreads();
        if (threadIdx.x < 6) {
            double v = sh[0][threadIdx.x];
            for (int k = 1; k < 8; ++k) v = threadIdx.x < 3 ? fmin(v, sh[k][threadIdx.x]) : fmax(v, sh[k][threadIdx.x]);
            bbox_partial[(size_t)blockIdx.x * 6 + threadIdx.x] = v;
        }
    }
}

// ---- pack -------------------------------------------------------------------------------------------------------
constexpr uint32_t kPackTile = 4096;
constexpr int kMaxRanks = 64;

struct PackArgs {
    PrefixArgs p;
    const int32_t* cell_to_rank;  // device, nbins; a negative entry drops the cell's points (dest 0xFF, not counted, not stored)
    uint32_t nranks, ntiles;
    const uint16_t* cells;  // optional: level-(k + cell_shift / 3) cells from the histogram call over the same points
    uint32_t cell_shift;
    uint8_t* dest;        // per point destination rank (written by the count pass)
    uint32_t* counts;     // [nranks][ntiles]; after the scan: first output slot of (rank, tile)
    const uint64_t* gidx_in;  // optional global indices of the local points
    uint64_t gidx_base;       // used when gidx_in == nullptr: global index = base + i
    double* out_xyz;          // n * 3 (AoS)
    uint8_t* out_rgb;
    float* out_intensity;
    uint64_t* out_idx;        // optional
    uint64_t out_base;        // first output slot of this call: successive calls over the chunks of one stream append
};

__global__ void __launch_bounds__(256) k_pack_count(const __grid_constant__ PackArgs a) {
    __shared__ uint32_t cnt[kMaxRanks];
    if (threadIdx.x < kMaxRanks) cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t t0 = (uint64_t)blockIdx.x * kPackTile;
    const uint32_t n = (uint32_t)min((uint64_t)kPackTile, a.p.pts.n - t0);
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned cell = a.cells ? (unsigned)a.cells[t0 + i] >> a.cell_shift : prefix_cell(a.p, t0 + i);
        const int r = a.cell_to_rank[cell];
        a.dest[t0 + i] = r < 0 ? (uint8_t)0xFFu : (uint8_t)r;
        if (r >= 0) atomicAdd(&cnt[r], 1u);
    }
    __syncthreads();
    if (threadIdx.x < a.nranks) a.counts[(size_t)threadIdx.x * a.ntiles + blockIdx.x] = cnt[threadIdx.x];
}

__global__ void __launch_bounds__(256) k_pack_scatter(const __grid_constant__ PackArgs a) {
    __shared__ uint32_t base[kMaxRanks];
    __shared__ uint32_t wc[8][kMaxRanks];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < a.nranks) base[threadIdx.x] = a.counts[(size_t)threadIdx.x * a.ntiles + blockIdx.x];
    const uint64_t t0 = (uint64_t)blockIdx.x * kPackTile;
    const uint32_t n = (uint32_t)min((uint64_t)kPackTile, a.p.pts.n - t0);
    for (uint32_t r0 = 0; r0 < n; r0 += 256) {
        for (int i = threadIdx.x; i < 8 * kMaxRanks; i += 256) (&wc[0][0])[i] = 0;
        __syncthreads();
        const uint32_t i = r0 + threadIdx.x;
        const uint32_t d = i < n ? a.dest[t0 + i] : 0xFFu;
        const unsigned mask = __match_any_sync(0xffffffffu, d);
        const uint32_t rank = __popc(mask & ((1u << lane) - 1u));
        if (d != 0xFFu && lane == __ffs(mask) - 1) wc[warp][d] = __popc(mask);
        __syncthreads();
        uint32_t before = 0;
        if (d != 0xFFu) {
            for (int w = 0; w < warp; ++w) before += wc[w][d];
            const uint64_t dst = a.out_base + base[d] + before + rank;
            const uint64_t g = t0 + i;
            a.out_xyz[3 * dst] = __ldg(a.p.pts.x + g * a.p.pts.stride);
            a.out_xyz[3 * dst + 1] = __ldg(a.p.pts.y + g * a.p.pts.stride);
            a.out_xyz[3 * dst + 2] = __ldg(a.p.pts.z + g * a.p.pts.stride);
            a.out_rgb[3 * dst] = __ldg(a.p.pts.rgb + 3 * g);
            a.out_rgb[3 * dst + 1] = __ldg(a.p.pts.rgb + 3 * g + 1);
            a.out_rgb[3 * dst + 2] = __ldg(a.p.pts.rgb + 3 * g + 2);
            if (a.out_intensity) a.out_intensity[dst] = __ldg(a.p.pts.intensity + g);
            if (a.out_idx) a.out_idx[dst] = a.gidx_in ? __ldg(a.gidx_in + g) : a.gidx_base + g;
        }
        __syncthreads();
        if (threadIdx.x < a.nranks) {
            uint32_t s = 0;
            for (int w = 0; w < 8; ++w) s += wc[w][threadIdx.x];
            base[threadIdx.x] += s;
        }
        __syncthreads();
    }
}

// ---- fused pack + exchange ------------------------------------------------------------------------------------------
// The same stable ranking as k_pack_scatter, but every record is stored straight into its destination rank's receive
// arrays - local memory for the own rank, peer memory mapped through CUDA IPC for the others, i.e. the stores travel over
// NVLink / NVSwitch while the kernel is still ranking the next points.  No send buffers, no separate collective: the
// exchange is finished when the kernel is (followed by one inter-process barrier).  Receive arrays are SoA (x, y, z,
// index, intensity, packed colour) so that the lanes of a warp that share a destination write contiguous runs.
struct PeerTable {
    double* x[kMaxRanks];
    double* y[kMaxRanks];
    double* z[kMaxRanks];
    uint64_t* idx[kMaxRanks];
    float* intensity[kMaxRanks];
    uint32_t* col[kMaxRanks];    // r | g << 8 | b << 16
    uint64_t first[kMaxRanks];   // first slot of this rank's block inside destination d's arrays
};

__global__ void __launch_bounds__(256) k_pack_exchange(const __grid_constant__ PackArgs a, const PeerTable* __restrict__ pt) {
    __shared__ uint64_t base[kMaxRanks];
    __shared__ uint32_t wc[8][kMaxRanks];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < a.nranks) {
        const uint32_t* row = a.counts + (size_t)threadIdx.x * a.ntiles;  // exclusive prefix over (rank, tile), rank-major
        base[threadIdx.x] = pt->first[threadIdx.x] + (row[blockIdx.x] - row[0]);
    }
    const uint64_t t0 = (uint64_t)blockIdx.x * kPackTile;
    const uint32_t n = (uint32_t)min((uint64_t)kPackTile, a.p.pts.n - t0);
    for (uint32_t r0 = 0; r0 < n; r0 += 256) {
        for (int i = threadIdx.x; i < 8 * kMaxRanks; i += 256) (&wc[0][0])[i] = 0;
        __syncthreads();
        const uint32_t i = r0 + threadIdx.x;
        const uint32_t d = i < n ? a.dest[t0 + i] : 0xFFu;
        const unsigned mask = __match_any_sync(0xffffffffu, d);
        const uint32_t rank = __popc(mask & ((1u << lane) - 1u));
        if (d != 0xFFu && lane == __ffs(mask) - 1) wc[warp][d] = __popc(mask);
        __syncthreads();
        if (d != 0xFFu) {
            uint32_t before = 0;
            for (int w = 0; w < warp; ++w) before += wc[w][d];
            const uint64_t dst = base[d] + before + rank;
            const uint64_t g = t0 + i;
            pt->x[d][dst] = __ldg(a.p.pts.x + g * a.p.pts.stride);
            pt->y[d][dst] = __ldg(a.p.pts.y + g * a.p.pts.stride);
            pt->z[d][dst] = __ldg(a.p.pts.z + g * a.p.pts.stride);
            const uint8_t* c = a.p.pts.rgb + 3 * g;
            pt->col[d][dst] = (uint32_t)__ldg(c) | ((uint32_t)__ldg(c + 1) << 8) | ((uint32_t)__ldg(c + 2) << 16);
            if (a.p.pts.intensity) pt->intensity[d][dst] = __ldg(a.p.pts.intensity + g);
            pt->idx[d][dst] = a.gidx_in ? __ldg(a.gidx_in + g) : a.gidx_base + g;
        }
        __syncthreads();
        if (threadIdx.x < a.nranks) {
            uint32_t s = 0;
            for (int w = 0; w < 8; ++w) s += wc[w][threadIdx.x];
            base[threadIdx.x] += s;
        }
        __syncthreads();
    }
}

// v2: the same exchange with the records of 1024 points first sorted by destination inside shared memory, so that the
// stores over NVLink are contiguous runs per destination (full 128-byte lines) instead of the few lanes of a warp that
// happen to share a destination - the more ranks, the shorter those were (pack+exchange at N = 2 / 4: 25 / 46 ms with v1).
constexpr int kXChunk = 1024;
__global__ void __launch_bounds__(256) k_pack_exchange_sorted(const __grid_constant__ PackArgs a, const PeerTable* __restrict__ pt) {
    __shared__ double sx[kXChunk], sy[kXChunk], sz[kXChunk];
    __shared__ uint64_t sidx[kXChunk];
    __shared__ uint32_t scol[kXChunk];
    __shared__ float sint[kXChunk];
    __shared__ uint8_t sdst[kXChunk];
    __shared__ uint64_t base[kMaxRanks];  // next free slot of this rank's block inside every destination's arrays
    __shared__ uint32_t ccount[kMaxRanks], cstart[kMaxRanks], fill[kMaxRanks];
    __shared__ uint32_t wc[8][kMaxRanks];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < (int)a.nranks) {
        const uint32_t* row = a.counts + (size_t)tid * a.ntiles;  // exclusive prefix over (rank, tile), rank-major
        base[tid] = pt->first[tid] + (row[blockIdx.x] - row[0]);
    }
    const uint64_t t0 = (uint64_t)blockIdx.x * kPackTile;
    const uint32_t n = (uint32_t)min((uint64_t)kPackTile, a.p.pts.n - t0);
    const bool has_int = a.p.pts.intensity != nullptr;
    for (uint32_t c0 = 0; c0 < n; c0 += kXChunk) {
        const uint32_t m = min((uint32_t)kXChunk, n - c0);
        // (1) per-destination counts of the chunk -> sorted start of every destination
        if (tid < kMaxRanks) ccount[tid] = 0;
        __syncthreads();
        for (uint32_t i = tid; i < m; i += 256) atomicAdd(&ccount[a.dest[t0 + c0 + i]], 1u);
        __syncthreads();
        if (tid == 0) {
            uint32_t run = 0;
            for (uint32_t r = 0; r < a.nranks; ++r) {
                cstart[r] = fill[r] = run;
                run += ccount[r];
            }
        }
        __syncthreads();
        // (2) stable sorted position of every point (round by round, warp by warp, lane rank), records staged there
        for (uint32_t r0 = 0; r0 < m; r0 += 256) {
            for (int i = tid; i < 8 * kMaxRanks; i += 256) (&wc[0][0])[i] = 0;
            __syncthreads();
            const uint32_t i = r0 + tid;
            const uint32_t d = i < m ? a.dest[t0 + c0 + i] : 0xFFu;
            const unsigned mask = __match_any_sync(0xffffffffu, d);
            const uint32_t rank = __popc(mask & ((1u << lane) - 1u));
            if (d != 0xFFu && lane == __ffs(mask) - 1) wc[warp][d] = __popc(mask);
            __syncthreads();
            if (d != 0xFFu) {
                uint32_t before = 0;
                for (int w = 0; w < warp; ++w) before += wc[w][d];
                const uint32_t lp = fill[d] + before + rank;
                const uint64_t g = t0 + c0 + i;
                sx[lp] = __ldg(a.p.pts.x + g * a.p.pts.stride);
                sy[lp] = __ldg(a.p.pts.y + g * a.p.pts.stride);
                sz[lp] = __ldg(a.p.pts.z + g * a.p.pts.stride);
                const uint8_t* c = a.p.pts.rgb + 3 * g;
                scol[lp] = (uint32_t)__ldg(c) | ((uint32_t)__ldg(c + 1) << 8) | ((uint32_t)__ldg(c + 2) << 16);
                if (has_int) sint[lp] = __ldg(a.p.pts.intensity + g);
                sidx[lp] = a.gidx_in ? __ldg(a.gidx_in + g) : a.gidx_base + g;
                sdst[lp] = (uint8_t)d;
            }
            __syncthreads();
            if (tid < (int)a.nranks) {
                uint32_t sum = 0;
                for (int w = 0; w < 8; ++w) sum += wc[w][tid];
                fill[tid] += sum;
            }
            __syncthreads();
        }
        // (3) consecutive threads store consecutive records of a destination's run
        for (uint32_t p = tid; p < m; p += 256) {
            const uint32_t d = sdst[p];
            const uint64_t dst = base[d] + (p - cstart[d]);
            pt->x[d][dst] = sx[p];
            pt->y[d][dst] = sy[p];
            pt->z[d][dst] = sz[p];
            pt->idx[d][dst] = sidx[p];
            pt->col[d][dst] = scol[p];
            if (has_int) pt->intensity[d][dst] = sint[p];
        }
        __syncthreads();
        if (tid < (int)a.nranks) base[tid] += ccount[tid];
        __syncthreads();
    }
}

// packed colours (as exchanged) -> the r, g, b byte array the build takes
// ---- exchange of ingested records (the multi-GPU path of round 2) ------------------------------------------------------------
// Every rank runs the ingest step on its own slice (level-1 codes + the digits of levels 1..2, kernels_build.cuh) and then moves
// each record ONCE into the receive slab of the rank that owns its level-k cell: 17 bytes per point over NVLink (three codes
// 12 B + packed colour 4 B in one 16-byte store, digits 1 B [+ intensity 4 B]; the record's index is its slot in the slab and is
// not transmitted) instead of the 40-byte raw point, and the owner's build starts at its
// first partition pass without repeating any arithmetic.  The kernel is the partition kernel's tile machinery with the
// destination rank as the bucket: stage the tile (TMA), rank by bucket with __match_any_sync, sort the tile by destination in
// shared memory, then store whole runs straight into the peers' memory (CUDA-IPC mapped slabs), so that the stores are full
// lines on the link and overlap the ranking of the next tiles.  Inside a destination the order is (source rank, local index),
// i.e. global index order - the reference's stable stream order.  idx of a stored record = its slot in the destination slab.
constexpr int kExThreads = 256;
struct ExchangeArgs {
    const void* rec;
    const uint32_t* col;
    const uint8_t* dig;
    const float* intensity;       // optional
    const uint32_t* tile_counts;  // [ntiles][nbins] exclusive prefix over the earlier tiles, per digit (scan of the ingest's histogram)
    uint64_t n;
    uint32_t ntiles;
    int nbins;                    // digits per record: 8 or 64
    int cell_shift;               // level-k cell = digit >> cell_shift
    int nranks;
    bool wide;
    uint8_t cell_to_rank[64];
    unsigned long long dst_first[kMaxRanks];  // first slot of this source's block in every destination
    void* dst_rec[kMaxRanks];
    uint32_t* dst_col[kMaxRanks];
    uint8_t* dst_dig[kMaxRanks];
    float* dst_intensity[kMaxRanks];
    uint8_t* dest_out;            // [n] destination rank of every local point (kept by the sender: provenance look-ups)
};
struct ExSmem {
    static constexpr size_t rec_bytes = 16;
    static constexpr size_t off_col = (size_t)kTilePoints * 32;  // sized for wide records
    static constexpr size_t off_dig = off_col + ((size_t)kTilePoints + 4) * 4;
    static constexpr size_t off_pfx = off_dig + (size_t)kTilePoints + 32;
    static constexpr size_t off_perm = off_pfx + 64 * 4;
    static constexpr size_t off_cnt = off_perm + (size_t)kTilePoints * 4;
    static constexpr size_t off_first = off_cnt + (size_t)(kExThreads / 32) * kMaxRanks * 4;
    static constexpr size_t off_start = off_first + (size_t)kMaxRanks * 8;
    static constexpr size_t off_c2r = off_start + (size_t)kMaxRanks * 4;
    static constexpr size_t off_bar = off_c2r + 64;
    static constexpr size_t bytes = off_bar + 16;
};
template <bool WIDE>
__global__ void __launch_bounds__(kExThreads, 2) k_exchange_records(const __grid_constant__ ExchangeArgs a) {
    constexpr int kWarps = kExThreads / 32, kWarpItems = kTilePoints / kWarps, kSubRounds = kWarpItems / 32;
    constexpr size_t recsz = WIDE ? 32 : 16;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const unsigned char* srec = smem_raw;
    uint32_t* scol_base = reinterpret_cast<uint32_t*>(smem_raw + ExSmem::off_col);
    uint8_t* sdig_base = smem_raw + ExSmem::off_dig;
    uint32_t* spfx = reinterpret_cast<uint32_t*>(smem_raw + ExSmem::off_pfx);
    uint32_t* perm = reinterpret_cast<uint32_t*>(smem_raw + ExSmem::off_perm);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(smem_raw + ExSmem::off_cnt);                     // [warps][kMaxRanks]
    unsigned long long* rfirst = reinterpret_cast<unsigned long long*>(smem_raw + ExSmem::off_first);  // [ranks] slot of sorted position 0
    uint32_t* rstart = reinterpret_cast<uint32_t*>(smem_raw + ExSmem::off_start);               // [ranks] sorted start
    uint8_t* c2r = smem_raw + ExSmem::off_c2r;  // shared-memory copy: a per-thread indexed read of the kernel parameters is slow
    uint64_t* mbar = reinterpret_cast<uint64_t*>(smem_raw + ExSmem::off_bar);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nr = a.nranks;
    if (tid < 64) c2r[tid] = a.cell_to_rank[tid];
    if (tid == 0) mbar_init(mbar, 1);
    __syncthreads();
    uint32_t par = 0;
    for (uint32_t tile = blockIdx.x; tile < a.ntiles; tile += gridDim.x) {
        const uint64_t start = (uint64_t)tile * kTilePoints;
        const uint64_t rem = a.n - start;
        const uint32_t count = (uint32_t)(rem < kTilePoints ? rem : kTilePoints);
        const uint32_t coff = (uint32_t)(start & 3), doff = (uint32_t)(start & 15);
        const uint32_t* scol = scol_base + coff;
        const uint8_t* sdig = sdig_base + doff;
        if (tid == 0) {
            const uint32_t rec_bytes = count * (uint32_t)recsz;
            const uint32_t col_bytes = ((coff + count) * 4u + 15u) & ~15u;
            const uint32_t dig_bytes = (doff + count + 15u) & ~15u;
            const uint32_t pfx_bytes = (uint32_t)a.nbins * 4u;
            mbar_expect_tx(mbar, rec_bytes + col_bytes + dig_bytes + pfx_bytes);
            tma_bulk_load(smem_raw, reinterpret_cast<const unsigned char*>(a.rec) + start * recsz, rec_bytes, mbar);
            tma_bulk_load(scol_base, a.col + (start - coff), col_bytes, mbar);
            tma_bulk_load(sdig_base, a.dig + (start - doff), dig_bytes, mbar);
            tma_bulk_load(spfx, a.tile_counts + (size_t)tile * a.nbins, pfx_bytes, mbar);
        }
        for (int i = tid; i < kWarps * kMaxRanks; i += kExThreads) cnt[i] = 0;
        mbar_wait(mbar, par);
        par ^= 1u;
        __syncthreads();
        // rank of every item from its digit; lanes grouped by destination
        uint32_t info[kSubRounds];
#pragma unroll
        for (int r = 0; r < kSubRounds; ++r) {
            const uint32_t i = warp * kWarpItems + r * 32 + lane;
            uint32_t lbv = 0xFFFFu;
            if (i < count) lbv = c2r[(sdig[i] & (uint32_t)(a.nbins - 1)) >> a.cell_shift];
            const unsigned mask = __match_any_sync(0xffffffffu, lbv);
            const uint32_t leader = (uint32_t)__ffs(mask) - 1u, gsize = (uint32_t)__popc(mask), rank = (uint32_t)__popc(mask & ((1u << lane) - 1u));
            info[r] = lbv | (rank << 16) | (leader << 21) | ((gsize - 1u) << 26);
            if (lbv != 0xFFFFu && lane == (int)leader) cnt[warp * kMaxRanks + lbv] += gsize;
            __syncwarp();
        }
        __syncthreads();
        if (warp == 0) {  // per destination: total, sorted start, slot of sorted position 0, per-warp offsets
            uint32_t tot[2] = {0, 0};
            unsigned long long early[2] = {0, 0};  // records of this source for the destination in earlier tiles
            for (int j = 0; j < 2; ++j) {
                const int lb = lane + 32 * j;
                if (lb < nr) {
                    for (int w = 0; w < kWarps; ++w) tot[j] += cnt[w * kMaxRanks + lb];
                    for (int d = 0; d < a.nbins; ++d)
                        if (c2r[d >> a.cell_shift] == lb) early[j] += spfx[d];
                }
            }
            uint32_t carry = 0;
            for (int j = 0; j < 2; ++j) {
                uint32_t incl = tot[j];
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += u;
                }
                const uint32_t excl = carry + incl - tot[j];
                carry += __shfl_sync(0xffffffffu, incl, 31);
                const int lb = lane + 32 * j;
                if (lb < nr) {
                    rstart[lb] = excl;
                    rfirst[lb] = a.dst_first[lb] + early[j];
                    uint32_t run = excl;
                    for (int w = 0; w < kWarps; ++w) {
                        const uint32_t c = cnt[w * kMaxRanks + lb];
                        cnt[w * kMaxRanks + lb] = run;
                        run += c;
                    }
                }
            }
        }
        __syncthreads();
#pragma unroll
        for (int r = 0; r < kSubRounds; ++r) {
            const uint32_t i = warp * kWarpItems + r * 32 + lane;
            const uint32_t lbv = info[r] & 0xFFFFu, rank = (info[r] >> 16) & 31u, gsize = ((info[r] >> 26) & 31u) + 1u;
            const int leader = (int)((info[r] >> 21) & 31u);
            uint32_t old = 0;
            if (lane == leader && lbv != 0xFFFFu) {
                old = cnt[warp * kMaxRanks + lbv];
                cnt[warp * kMaxRanks + lbv] = old + gsize;
            }
            old = __shfl_sync(0xffffffffu, old, leader);
            if (lbv != 0xFFFFu) perm[old + rank] = i | (lbv << 12);
            __syncwarp();
        }
        __syncthreads();
        // whole runs into the owners' slabs (peer memory over NVLink, or local memory for the own rank)
        for (uint32_t p = tid; p < count; p += kExThreads) {
            const uint32_t e = perm[p], i = e & 2047u, lb = e >> 12;
            const unsigned long long slot = rfirst[lb] + (p - rstart[lb]);
            uint64_t c[3];
            uint32_t idx;
            smem_load_rec<WIDE>(srec, i, c, idx);
            if (WIDE) {
                store_rec<WIDE>(a.dst_rec[lb], slot, c, (uint32_t)slot);
                a.dst_col[lb][slot] = scol[i];
            } else {  // on the wire a narrow record is {code x 3, packed colour}: its index is its slot, which the owner knows
                store_rec<WIDE>(a.dst_rec[lb], slot, c, scol[i]);
            }
            a.dst_dig[lb][slot] = sdig[i];
            if (a.intensity) a.dst_intensity[lb][slot] = a.intensity[start + i];
            a.dest_out[start + i] = (uint8_t)lb;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_unpack_colours(const uint32_t* __restrict__ col, uint64_t n, uint8_t* __restrict__ rgb) {
    const uint64_t step = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += step) {
        const uint32_t c = __ldg(col + i);
        rgb[3 * i] = (uint8_t)c;
        rgb[3 * i + 1] = (uint8_t)(c >> 8);
        rgb[3 * i + 2] = (uint8_t)(c >> 16);
    }
}

}  // namespace pcv
