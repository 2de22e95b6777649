// query_batch_points_plan.h — host-only planning of the batched point queries that return their points
// (pcv_query_batch_points_device and its cell-union and S2 forms, query_batch_points.inl).  No CUDA: tests compile it with g++.
//
//   qbp_key_bits:  the radix-sort key of a (location, node) pair: location above node index, so that sorting by key puts the
//                  pairs in (location, node index) order; the bits the sort has to look at.
//   qbp_slabs:     the sorted work list (tiles of at most kQueryTile points) cut into consecutive slabs of at most
//                  kQbpSlabTiles tiles; every slab is counted, scanned and placed before the next, so the mask and work-list
//                  scratch never exceeds qbp_slab_bytes() whatever the batch.
//   qbp_offsets:   the per-location offsets of the output from the per-location survivor counts, and the total.
#pragma once
#include <cstdint>
#include <vector>

namespace pcv {

// Tiles per slab.  2^18 tiles of at most 2048 points: at most 2^29 survivors per slab, so slab-local offsets fit in u32.
constexpr uint64_t kQbpSlabTiles = 1ull << 18;
// The scratch of one slab tile: its QTile (16 B), its 2048-bit survivor mask (256 B), its survivor count and its offset (4 B each).
constexpr uint64_t kQbpTileBytes = 16 + 256 + 4 + 4;
// The scratch of one selected (location, node) pair besides the selection's own: sort keys in and out (8 B each), the sorted
// pair (8 B), its tile count and its first tile (8 B each).
constexpr uint64_t kQbpPairBytes = 8 + 8 + 8 + 8 + 8;

inline uint64_t qbp_slab_bytes(uint64_t slab_tiles = kQbpSlabTiles) { return slab_tiles * kQbpTileBytes; }

// Number of bits needed to hold every value below n (at least 1).
inline int qbp_bits_below(uint64_t n) {
    if (n <= 1) return 1;
    int b = 1;
    while (b < 64 && (n - 1) >> b) ++b;
    return b;
}

struct QbpKeyBits {
    int node_bits;  // key = location << node_bits | node
    int end_bit;    // the sort looks at bits [0, end_bit)
};
// nloc locations over nnodes nodes (or S2 cells); both are at most 2^32, so the key fits in 64 bits.
inline QbpKeyBits qbp_key_bits(uint64_t nloc, uint64_t nnodes) {
    const int nb = qbp_bits_below(nnodes), lb = qbp_bits_below(nloc);
    return QbpKeyBits{nb, nb + lb};
}
inline uint64_t qbp_key(uint32_t loc, uint32_t node, const QbpKeyBits& kb) { return ((uint64_t)loc << kb.node_bits) | node; }

struct QbpSlab {
    uint64_t first;  // first tile of the slab in the sorted work list
    uint64_t n;      // tiles in the slab
};
inline std::vector<QbpSlab> qbp_slabs(uint64_t ntiles, uint64_t slab_tiles = kQbpSlabTiles) {
    std::vector<QbpSlab> v;
    for (uint64_t f = 0; f < ntiles; f += slab_tiles) v.push_back(QbpSlab{f, ntiles - f < slab_tiles ? ntiles - f : slab_tiles});
    return v;
}

// off[0..n]: off[0] = 0, off[i + 1] = off[i] + counts[i]; returns off[n].
inline uint64_t qbp_offsets(const uint64_t* counts, uint32_t n, uint64_t* off) {
    off[0] = 0;
    for (uint32_t i = 0; i < n; ++i) off[i + 1] = off[i] + counts[i];
    return off[n];
}

}  // namespace pcv
