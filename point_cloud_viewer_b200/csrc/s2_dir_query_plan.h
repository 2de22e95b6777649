// s2_dir_query_plan.h — host-only planning of point queries straight from an S2 directory (s2_dir_query.inl; no CUDA: the CPU
// tests compile it with g++).
//   s2_dir_select_bytes: what one cell selection of some locations takes on the device
//   s2_dir_open_bytes:   what open checks the budget against: the cell table, one selection of one location, one chunk
//   s2_dir_scan_chunk:   the box scan's chunk (points, pieces) within what the budget leaves
//   s2_dir_loc_chunk:    how many locations one selection of a batch takes within what the budget leaves
#pragma once
#include <algorithm>
#include <cstdint>

#include "dir_query_plan.h"
#include "s2_dir_xray_plan.h"

namespace pcv {

// The selection of nloc locations over nc cells (s2_select): per location its projections (proj_bytes) and tested counter,
// the pair list of every (location, cell), and the counters.
inline uint64_t s2_dir_select_bytes(uint64_t nloc, uint64_t nc, uint64_t proj_bytes) { return nloc * (proj_bytes + 8 + 8 * nc) + 4 + 32; }

// Slack of a single-location call besides its selection: the location's geometry and the filter intervals.
constexpr uint64_t kS2DirCallSlack = 4096;

// The least budget open accepts: the cell table (query node, id and point box per cell: kS2WindowCellBytes), the selection of
// one location with its geometry (geom_bytes) and filters, and the smallest chunk of a query.
inline uint64_t s2_dir_open_bytes(uint64_t nc, uint64_t proj_bytes, uint64_t geom_bytes) {
    return kS2WindowCellBytes * nc + s2_dir_select_bytes(1, nc, proj_bytes) + geom_bytes + kS2DirCallSlack + dir_min_chunk_bytes();
}

// Device bytes of one scan chunk of `chunk` points and `pieces` pieces: positions, a query node (64 B) and a cell index per
// piece, and the work tiles (16 B each: a piece's tiles, at most one more per piece than the chunk's whole tiles).
inline uint64_t s2_dir_scan_bytes(uint64_t chunk, uint64_t pieces) { return 24 * chunk + pieces * (64 + 4) + (pieces + chunk / kDirTile + 1) * 16; }

// The scan's chunk within `room` bytes: at most 64 MiB of positions, pieces = max(64, chunk / 64) as the X-ray scan takes
// them, halved until it fits.  False: not even one tile of points fits.
inline bool s2_dir_scan_chunk(uint64_t room, uint64_t& chunk, uint64_t& pieces) {
    chunk = (64ull << 20) / 24;
    for (;;) {
        pieces = std::max<uint64_t>(64, chunk / 64);
        if (s2_dir_scan_bytes(chunk, pieces) <= room) return true;
        if (chunk <= kDirTile) return false;
        chunk = std::max<uint64_t>(kDirTile, chunk / 2);
    }
}

// Locations per selection of a batch of nloc over nc cells: as many as `room` holds (s2_dir_select_bytes), at most the
// selection kernel's grid height (65535) and 2^25 pairs (256 MiB of pair list).  0: not even one location fits.
inline uint64_t s2_dir_loc_chunk(uint64_t nloc, uint64_t nc, uint64_t proj_bytes, uint64_t room) {
    const uint64_t per = proj_bytes + 8 + 8 * nc;
    if (room < 36 + per) return 0;
    const uint64_t fit = (room - 36) / per;
    return std::min<uint64_t>({nloc, fit, 65535, std::max<uint64_t>(1, (1ull << 25) / std::max<uint64_t>(nc, 1))});
}

}  // namespace pcv
