// s2_dir_xray_plan.h — host-only planning of the X-ray quadtree built straight from S2 directories (s2_dir_xray.inl; no
// CUDA: the CPU tests compile it with g++).
//   s2_scan_chunks:     the scan pass's chunks: runs of cell pieces, a cell larger than a chunk cut across chunks
//   s2_window_bytes:    what one window of cells takes on the device
//   s2_dir_block_depth: the block depth from the budget, the images and the largest window of the occupied blocks
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "xray_dir_plan.h"
#include "xray_plan.h"

namespace pcv {

// Points [first, first + count) of cell `cell` of the directory-wide table.
struct S2Piece {
    uint32_t cell;
    uint32_t count;
    uint64_t first;
};

// The cells' points in table order, cut into chunks of at most `chunk_points` points and `max_pieces` pieces: a cell goes into
// the current chunk as far as it fits and its remainder starts the next one; cells without points are skipped.  Returns the
// chunk starts into `pieces` plus an end sentinel (just {0} when there is no point).  chunk_points and max_pieces >= 1.
inline std::vector<size_t> s2_scan_chunks(const std::vector<uint64_t>& counts, uint64_t chunk_points, uint64_t max_pieces, std::vector<S2Piece>& pieces) {
    pieces.clear();
    std::vector<size_t> starts{0};
    uint64_t used = 0;  // points in the current chunk
    for (size_t k = 0; k < counts.size(); ++k)
        for (uint64_t first = 0; first < counts[k];) {
            if (used == chunk_points || pieces.size() - starts.back() == max_pieces) starts.push_back(pieces.size()), used = 0;
            const uint64_t take = std::min(counts[k] - first, chunk_points - used);
            pieces.push_back(S2Piece{(uint32_t)k, (uint32_t)take, first});
            first += take;
            used += take;
        }
    if (pieces.size() > starts.back()) starts.push_back(pieces.size());
    return starts;
}

// Device bytes per window cell besides its points: the query node (64 B), the id (8 B) and the point box (48 B).
constexpr uint64_t kS2WindowCellBytes = 64 + 8 + 48;

// What one window of `points` points in `cells` cells (`tiles` work tiles) takes on the device: positions (24 B per point),
// colours only for PCV_XRAY_COLORED (3 B), intensities only for PCV_XRAY_INTENSITY or filters (4 B), the cell tables, and what
// the S2 leaf producer holds for the window's cells (s2_xray_fixed_bytes; the filter intervals are the run's).
inline uint64_t s2_window_bytes(uint64_t points, uint64_t cells, uint64_t tiles, int strategy, uint32_t nfilt) {
    return 24 * points + (strategy == PCV_XRAY_COLORED ? 3 * points : 0) + (strategy == PCV_XRAY_INTENSITY || nfilt ? 4 * points : 0) +
           kS2WindowCellBytes * cells + s2_xray_fixed_bytes(cells, tiles, 0);
}

// The block depth of the S2 directory driver: the largest g <= g_max at which s2_xray_plan fits the block images and the keys
// (or an attribute slice) besides `fixed` and the largest window of the occupied blocks at depth g.  -1: not even g = 0 fits.
inline int s2_dir_block_depth(uint64_t budget, uint64_t fixed, int depth, int g_max, uint64_t leaf_bytes, uint64_t tile_bytes, uint64_t slice_bytes,
                              const std::function<uint64_t(int)>& window_max) {
    return xray_dir_block_depth(g_max, window_max, [&](int g, uint64_t w) {
        return s2_xray_plan(budget, fixed + w, depth, g, leaf_bytes, tile_bytes, slice_bytes).g == g;
    });
}

}  // namespace pcv
