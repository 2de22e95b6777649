// s2_stream_plan.h — host-only planning of the streamed S2 split (s2_stream.inl; no CUDA: the CPU tests compile it with g++).
// The split holds two batches of B points at once (batch k + 1 fills while batch k is split and its output goes to the host):
//   per point  2 x input (the gathered batch: 24 B positions + 3 B colour + 4 B intensity, each when present)
//            + 2 x output (the same bytes, cell-contiguous)
//            + keys 2 x 8 + index 2 x 4 + run starts 16 (at most one cell per point) + the radix sort's scratch per point
//   fixed      the radix sort's constant scratch + kS2PlanSlack (counters, box partials, alignment)
//   source     the source's device buffers: src_chunk_bytes per point of its chunk
// B is a whole number of source chunks, below 2^32 and at most kS2MaxBatchPoints (it sizes the pinned output ring on the
// host).  When the budget cannot hold a batch of one full chunk, the chunk shrinks with the batch, down to one granule (the
// source's smallest chunk); below that the budget is too small.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <string>

namespace pcv {

constexpr uint64_t kS2PlanSlack = (uint64_t)1 << 20;
constexpr uint64_t kS2MaxBatchPoints = (uint64_t)1 << 24;  // 2 pinned output slots of <= 512 MiB each

struct S2StreamPlanIn {
    uint64_t budget = 0;          // device bytes the call may hold (0: 7/8 of `free_bytes`)
    uint64_t free_bytes = 0;      // device bytes the context can allocate now
    uint64_t n = 0;               // points of the input
    uint64_t attr_bytes = 24;     // bytes per point of one batch (input) and of one output slot: 24 + 3 (colour) + 4 (intensity)
    uint64_t sort_per_point = 0;  // radix sort scratch: bytes per point ...
    uint64_t sort_fixed = 0;      // ... plus a constant
    uint64_t chunk = 0;           // points of one full source chunk (a multiple of `granule`)
    uint64_t granule = 256;       // the source's smallest chunk
    uint64_t src_chunk_bytes = 0; // device bytes the source holds per point of its chunk
};

struct S2StreamPlan {
    uint64_t budget = 0;       // the budget used
    uint64_t batch = 0;        // B
    uint64_t chunk = 0;        // points per source chunk (B is a multiple of it)
    uint64_t per_point = 0;    // device bytes per batch point
    uint64_t fixed = 0;        // device bytes independent of B (source buffers excluded)
    uint64_t planned = 0;      // fixed + source buffers + B x per_point
    std::string error;         // non-empty: the budget cannot hold one granule
};

inline uint64_t s2_plan_per_point(const S2StreamPlanIn& in) { return 4 * in.attr_bytes + 16 + 8 + 16 + in.sort_per_point; }

inline S2StreamPlan plan_s2_stream(const S2StreamPlanIn& in) {
    S2StreamPlan p;
    p.budget = in.budget ? in.budget : in.free_bytes - in.free_bytes / 8;
    p.per_point = s2_plan_per_point(in);
    p.fixed = in.sort_fixed + kS2PlanSlack;
    const uint64_t g = std::max<uint64_t>(1, in.granule);
    const uint64_t full = std::max<uint64_t>(g, in.chunk / g * g);
    const uint64_t src = in.src_chunk_bytes;
    // the most points any batch needs: the whole input, rounded up to a granule
    const uint64_t need = std::max<uint64_t>(g, (in.n + g - 1) / g * g);
    const uint64_t cap = std::min<uint64_t>(kS2MaxBatchPoints, 0xFFFFFFFEull) / g * g;
    const uint64_t min_bytes = p.fixed + g * (p.per_point + src);
    if (p.budget < min_bytes) {
        char msg[256];
        snprintf(msg, sizeof msg, "a device budget of %llu bytes cannot hold one batch of %llu points: at least %llu bytes",
                 (unsigned long long)p.budget, (unsigned long long)g, (unsigned long long)min_bytes);
        p.error = msg;
        return p;
    }
    const uint64_t room = p.budget - p.fixed;
    uint64_t c = std::min<uint64_t>(full, need);
    uint64_t b = 0;
    if (room >= c * src + c * p.per_point) {  // whole chunks of the source's size
        b = (room - c * src) / p.per_point / c * c;
        b = std::min<uint64_t>(b, (need + c - 1) / c * c);
        b = std::max<uint64_t>(c, std::min<uint64_t>(b, cap / c * c));
    } else {  // smaller chunks: one chunk per batch
        b = room / (p.per_point + src) / g * g;
        c = b;
    }
    p.batch = b;
    p.chunk = c;
    p.planned = p.fixed + c * src + b * p.per_point;
    return p;
}

}  // namespace pcv
