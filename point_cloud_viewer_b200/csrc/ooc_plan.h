// ooc_plan.h — host-only planning of the prefix-sharded builds (no CUDA: the CPU tests compile it with g++).
//   level_counts_of / usable_prefix_levels: distributed.py level_counts / usable_prefix_levels, restated (sharded_build.inl)
//   plan_ooc_groups: the groups of the out-of-core build (ooc_build.inl) - consecutive level-k cells, each group one in-core build
#pragma once
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

namespace pcv {

// counts of the 8^level cells of `level` from the 8^k counts of level k >= level
inline std::vector<uint64_t> level_counts_of(const std::vector<uint64_t>& ck, int k, int level) {
    std::vector<uint64_t> out((size_t)1 << (3 * level), 0);
    const int shift = 3 * (k - level);
    for (size_t i = 0; i < ck.size(); ++i) out[i >> shift] += ck[i];
    return out;
}

// Largest k' <= k such that every non-empty node of levels 1..k'-1 is split by the reference's rule (count > max_points and
// edge > resolution, generation.rs:128-150), i.e. no leaf sits above the shard level.
inline int usable_prefix_levels(const std::vector<uint64_t>& ck, int k, double root_edge, double resolution, uint64_t max_points) {
    int ok = 1;
    double edge = root_edge;
    for (int j = 1; j < k; ++j) {
        edge = edge / 2.0;
        const std::vector<uint64_t> c = level_counts_of(ck, k, j);
        bool any = false, all = true;
        for (uint64_t v : c)
            if (v) {
                any = true;
                all = all && v > max_points;
            }
        if (any && all && edge > resolution)
            ok = j + 1;
        else
            break;
    }
    return ok;
}

// NodeId Display of level-k cell `cell`: 'r' + k octal digits
inline std::string cell_name(uint64_t cell, int k) {
    std::string s(1, 'r');
    for (int i = k - 1; i >= 0; --i) s.push_back((char)('0' + (int)((cell >> (3 * i)) & 7)));
    return s;
}

struct OocPlan {
    int k = 1;                             // prefix level the groups are made of
    std::vector<uint64_t> counts;          // 8^k cell counts at level k
    std::vector<uint64_t> prefix_counts;   // levels 1..k concatenated (ShardSpec layout)
    std::vector<uint32_t> group_first;     // per group: first cell; group g holds cells [group_first[g], group_first[g + 1])
    std::vector<uint64_t> group_points;    // per group: points
    std::string error;                     // non-empty: a single cell exceeds the budget (PCV_ERR_UNSUPPORTED)
};

// counts_K: the 8^K level-K cell counts of the whole cloud.  k = usable_prefix_levels(.., K, ..); groups are runs of consecutive
// non-empty level-k cells in cell-index order, each filled greedily up to `budget` points.  Empty cells belong to no group.
inline OocPlan plan_ooc_groups(const std::vector<uint64_t>& counts_K, int K, double root_edge, double resolution, uint64_t max_points, uint64_t budget) {
    OocPlan p;
    p.k = usable_prefix_levels(counts_K, K, root_edge, resolution, max_points);
    p.counts = level_counts_of(counts_K, K, p.k);
    for (int j = 1; j <= p.k; ++j) {
        const std::vector<uint64_t> lc = level_counts_of(counts_K, K, j);
        p.prefix_counts.insert(p.prefix_counts.end(), lc.begin(), lc.end());
    }
    for (size_t cell = 0; cell < p.counts.size(); ++cell) {
        const uint64_t v = p.counts[cell];
        if (v == 0) continue;
        if (v > budget) {
            char buf[256];
            snprintf(buf, sizeof buf, "octree cell %s holds %llu points, more than the %llu points one in-core build may take", cell_name(cell, p.k).c_str(),
                     (unsigned long long)v, (unsigned long long)budget);
            p.error = buf;
            if (p.k < K) p.error += " (a node above it is a leaf, so the cloud cannot be cut below that level)";
            p.group_first.clear();
            p.group_points.clear();
            return p;
        }
        if (p.group_points.empty() || p.group_points.back() + v > budget) {
            p.group_first.push_back((uint32_t)cell);
            p.group_points.push_back(0);
        }
        p.group_points.back() += v;
    }
    p.group_first.push_back((uint32_t)p.counts.size());  // end sentinel
    return p;
}

}  // namespace pcv
