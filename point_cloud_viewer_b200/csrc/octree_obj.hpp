// octree_obj.hpp — the opaque handles behind the C ABI.
#pragma once
#include <cuda_runtime.h>

#include <array>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/pcv.h"
#include "disk_io.hpp"
#include "kernels_build.cuh"

struct pcv_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    pcv_config cfg{};
    pcv::CudaBackend* be = nullptr;
    pcv_build_stats stats{};
    int sm_count = 132;
    std::mutex mu;  // build / query entry points serialise on the context's stream
    // cells of the last pcv_prefix_histogram_device call, reused by the pack over the same points (shard_api.inl)
    uint16_t* shard_cells = nullptr;
    const double* shard_cells_x = nullptr;
    uint64_t shard_cells_n = 0;
    uint32_t shard_cells_k = 0;
    double shard_cells_geom[7] = {0, 0, 0, 0, 0, 0, 0};  // resolution, bbox
    pcv_query_stats qstats{};
    pcv_xray_stats xstats{};
    uint8_t* ply_pin[3] = {nullptr, nullptr, nullptr};  // pinned staging ring of the PLY loader (ply_api.inl)
    size_t ply_pin_bytes = 0;
};

struct pcv_octree {
    pcv_ctx* ctx = nullptr;
    double resolution = 0;
    double bbox_min[3] = {0, 0, 0}, bbox_max[3] = {0, 0, 0};
    bool has_intensity = false;
    uint64_t n = 0, xyz_bytes = 0;
    std::vector<pcv_node_meta> nodes;                       // sorted by NodeId
    std::vector<uint64_t> nsub;                             // n(X) when X is subsampled into its parent
    uint8_t* d_xyz = nullptr;
    uint8_t* d_rgb = nullptr;
    float* d_intensity = nullptr;
    uint32_t* d_src = nullptr;
    // query-side device tables, built lazily (query.cuh)
    void* d_qnodes = nullptr;
    int32_t* d_children = nullptr;     // [nodes][8] index of the child in the node table, -1 if absent
    std::vector<int32_t> children_of;  // 8 per node, -1 if absent
    bool tables_ready = false;

    int find(uint64_t hi, uint64_t lo) const { return pcv::find_node(nodes, hi, lo); }
};
