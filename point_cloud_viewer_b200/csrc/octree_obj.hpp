// octree_obj.hpp — the opaque handles behind the C ABI, and the scope-bound owners of the CUDA resources the ABI layer uses.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <map>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/pcv.h"
#include "disk_io.hpp"
#include "kernels_build.cuh"

#define CU(x) PCV_CUDA_CHECK(x)

struct DevBytes {  // live and peak bytes of a group of allocations (the bounded drivers report their own)
    uint64_t live = 0, peak = 0;
    void add(uint64_t n) {
        live += n;
        peak = std::max(peak, live);
    }
};

struct Pinned {  // one pinned host buffer, grown on demand
    uint8_t* p = nullptr;
    size_t cap = 0;
    Pinned() = default;
    Pinned(const Pinned&) = delete;
    Pinned& operator=(const Pinned&) = delete;
    uint8_t* get(size_t n) {
        if (n > cap) {
            if (p) cudaFreeHost(p);
            p = nullptr;
            cap = 0;
            CU(cudaMallocHost(&p, n));
            cap = n;
        }
        return p;
    }
    ~Pinned() {
        if (p) cudaFreeHost(p);
    }
};

template <int N = 4, unsigned Flags = cudaEventDefault>
struct Events {
    cudaEvent_t e[N] = {};
    Events() {
        for (auto& x : e) CU(cudaEventCreateWithFlags(&x, Flags));
    }
    Events(const Events&) = delete;
    Events& operator=(const Events&) = delete;
    ~Events() {
        for (auto& x : e)
            if (x) cudaEventDestroy(x);
    }
};

// Runs `f` when the scope is left, normally or by an exception: the exit actions that are not memory (joining threads,
// draining the stream before a pinned buffer is reused).
template <class F>
struct OnExit {
    F f;
    ~OnExit() { f(); }
};
template <class F>
OnExit(F) -> OnExit<F>;

constexpr int kPinSlots = 3;  // pinned staging chunks of the streamed inputs (pcv_ctx::ply_pin)

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
    Pinned ply_pin[kPinSlots];  // pinned staging ring of the PLY loader and the out-of-core build (ply_api.inl)
};

struct Scratch {  // stream-ordered device allocations released on scope exit, in allocation order
    pcv_ctx* c;
    std::vector<void*> ptrs;
    DevBytes* bytes = nullptr;  // optional: counts what this scratch holds
    uint64_t held = 0;
    explicit Scratch(pcv_ctx* ctx, DevBytes* b = nullptr) : c(ctx), bytes(b) {}
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    template <class T>
    T* alloc(size_t n) {
        T* p = (T*)c->be->dmalloc(n * sizeof(T));
        ptrs.push_back(p);
        if (bytes) bytes->add(n * sizeof(T)), held += n * sizeof(T);
        return p;
    }
    template <class T>
    T* upload(const T* h, size_t n) {
        T* p = alloc<T>(n ? n : 1);
        if (n) c->be->h2d(p, h, n * sizeof(T));
        return p;
    }
    // frees everything allocated so far, now
    void reset() {
        for (void* p : ptrs) c->be->dfree(p);
        ptrs.clear();
        if (bytes) bytes->live -= held;
        held = 0;
    }
    // hands everything allocated so far over to the caller (a result handle): nothing is freed
    void release() {
        ptrs.clear();
        if (bytes) bytes->live -= held;
        held = 0;
    }
    ~Scratch() { reset(); }
};

struct DevBuf {  // one counted device allocation
    pcv_ctx* c;
    DevBytes* b;
    uint8_t* p = nullptr;
    uint64_t n = 0;
    DevBuf(pcv_ctx* ctx, DevBytes* bytes, uint64_t size) : c(ctx), b(bytes), n(size) {
        p = (uint8_t*)c->be->dmalloc(size);
        b->add(size);
    }
    ~DevBuf() {
        c->be->dfree(p);
        b->live -= n;
    }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
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

    pcv_octree() = default;
    pcv_octree(const pcv_octree&) = delete;
    pcv_octree& operator=(const pcv_octree&) = delete;
    ~pcv_octree() {  // stream-ordered frees on the context's stream; the caller has selected the context's device
        if (!ctx) return;
        for (void* p : {(void*)d_xyz, (void*)d_rgb, (void*)d_intensity, (void*)d_src, d_qnodes, (void*)d_children}) ctx->be->dfree(p);
    }
    int find(uint64_t hi, uint64_t lo) const { return pcv::find_node(nodes, hi, lo); }
};
