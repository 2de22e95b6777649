// The query_batch_points overloads of pcv::S2CellsDir and pcv::OctreeDir (include/pcv.hpp) run once from C++, over an S2
// directory and an octree directory of the same points: the size query, then the device arrays filled, every segment equal to
// what for_each_batch streams for its location or cell union, in order and in every field.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <algorithm>
#include <array>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>

#include "../../include/pcv.hpp"

#define CHECK(c)                                                                   \
    do {                                                                           \
        if (!(c)) {                                                                \
            fprintf(stderr, "%s:%d: check failed: %s\n", __FILE__, __LINE__, #c); \
            exit(1);                                                               \
        }                                                                          \
    } while (0)

template <class T>
static std::vector<T> host(const T* d, size_t n) {
    std::vector<T> h(n);
    if (n) CHECK(cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost) == cudaSuccess);
    return h;
}

template <class Q>
static void check_segments(const std::vector<Q>& qs, const std::vector<uint64_t>& off, const double* dx, const uint8_t* dc, const float* di,
                           const uint64_t* ds, size_t total, const std::function<std::vector<pcv::PointsBatch>(const Q&)>& stream) {
    const std::vector<double> x = host(dx, 3 * total);
    const std::vector<uint8_t> c = host(dc, 3 * total);
    const std::vector<float> in = host(di, total);
    const std::vector<uint64_t> s = host(ds, total);
    for (size_t i = 0; i < qs.size(); ++i) {
        uint64_t j = off[i];
        for (const pcv::PointsBatch& b : stream(qs[i]))
            for (size_t k = 0; k < b.position.size(); ++k, ++j) {
                CHECK(j < off[i + 1]);
                for (int a = 0; a < 3; ++a) CHECK(std::memcmp(&x[3 * j + a], &b.position[k][a], 8) == 0 && c[3 * j + a] == b.color[k][a]);
                CHECK(in[j] == b.intensity[k] && s[j] == b.source_index[k]);
            }
        CHECK(j == off[i + 1]);
    }
}

// The batch through a handle's overload into the device arrays, each segment against the handle's stream.
template <class H, class Q>
static void run_batch(const H& h, const std::vector<Q>& qs, const std::vector<pcv::ClosedInterval>& filt, uint64_t total, double* dx, uint8_t* dc,
                      float* di, uint64_t* ds, const std::function<std::vector<pcv::PointsBatch>(const Q&)>& stream) {
    std::vector<uint64_t> off;
    CHECK(h.query_batch_points(qs, filt, off, dx, dc, di, ds, total) == total && off.size() == qs.size() + 1);
    const pcv_dir_query_stats st = h.last_stats();
    CHECK(st.returned_points == total && st.peak_device_bytes <= st.max_device_bytes);
    check_segments<Q>(qs, off, dx, dc, di, ds, total, stream);
}

int main(int argc, char** argv) {
    const std::string dir = argc > 1 ? argv[1] : "/tmp/pcv_cpp_dir_batch_points";
    pcv::Context ctx(0);
    const size_t n = 200000;  // a 2 km x 2 km patch of the earth's surface, as tests/cpp/test_s2_dir.cpp
    std::vector<double> x(n), y(n), z(n);
    std::vector<uint8_t> rgb(3 * n);
    std::vector<float> inten(n);
    for (size_t i = 0; i < n; ++i) {
        const double lat = 0.8 + 3e-4 * (double)((i * 7919) % 1000) / 1000.0, lng = 0.15 + 3e-4 * (double)((i * 104729) % 997) / 997.0;
        const double r = 6371000.0 + (double)(i % 13);
        x[i] = r * std::cos(lat) * std::cos(lng), y[i] = r * std::cos(lat) * std::sin(lng), z[i] = r * std::sin(lat);
        rgb[3 * i] = (uint8_t)i, rgb[3 * i + 1] = (uint8_t)(i >> 8), rgb[3 * i + 2] = (uint8_t)(i >> 16);
        inten[i] = (float)(i % 100);
    }
    const pcv_points pts{x.data(), y.data(), z.data(), 1, rgb.data(), inten.data(), n};
    pcv::S2Cells::build_to_directory(ctx, pts, dir);
    pcv::S2CellsDir cells(ctx, dir, 64ull << 20);
    double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
    for (size_t i = 0; i < n; ++i) {
        const double p[3] = {x[i], y[i], z[i]};
        for (int a = 0; a < 3; ++a) lo[a] = std::fmin(lo[a], p[a]), hi[a] = std::fmax(hi[a], p[a]);
    }
    // the same points as an octree directory, with intensity
    pcv::PointsBatch batch;
    for (size_t i = 0; i < n; ++i) {
        batch.position.push_back({x[i], y[i], z[i]});
        batch.color.push_back({rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]});
        batch.intensity.push_back(inten[i]);
    }
    const std::vector<pcv::PointsBatch> input{batch};
    const std::string odir = dir + "_octree";
    pcv::build_octree(ctx, odir, 0.001, pcv::Aabb({lo[0] - 1, lo[1] - 1, lo[2] - 1}, {hi[0] + 1, hi[1] + 1, hi[2] + 1}), input.begin(), input.end(),
                      {"color", "intensity"});
    pcv::OctreeDir octree(ctx, odir, 64ull << 20);

    std::vector<pcv::PointLocation> locs;
    for (double f : {0.1, 0.3, 0.5}) {
        std::array<double, 3> a, b;
        for (int k = 0; k < 3; ++k) a[k] = lo[k] + f * (hi[k] - lo[k]), b[k] = lo[k] + (f + 0.35) * (hi[k] - lo[k]);
        locs.push_back(pcv::PointLocation::from(pcv::Aabb(a, b)));
    }
    locs.push_back(pcv::PointLocation::AllPoints());
    const std::vector<pcv::ClosedInterval> filt = {pcv::ClosedInterval{10.0, 60.0}};
    // the cell-union batch: every cell of the S2 directory as one union, and its first half
    const std::vector<pcv::CellID> all = cells.nodes_in_location(nullptr);
    const std::vector<pcv::CellUnion> unions = {all, pcv::CellUnion(all.begin(), all.begin() + all.size() / 2)};

    // size queries: the offsets against query_batch's counts (query_batch takes no filters), and every batch's total
    std::vector<uint64_t> off0, counts, tested, off;
    cells.query_batch_points(locs, {}, off0);
    cells.query_batch(locs, counts, tested);
    CHECK(off0.size() == locs.size() + 1 && off0.back() > 0);
    for (size_t i = 0; i < locs.size(); ++i) CHECK(off0[i + 1] - off0[i] == counts[i]);
    octree.query_batch_points(locs, {}, off);
    octree.query_batch(locs, counts, tested);
    for (size_t i = 0; i < locs.size(); ++i) CHECK(off[i + 1] - off[i] == counts[i]);
    const uint64_t s2_total = cells.query_batch_points(locs, filt, off);
    CHECK(s2_total > 0 && s2_total < off0.back());
    const uint64_t s2_union_total = cells.query_batch_points(unions, {}, off);
    CHECK(off[1] == n && s2_union_total > n);
    const uint64_t oct_total = octree.query_batch_points(locs, filt, off);
    const uint64_t oct_union_total = octree.query_batch_points(unions, {}, off);
    CHECK(oct_total > 0 && off[1] > 0 && oct_union_total > off[1]);  // the octree's positions are quantised: edges may differ from the S2 cells'
    // device arrays for the largest batch
    const uint64_t room = std::max({s2_total, s2_union_total, oct_total, oct_union_total});
    double* dx;
    uint8_t* dc;
    float* di;
    uint64_t* ds;
    CHECK(cudaMalloc(&dx, 24 * room) == cudaSuccess && cudaMalloc(&dc, 3 * room) == cudaSuccess && cudaMalloc(&di, 4 * room) == cudaSuccess &&
          cudaMalloc(&ds, 8 * room) == cudaSuccess);

    auto box_stream = [&](auto& h) {
        return [&](const pcv::PointLocation& l) {
            pcv::PointQuery q;
            q.location = l;
            q.filter_intervals = filt;
            std::vector<pcv::PointsBatch> v;
            CHECK(h.for_each_batch(q, 1000, [&](pcv::PointsBatch&& p) { v.push_back(std::move(p)); return true; }));
            return v;
        };
    };
    auto union_stream = [&](auto& h) {
        return [&](const pcv::CellUnion& u) {
            std::vector<pcv::PointsBatch> v;
            CHECK(h.for_each_batch(u, {}, 1000, [&](pcv::PointsBatch&& p) { v.push_back(std::move(p)); return true; }));
            return v;
        };
    };
    run_batch<pcv::S2CellsDir, pcv::PointLocation>(cells, locs, filt, s2_total, dx, dc, di, ds, box_stream(cells));
    run_batch<pcv::S2CellsDir, pcv::CellUnion>(cells, unions, {}, s2_union_total, dx, dc, di, ds, union_stream(cells));
    run_batch<pcv::OctreeDir, pcv::PointLocation>(octree, locs, filt, oct_total, dx, dc, di, ds, box_stream(octree));
    run_batch<pcv::OctreeDir, pcv::CellUnion>(octree, unions, {}, oct_union_total, dx, dc, di, ds, union_stream(octree));
    cudaFree(dx), cudaFree(dc), cudaFree(di), cudaFree(ds);
    printf("OK\n");
    return 0;
}
