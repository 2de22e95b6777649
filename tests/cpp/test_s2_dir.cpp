// pcv::S2CellsDir against pcv::S2Cells::from_directory over the same S2 directory, through include/pcv.hpp: the cell lists of
// AllPoints and an Aabb, the streamed points of the Aabb, and the batched counts, equal; no call reads more than it selects.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>

#include "../../include/pcv.hpp"

#define CHECK(c)                                                          \
    do {                                                                  \
        if (!(c)) {                                                       \
            fprintf(stderr, "%s:%d: check failed: %s\n", __FILE__, __LINE__, #c); \
            exit(1);                                                      \
        }                                                                 \
    } while (0)

int main(int argc, char** argv) {
    const std::string dir = argc > 1 ? argv[1] : "/tmp/pcv_cpp_s2_dir";
    pcv::Context ctx(0);
    // a 2 km x 2 km patch of the earth's surface, 200 000 points
    const size_t n = 200000;
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
    pcv::S2Cells loaded = pcv::S2Cells::from_directory(ctx, dir);
    pcv::S2CellsDir cells(ctx, dir, 64ull << 20);

    CHECK(cells.nodes_in_location(nullptr) == loaded.nodes_in_location(nullptr));
    CHECK(cells.last_stats().bytes_read == 0);
    double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
    for (size_t i = 0; i < n; ++i) {
        const double p[3] = {x[i], y[i], z[i]};
        for (int a = 0; a < 3; ++a) lo[a] = std::fmin(lo[a], p[a]), hi[a] = std::fmax(hi[a], p[a]);
    }
    std::array<double, 3> a, b;
    for (int k = 0; k < 3; ++k) a[k] = lo[k] + 0.3 * (hi[k] - lo[k]), b[k] = lo[k] + 0.6 * (hi[k] - lo[k]);
    const pcv::PointLocation box = pcv::PointLocation::from(pcv::Aabb(a, b));
    CHECK(cells.nodes_in_location(box) == loaded.nodes_in_location(box));
    CHECK(cells.last_stats().bytes_read == 0);  // the box scan ran once, in the counting call; the listing call reads nothing

    pcv::PointQuery q;
    q.location = box;
    q.filter_intervals = {pcv::ClosedInterval{10.0, 60.0}};
    std::vector<pcv::PointsBatch> got, want;
    CHECK(cells.for_each_batch(q, 1000, [&](pcv::PointsBatch&& p) { got.push_back(std::move(p)); return true; }));
    CHECK(loaded.for_each_batch(q, 1000, [&](pcv::PointsBatch&& p) { want.push_back(std::move(p)); return true; }));
    CHECK(got.size() == want.size() && !got.empty());
    for (size_t k = 0; k < got.size(); ++k)
        CHECK(got[k].position == want[k].position && got[k].color == want[k].color && got[k].intensity == want[k].intensity &&
              got[k].source_index == want[k].source_index);
    const pcv_dir_query_stats st = cells.last_stats();
    CHECK(st.peak_device_bytes <= st.max_device_bytes && st.tested_points > 0);

    std::vector<uint64_t> c0, t0, c1, t1;
    cells.query_batch({box, pcv::PointLocation::AllPoints()}, c0, t0);
    loaded.query_batch({box, pcv::PointLocation::AllPoints()}, c1, t1);
    CHECK(c0 == c1 && t0 == t1 && c0[1] == n);
    printf("OK\n");
    return 0;
}
