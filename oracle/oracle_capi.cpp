// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_core.hpp header).
// C interface for tests/ (ctypes), __graft_entry__.smoke() and bench.py's CPU-baseline legs.
#include <thread>
#include <chrono>

#include "oracle_build.hpp"
#include "oracle_disk.hpp"
#include "oracle_ply.hpp"
#include "oracle_query.hpp"
#include "oracle_xray_pyramid.hpp"
#include "oracle_s2.hpp"
#include "../include/pcv_synth.h"  // input-data generators shared with the benchmark (no algorithm code)

using namespace orc;

extern "C" {

// Shared by the oracle and (same layout) the product's pcv_location, so tests build one struct.
struct orc_location {
    int32_t kind;  // 0 all, 1 aabb, 2 frustum, 3 obb
    int32_t pad;
    double aabb_min[3], aabb_max[3];
    double clip_from_query[16], query_from_clip[16];  // column-major (nalgebra)
    double query_from_obb[7], obb_from_query[7];      // tx,ty,tz, qi,qj,qk,qw
    double half_extent[3];
};

static Iso3 iso_from7(const double* v) {
    Iso3 r;
    r.t = {v[0], v[1], v[2]};
    r.q[0] = v[3];
    r.q[1] = v[4];
    r.q[2] = v[5];
    r.q[3] = v[6];
    return r;
}

static Location to_loc(const orc_location* l) {
    Location r;
    r.kind = l->kind;
    r.aabb = Aabb::make({l->aabb_min[0], l->aabb_min[1], l->aabb_min[2]}, {l->aabb_max[0], l->aabb_max[1], l->aabb_max[2]});
    std::memcpy(r.frustum.clip_from_query.m, l->clip_from_query, sizeof(double) * 16);
    std::memcpy(r.frustum.query_from_clip.m, l->query_from_clip, sizeof(double) * 16);
    r.obb.query_from_obb = iso_from7(l->query_from_obb);
    r.obb.obb_from_query = iso_from7(l->obb_from_query);
    r.obb.half_extent = {l->half_extent[0], l->half_extent[1], l->half_extent[2]};
    return r;
}

struct Handle {
    Octree oct;
    std::vector<NodeId> order;  // sorted meta ids
    double build_seconds = 0;
};

void orc_bbox(uint64_t n, const double* x, const double* y, const double* z, uint64_t stride, double* out6) {
    Aabb b = find_bounding_box((size_t)n, x, y, z, (size_t)stride);
    out6[0] = b.mins.x;
    out6[1] = b.mins.y;
    out6[2] = b.mins.z;
    out6[3] = b.maxs.x;
    out6[4] = b.maxs.y;
    out6[5] = b.maxs.z;
}

void* orc_build(uint64_t n, const double* x, const double* y, const double* z, uint64_t stride, const uint8_t* rgb,
                const float* intensity, double resolution, const double* bbox_min, const double* bbox_max,
                int64_t max_points_per_node, int num_threads) {
    Builder b;
    b.num_threads = num_threads > 0 ? num_threads : (int)std::max(1u, std::thread::hardware_concurrency());
    b.P.resolution = resolution;
    b.P.bbox = Aabb::make({bbox_min[0], bbox_min[1], bbox_min[2]}, {bbox_max[0], bbox_max[1], bbox_max[2]});
    b.P.with_intensity = intensity != nullptr;
    if (max_points_per_node > 0) b.P.max_points_per_node = max_points_per_node;
    auto t0 = std::chrono::steady_clock::now();
    Handle* h = new Handle();
    h->oct = b.build((size_t)n, x, y, z, (size_t)stride, rgb, intensity);
    h->build_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (auto& kv : h->oct.nodes) h->order.push_back(kv.first);
    return h;
}
double orc_build_seconds(void* hp) { return ((Handle*)hp)->build_seconds; }

// The "faithful" variant of build_octree: node contents round-trip through files of `dir` between the steps, as in the
// reference (generation.rs:39-126,195-253); the directory ends up holding the finished octree (node files + meta.pb,
// generation.rs:399-402).  Returns the build time in seconds (< 0 on failure).  Same arithmetic and results as orc_build.
double orc_build_faithful(uint64_t n, const double* x, const double* y, const double* z, uint64_t stride, const uint8_t* rgb, const float* intensity,
                          double resolution, const double* bbox_min, const double* bbox_max, int64_t max_points_per_node, int num_threads, const char* dir,
                          uint64_t* num_nodes_out) {
    try {
        Builder b;
        b.num_threads = num_threads > 0 ? num_threads : (int)std::max(1u, std::thread::hardware_concurrency());
        b.P.resolution = resolution;
        b.P.bbox = Aabb::make({bbox_min[0], bbox_min[1], bbox_min[2]}, {bbox_max[0], bbox_max[1], bbox_max[2]});
        b.P.with_intensity = intensity != nullptr;
        if (max_points_per_node > 0) b.P.max_points_per_node = max_points_per_node;
        b.disk_dir = dir;
        auto t0 = std::chrono::steady_clock::now();
        Octree oct = b.build((size_t)n, x, y, z, (size_t)stride, rgb, intensity);
        const std::string m = meta_pb(oct);
        if (!write_file(std::string(dir) + "/meta.pb", m.data(), m.size())) return -1.0;
        if (num_nodes_out) *num_nodes_out = oct.nodes.size();
        return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    } catch (const std::exception&) {
        return -1.0;
    }
}

// Synthetic inputs (include/pcv_synth.h), generated on `num_threads` host threads.
void orc_synth_points(int kind, uint64_t seed, uint64_t first, uint64_t n, double* x, double* y, double* z, uint8_t* rgb, int num_threads) {
    const int nt = num_threads > 0 ? num_threads : (int)std::max(1u, std::thread::hardware_concurrency());
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t)
        th.emplace_back([=] {
            const uint64_t lo = n * (uint64_t)t / (uint64_t)nt, hi = n * (uint64_t)(t + 1) / (uint64_t)nt;
            for (uint64_t i = lo; i < hi; ++i) {
                double p[3];
                uint8_t c[3];
                pcv::synth_point(kind, seed, first + i, p, c);
                x[i] = p[0], y[i] = p[1], z[i] = p[2];
                rgb[3 * i] = c[0], rgb[3 * i + 1] = c[1], rgb[3 * i + 2] = c[2];
            }
        });
    for (auto& t : th) t.join();
}
void orc_synth_bbox(int kind, double* bbox_min, double* bbox_max, double* resolution) { pcv::synth_bbox(kind, bbox_min, bbox_max, resolution); }
int orc_max_threads() { return (int)std::max(1u, std::thread::hardware_concurrency()); }

void orc_free(void* hp) { delete (Handle*)hp; }

uint64_t orc_num_nodes(void* hp) { return ((Handle*)hp)->order.size(); }

void orc_node_info(void* hp, uint64_t i, uint64_t* hi, uint64_t* lo, int64_t* num_points, int32_t* enc, double* cube4) {
    Handle* h = (Handle*)hp;
    NodeId id = h->order[i];
    const NodeMeta& m = h->oct.nodes[id];
    *hi = id.high();
    *lo = id.low();
    *num_points = m.num_points;
    *enc = (int32_t)m.enc;
    cube4[0] = m.cube.min.x;
    cube4[1] = m.cube.min.y;
    cube4[2] = m.cube.min.z;
    cube4[3] = m.cube.edge;
}

// Copies node content; any out pointer may be null. Returns number of points or -1 if unknown id.
int64_t orc_node_data(void* hp, uint64_t hi, uint64_t lo, uint8_t* xyz, uint8_t* rgb, float* intensity, uint64_t* src) {
    Handle* h = (Handle*)hp;
    NodeId id = NodeId::from_high_low(hi, lo);
    if (!h->oct.nodes.count(id)) return -1;
    auto it = h->oct.files.find(id);
    if (it == h->oct.files.end()) return 0;
    const NodeFile& f = it->second;
    if (xyz) std::memcpy(xyz, f.xyz.data(), f.xyz.size());
    if (rgb) std::memcpy(rgb, f.rgb.data(), f.rgb.size());
    if (intensity && !f.intensity.empty()) std::memcpy(intensity, f.intensity.data(), f.intensity.size() * 4);
    if (src) std::memcpy(src, f.src.data(), f.src.size() * 8);
    return f.num_points();
}

// ---- scalar codec / node-id vectors ----
uint64_t orc_encode(double value, double min, double edge, int enc) { return encode_coord(value, min, edge, (Enc)enc); }
double orc_decode(uint64_t bits, double min, double edge, int enc) { return decode_coord(bits, min, edge, (Enc)enc); }
int orc_position_encoding(double edge, double resolution) { return (int)position_encoding(Cube{{0, 0, 0}, edge}, resolution); }
void orc_find_bounding_cube(uint64_t hi, uint64_t lo, const double* root_min, double root_edge, double* out4) {
    Cube c = find_bounding_cube(NodeId::from_high_low(hi, lo), Cube{{root_min[0], root_min[1], root_min[2]}, root_edge});
    out4[0] = c.min.x;
    out4[1] = c.min.y;
    out4[2] = c.min.z;
    out4[3] = c.edge;
}
void orc_cube_bounding(const double* mn, const double* mx, double* out4) {
    Cube c = Cube::bounding(Aabb::make({mn[0], mn[1], mn[2]}, {mx[0], mx[1], mx[2]}));
    out4[0] = c.min.x;
    out4[1] = c.min.y;
    out4[2] = c.min.z;
    out4[3] = c.edge;
}
int orc_child_index(const double* cube4, const double* p) {
    return (int)child_index_of(Cube{{cube4[0], cube4[1], cube4[2]}, cube4[3]}, {p[0], p[1], p[2]});
}
void orc_node_id_from_string(const char* s, uint64_t* hi, uint64_t* lo) {
    NodeId id = NodeId::from_string(s);
    *hi = id.high();
    *lo = id.low();
}
void orc_node_id_to_string(uint64_t hi, uint64_t lo, char* out, int cap) {
    std::string s = NodeId::from_high_low(hi, lo).to_string();
    std::snprintf(out, (size_t)cap, "%s", s.c_str());
}
void orc_node_id_parent(uint64_t hi, uint64_t lo, uint64_t* phi, uint64_t* plo, int* child_index) {
    NodeId id = NodeId::from_high_low(hi, lo);
    *child_index = id.child_index();
    NodeId p = id.has_parent() ? id.parent() : id;
    *phi = p.high();
    *plo = p.low();
}
void orc_node_id_child(uint64_t hi, uint64_t lo, int k, uint64_t* chi, uint64_t* clo) {
    NodeId c = NodeId::from_high_low(hi, lo).child((unsigned)k);
    *chi = c.high();
    *clo = c.low();
}

// ---- SAT pins ----
static Intersector mk_isec(const double* corners24, const double* edges, int ne, const double* faces, int nf) {
    Intersector r;
    for (int i = 0; i < 8; ++i) r.corners[i] = {corners24[3 * i], corners24[3 * i + 1], corners24[3 * i + 2]};
    for (int i = 0; i < ne; ++i) r.edges.push_back({edges[3 * i], edges[3 * i + 1], edges[3 * i + 2]});
    for (int i = 0; i < nf; ++i) r.face_normals.push_back({faces[3 * i], faces[3 * i + 1], faces[3 * i + 2]});
    return r;
}
// Intersector::intersect (sat.rs:145-151)
int orc_intersector_intersect(const double* ca, const double* ea, int nea, const double* fa, int nfa, const double* cb,
                              const double* eb, int neb, const double* fb, int nfb) {
    Intersector a = mk_isec(ca, ea, nea, fa, nfa), b = mk_isec(cb, eb, neb, fb, nfb);
    return (int)sat(separating_axes(a, b.edges, b.face_normals), a.corners, 8, b.corners, 8);
}
static Intersector loc_intersector(const Location& l) {
    if (l.kind == LOC_FRUSTUM) return l.frustum.intersector();
    if (l.kind == LOC_OBB) return l.obb.intersector();
    return aabb_intersector_generic(l.aabb);
}
// location.intersector().intersect(&aabb.intersector())   (math/mod.rs:212-215)
int orc_location_intersect_aabb_generic(const orc_location* l, const double* mn, const double* mx) {
    Location loc = to_loc(l);
    Intersector a = loc_intersector(loc);
    Intersector b = aabb_intersector_generic(Aabb::make({mn[0], mn[1], mn[2]}, {mx[0], mx[1], mx[2]}));
    return (int)sat(separating_axes(a, b.edges, b.face_normals), a.corners, 8, b.corners, 8);
}
// location.intersector().cache_separating_axes_for_aabb(): number of axes + relation against an aabb
int orc_cached_axes(const orc_location* l, double* axes_out, int cap) {
    Location loc = to_loc(l);
    CachedAxesIntersector c = cache_separating_axes_for_aabb(loc_intersector(loc));
    for (int i = 0; i < (int)c.axes.size() && i < cap; ++i) {
        axes_out[3 * i] = c.axes[i].x;
        axes_out[3 * i + 1] = c.axes[i].y;
        axes_out[3 * i + 2] = c.axes[i].z;
    }
    return (int)c.axes.size();
}
int orc_cached_intersect_aabb(const orc_location* l, const double* mn, const double* mx) {
    Location loc = to_loc(l);
    AabbIntersector isec = make_aabb_intersector(loc);
    if (isec.all) return REL_IN;
    Vec3 c[8];
    Aabb::make({mn[0], mn[1], mn[2]}, {mx[0], mx[1], mx[2]}).corners(c);
    return (int)isec.isec.intersect(c, 8);
}
int orc_location_contains(const orc_location* l, const double* p) { return to_loc(l).contains({p[0], p[1], p[2]}) ? 1 : 0; }
// orc_location_contains of n points (xyz: n x 3, AoS) into out[n]
void orc_location_contains_n(const orc_location* l, const double* xyz, uint64_t n, uint8_t* out) {
    const Location loc = to_loc(l);
    for (uint64_t i = 0; i < n; ++i) out[i] = loc.contains({xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]}) ? 1 : 0;
}
void orc_location_corners(const orc_location* l, double* out24) {
    Intersector a = loc_intersector(to_loc(l));
    for (int i = 0; i < 8; ++i) {
        out24[3 * i] = a.corners[i].x;
        out24[3 * i + 1] = a.corners[i].y;
        out24[3 * i + 2] = a.corners[i].z;
    }
}
// contains via SAT with face normals only against a single point (point_cloud_test/tests/main.rs:104-127)
int orc_location_contains_sat(const orc_location* l, const double* p) {
    Intersector a = loc_intersector(to_loc(l));
    Vec3 pt{p[0], p[1], p[2]};
    return sat(a.face_normals, a.corners, 8, &pt, 1) == REL_IN ? 1 : 0;
}
int orc_try_inverse(const double* m16, double* out16) {
    Mat4 a, b;
    std::memcpy(a.m, m16, sizeof(a.m));
    if (!try_inverse(a, b)) return 0;
    std::memcpy(out16, b.m, sizeof(b.m));
    return 1;
}

// ---- queries ----
int64_t orc_nodes_in_location(void* hp, const orc_location* l, uint64_t* hi_lo_out, int64_t cap) {
    Handle* h = (Handle*)hp;
    std::vector<NodeId> ids = nodes_in_location(h->oct, to_loc(l));
    for (int64_t i = 0; i < (int64_t)ids.size() && i < cap; ++i) {
        hi_lo_out[2 * i] = ids[i].high();
        hi_lo_out[2 * i + 1] = ids[i].low();
    }
    return (int64_t)ids.size();
}

int64_t orc_visible_nodes(void* hp, const double* m16, uint64_t* hi_lo_out, int64_t cap) {
    Handle* h = (Handle*)hp;
    Mat4 M;
    std::memcpy(M.m, m16, sizeof(M.m));
    std::vector<NodeId> ids;
    if (!get_visible_nodes(h->oct, M, ids)) return -1;
    for (int64_t i = 0; i < (int64_t)ids.size() && i < cap; ++i) {
        hi_lo_out[2 * i] = ids[i].high();
        hi_lo_out[2 * i + 1] = ids[i].low();
    }
    return (int64_t)ids.size();
}

// All points matching the query, nodes visited in nodes_in_location order (the reference's batch order
// across nodes is unspecified; per node it is file order).  Two-call protocol: call with null outputs
// to get the count.  `filters` = nfilt * {lo,hi} closed intervals on intensity.
int64_t orc_query(void* hp, const orc_location* l, const double* filters, int nfilt, double* xyz, uint8_t* rgb, float* intensity,
                  uint64_t* src, int64_t cap, int64_t* tested_points) {
    Handle* h = (Handle*)hp;
    Location loc = to_loc(l);
    std::vector<Interval> fi;
    for (int i = 0; i < nfilt; ++i) fi.push_back({0, filters[2 * i], filters[2 * i + 1]});
    QueryOut out;
    int64_t tested = 0;
    for (NodeId id : nodes_in_location(h->oct, loc)) {
        tested += h->oct.nodes[id].num_points;
        query_node(h->oct, id, loc, fi, out);
    }
    if (tested_points) *tested_points = tested;
    int64_t n = (int64_t)out.src.size();
    if (xyz && n <= cap) {
        std::memcpy(xyz, out.xyz.data(), out.xyz.size() * 8);
        if (rgb) std::memcpy(rgb, out.rgb.data(), out.rgb.size());
        if (intensity && !out.intensity.empty()) std::memcpy(intensity, out.intensity.data(), out.intensity.size() * 4);
        if (src) std::memcpy(src, out.src.data(), out.src.size() * 8);
    }
    return n;
}

// ParallelIterator::try_for_each_batch (iterator.rs:255-333) as bench.py's CPU baseline of the query path: `num_threads`
// workers steal nodes from a shared queue (crossbeam deque in the reference), each decodes + culls its node through the same
// FilteredIterator restatement as orc_query and re-chunks into batches of `batch_size` that the consumer only counts.  Runs the
// locations one after the other (one PointQuery per call in the reference, point_cloud_client/src/lib.rs:42-70).  Returns seconds.
double orc_query_batch_timed(void* hp, const orc_location* locs, uint32_t nloc, int num_threads, uint64_t batch_size, uint64_t* tested_out,
                             uint64_t* returned_out, uint64_t* bytes_out) {
    Handle* h = (Handle*)hp;
    const int nt = std::max(1, num_threads);
    uint64_t tested = 0, returned = 0, bytes = 0;
    auto t0 = std::chrono::steady_clock::now();
    for (uint32_t li = 0; li < nloc; ++li) {
        const Location loc = to_loc(&locs[li]);
        const std::vector<NodeId> ids = nodes_in_location(h->oct, loc);
        std::atomic<size_t> next{0};
        std::atomic<uint64_t> ret{0};
        std::vector<std::thread> th;
        const int workers = (int)std::min<size_t>((size_t)nt, std::max<size_t>(1, ids.size()));
        for (int t = 0; t < workers; ++t)
            th.emplace_back([&] {
                std::vector<Interval> none;
                QueryOut buf;
                uint64_t mine = 0;
                for (;;) {
                    const size_t k = next.fetch_add(1);
                    if (k >= ids.size()) break;
                    query_node(h->oct, ids[k], loc, none, buf);
                    while (buf.src.size() >= batch_size) {  // PointStream::push_points_and_callback (iterator.rs:159-165): split_off a full batch
                        QueryOut rest;
                        rest.xyz.assign(buf.xyz.begin() + 3 * batch_size, buf.xyz.end());
                        rest.rgb.assign(buf.rgb.begin() + 3 * batch_size, buf.rgb.end());
                        rest.src.assign(buf.src.begin() + batch_size, buf.src.end());
                        mine += batch_size;
                        buf = std::move(rest);
                    }
                }
                mine += buf.src.size();
                ret += mine;
            });
        for (auto& t : th) t.join();
        for (NodeId id : ids) {
            const NodeMeta& m = h->oct.nodes[id];
            tested += (uint64_t)m.num_points;
            bytes += (uint64_t)m.num_points * (3ull * (uint64_t)bytes_per_coordinate(m.enc) + 3ull);
        }
        returned += ret.load();
    }
    if (tested_out) *tested_out = tested;
    if (returned_out) *returned_out = returned;
    if (bytes_out) *bytes_out = bytes + 27ull * returned;
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// reshuffle (sdl_viewer/src/node_drawer.rs:34-43): new_data = concat(old_data[i * bpv .. (i + 1) * bpv] for i in new_order).
int orc_reshuffle(const uint64_t* new_order, uint64_t n, const uint8_t* old_data, uint64_t old_len, uint64_t bytes_per_vertex, uint8_t* new_data) {
    if (n * bytes_per_vertex != old_len) return -1;  // assert_eq!(new_order.len() * bytes_per_vertex, old_data.len())
    uint64_t o = 0;
    for (uint64_t k = 0; k < n; ++k) {
        const uint64_t i = new_order[k] * bytes_per_vertex;
        if (i + bytes_per_vertex > old_len) return -2;
        std::memcpy(new_data + o, old_data + i, bytes_per_vertex);
        o += bytes_per_vertex;
    }
    return o == old_len ? 0 : -3;
}

int orc_xray_tile(void* hp, const double* bbox_min, const double* bbox_max, uint32_t w, uint32_t hgt, const double* query_from_global7,
                  uint8_t* rgba_out, uint32_t* zbits_out, uint8_t* zover_out) {
    Handle* h = (Handle*)hp;
    Aabb bb = Aabb::make({bbox_min[0], bbox_min[1], bbox_min[2]}, {bbox_max[0], bbox_max[1], bbox_max[2]});
    Iso3 q{};
    if (query_from_global7) q = iso_from7(query_from_global7);
    std::vector<uint8_t> rgba, zover;
    std::vector<uint32_t> zb;
    bool any = xray_tile(h->oct, bb, w, hgt, query_from_global7 != nullptr, q, rgba, &zb, &zover);
    std::memcpy(rgba_out, rgba.data(), rgba.size());
    if (zbits_out && any) std::memcpy(zbits_out, zb.data(), zb.size() * 4);
    if (zover_out && any) std::memcpy(zover_out, zover.data(), zover.size());
    return any ? 1 : 0;
}

int orc_xray_tile_attr(void* hp, const double* bbox_min, const double* bbox_max, uint32_t w, uint32_t hgt, const double* query_from_global7, int mode,
                       float p0, float p1, int colormap, uint8_t* rgba_out) {
    Handle* h = (Handle*)hp;
    Aabb bb = Aabb::make({bbox_min[0], bbox_min[1], bbox_min[2]}, {bbox_max[0], bbox_max[1], bbox_max[2]});
    Iso3 q{};
    if (query_from_global7) q = iso_from7(query_from_global7);
    std::vector<uint8_t> rgba;
    bool any = xray_tile_attr(h->oct, bb, w, hgt, query_from_global7 != nullptr, q, mode, p0, p1, colormap, rgba);
    std::memcpy(rgba_out, rgba.data(), rgba.size());
    return any ? 1 : 0;
}

// ---- the rest of the X-ray pipeline (oracle_xray_pyramid.hpp) ----
int orc_xray_tile_attr_binned(void* hp, const double* bbox_min, const double* bbox_max, uint32_t w, uint32_t hgt, const double* query_from_global7,
                              int mode, float p0, float p1, double bin_size, uint8_t* rgba_out) {
    Handle* h = (Handle*)hp;
    Aabb bb = Aabb::make({bbox_min[0], bbox_min[1], bbox_min[2]}, {bbox_max[0], bbox_max[1], bbox_max[2]});
    Iso3 q{};
    if (query_from_global7) q = iso_from7(query_from_global7);
    std::vector<uint8_t> rgba;
    bool any = xray_tile_attr_binned(h->oct, bb, w, hgt, query_from_global7 != nullptr, q, mode, p0, p1, bin_size, rgba);
    std::memcpy(rgba_out, rgba.data(), rgba.size());
    return any ? 1 : 0;
}
void orc_resize_lanczos3(const uint8_t* src, uint32_t w, uint32_t hgt, uint32_t nw, uint32_t nh, uint8_t* out) {
    Image im;
    im.w = w;
    im.h = hgt;
    im.px.assign(src, src + (size_t)w * hgt * 4);
    const Image r = resize_lanczos3(im, nw, nh);
    std::memcpy(out, r.px.data(), r.px.size());
}
// build_node without the files: build_parent + resize to tile_px (children[i] may be null)
void orc_build_parent_tile(const uint8_t* const children[4], uint32_t child_px, const uint8_t* bg4, uint32_t tile_px, uint8_t* out, uint8_t* mosaic_out) {
    Image ch[4];
    const Image* pc[4];
    for (int k = 0; k < 4; ++k) {
        pc[k] = nullptr;
        if (children[k]) {
            ch[k].w = ch[k].h = child_px;
            ch[k].px.assign(children[k], children[k] + (size_t)child_px * child_px * 4);
            pc[k] = &ch[k];
        }
    }
    const Image large = build_parent(pc, bg4);
    if (mosaic_out) std::memcpy(mosaic_out, large.px.data(), large.px.size());
    const Image r = resize_lanczos3(large, tile_px, tile_px);
    std::memcpy(out, r.px.data(), r.px.size());
}
void orc_assign_background(uint8_t* rgba, uint64_t npix, const uint8_t* bg4) {
    Image im;
    im.w = (uint32_t)npix;
    im.h = 1;
    im.px.assign(rgba, rgba + npix * 4);
    assign_background(im, bg4);
    std::memcpy(rgba, im.px.data(), npix * 4);
}
struct orc_xray_quadtree_params {
    int32_t strategy;
    float p0, p1;
    int32_t colormap;
    double bin_size;
    int32_t has_query_from_global;
    double query_from_global[7];
    uint8_t background[4];
    uint32_t tile_size_px;
    double pixel_size_m;
    uint8_t root_level;
    uint64_t root_index;
};
void* orc_xray_quadtree_build(void* hp, const orc_xray_quadtree_params* p) {
    Handle* h = (Handle*)hp;
    XrayQuadtreeParams pr;
    pr.strategy = p->strategy;
    pr.p0 = p->p0;
    pr.p1 = p->p1;
    pr.colormap = p->colormap;
    pr.bin_size = p->bin_size;
    pr.has_q = p->has_query_from_global != 0;
    if (pr.has_q) pr.query_from_global = iso_from7(p->query_from_global);
    std::memcpy(pr.background, p->background, 4);
    pr.tile_size_px = p->tile_size_px;
    pr.pixel_size_m = p->pixel_size_m;
    pr.root = QuadId{p->root_level, p->root_index};
    XrayQuadtree* q = new XrayQuadtree();
    if (!build_xray_quadtree(h->oct, pr, *q)) {
        delete q;
        return nullptr;
    }
    return q;
}
void orc_xray_quadtree_info(void* qp, double* rect3, int* deepest, uint64_t* ntiles) {
    XrayQuadtree* q = (XrayQuadtree*)qp;
    rect3[0] = q->bounding_rect.min_x, rect3[1] = q->bounding_rect.min_y, rect3[2] = q->bounding_rect.edge;
    *deepest = q->deepest_level;
    *ntiles = q->tiles.size();
}
void orc_xray_quadtree_ids(void* qp, uint8_t* levels, uint64_t* indices) {
    size_t k = 0;
    for (auto& kv : ((XrayQuadtree*)qp)->tiles) levels[k] = kv.first.level, indices[k] = kv.first.index, ++k;
}
int orc_xray_quadtree_tile(void* qp, uint8_t level, uint64_t index, uint8_t* rgba_out) {
    XrayQuadtree* q = (XrayQuadtree*)qp;
    auto it = q->tiles.find(QuadId{level, index});
    if (it == q->tiles.end()) return -1;
    std::memcpy(rgba_out, it->second.px.data(), it->second.px.size());
    return 0;
}
void orc_xray_quadtree_free(void* qp) { delete (XrayQuadtree*)qp; }

// ---- S2 (oracle_s2.hpp) ----
void orc_s2_cell_ids(uint64_t n, const double* x, const double* y, const double* z, uint64_t stride, int level, uint64_t* out) {
    for (uint64_t k = 0; k < n; ++k) out[k] = s2::parent(s2::cell_id_from_point(x[k * stride], y[k * stride], z[k * stride]), level);
}
void orc_s2_face_ij(uint64_t id, int* f, int* i, int* j) { s2::face_ij(id, *f, *i, *j); }
void orc_s2_centre(uint64_t id, double* out3) {
    const s2::V3 c = s2::cell_centre_raw(id);
    out3[0] = c.x, out3[1] = c.y, out3[2] = c.z;
}
uint64_t orc_s2_from_face_ij(int f, int i, int j) { return s2::from_face_ij(f, i, j); }
uint64_t orc_s2_parent(uint64_t id, int level) { return s2::parent(id, level); }
uint64_t orc_s2_next(uint64_t id) { return s2::next(id); }
int orc_s2_level(uint64_t id) { return s2::level_of(id); }
void orc_s2_token(uint64_t id, char* buf, int cap) { snprintf(buf, cap, "%s", s2::to_token(id).c_str()); }
uint64_t orc_s2_normalize(uint64_t* ids, uint64_t n) {
    std::vector<uint64_t> v(ids, ids + n);
    s2::normalize(v);
    std::copy(v.begin(), v.end(), ids);
    return v.size();
}
void orc_s2_union_test(const uint64_t* cu, uint64_t ncu, const uint64_t* ids, uint64_t m, uint8_t* contains_out, uint8_t* intersects_out) {
    const std::vector<uint64_t> v(cu, cu + ncu);
    for (uint64_t k = 0; k < m; ++k) {
        if (contains_out) contains_out[k] = s2::union_contains(v, ids[k]) ? 1 : 0;
        if (intersects_out) intersects_out[k] = s2::union_intersects(v, ids[k]) ? 1 : 0;
    }
}
void* orc_s2_split(uint64_t n, const double* x, const double* y, const double* z, uint64_t stride, int level) {
    return new s2::SplitResult(s2::split(x, y, z, stride, n, level));
}
void orc_s2_split_info(void* hp, int* ok, uint64_t* bad_index, double* bbox6, uint64_t* ncells) {
    auto* r = (s2::SplitResult*)hp;
    *ok = r->ok ? 1 : 0;
    *bad_index = r->bad_index;
    for (int a = 0; a < 3; ++a) bbox6[a] = r->bmin[a], bbox6[3 + a] = r->bmax[a];
    *ncells = r->cells.size();
}
void orc_s2_split_cells(void* hp, uint64_t* ids, uint64_t* counts, uint64_t* order) {
    auto* r = (s2::SplitResult*)hp;
    size_t c = 0, o = 0;
    for (auto& kv : r->cells) {
        ids[c] = kv.first;
        counts[c] = kv.second.size();
        ++c;
        for (uint64_t i : kv.second) order[o++] = i;
    }
}
void orc_s2_split_free(void* hp) { delete (s2::SplitResult*)hp; }

// ---- disk ----
int orc_write_dir(void* hp, const char* dir) { return write_dir(((Handle*)hp)->oct, dir) ? 0 : -1; }
void* orc_load_dir(const char* dir) {
    Handle* h = new Handle();
    if (!load_dir(dir, h->oct)) {
        delete h;
        return nullptr;
    }
    for (auto& kv : h->oct.nodes) h->order.push_back(kv.first);
    return h;
}
void orc_octree_meta(void* hp, double* resolution, double* bbox6, int* with_intensity) {
    Handle* h = (Handle*)hp;
    *resolution = h->oct.resolution;
    bbox6[0] = h->oct.bbox.mins.x;
    bbox6[1] = h->oct.bbox.mins.y;
    bbox6[2] = h->oct.bbox.mins.z;
    bbox6[3] = h->oct.bbox.maxs.x;
    bbox6[4] = h->oct.bbox.maxs.y;
    bbox6[5] = h->oct.bbox.maxs.z;
    *with_intensity = h->oct.with_intensity ? 1 : 0;
}

// ---- /nodes_data reply (octree_web_viewer/src/backend.rs:66-75 pad, :92-165 get_nodes_data) ----
// Literal restatement: for each requested id, get_node_data (octree/mod.rs:285-307: NodeNotFound when the node has no
// files, i.e. unknown id or zero points), then min xyz, edge (f64 LE), num_points as u32, bytes_per_coordinate as u8, pad
// to 8, position bytes, pad, colour bytes, pad.  Returns the blob size, or -1 - k if request k cannot be served.
int64_t orc_nodes_data_blob(void* hp, const uint64_t* ids_hi_lo, uint32_t num_nodes, uint8_t* out, uint64_t cap) {
    Handle* h = (Handle*)hp;
    std::vector<uint8_t> blob;
    auto pad = [&]() {
        while (blob.size() % 8) blob.push_back(0);
    };
    auto put = [&](const void* p, size_t n) { blob.insert(blob.end(), (const uint8_t*)p, (const uint8_t*)p + n); };
    for (uint32_t k = 0; k < num_nodes; ++k) {
        NodeId id = NodeId::from_high_low(ids_hi_lo[2 * k], ids_hi_lo[2 * k + 1]);
        auto f = h->oct.files.find(id);
        if (!h->oct.nodes.count(id) || f == h->oct.files.end()) return -1 - (int64_t)k;
        const NodeMeta& m = h->oct.nodes[id];
        put(&m.cube.min.x, 8), put(&m.cube.min.y, 8), put(&m.cube.min.z, 8), put(&m.cube.edge, 8);
        const uint32_t n32 = (uint32_t)m.num_points;
        put(&n32, 4);
        const uint8_t bpc = (uint8_t)bytes_per_coordinate(m.enc);
        put(&bpc, 1);
        pad();
        put(f->second.xyz.data(), f->second.xyz.size());
        pad();
        put(f->second.rgb.data(), f->second.rgb.size());
        pad();
    }
    if (out && cap >= blob.size()) std::memcpy(out, blob.data(), blob.size());
    return (int64_t)blob.size();
}

// ---- PLY input (oracle_ply.hpp) ----
struct orc_ply_info {
    uint64_t num_points, header_bytes;
    uint32_t record_bytes;
    int32_t has_color, has_intensity, num_fields;
    double offset[3];
};
static thread_local std::string g_ply_err;
const char* orc_ply_error() { return g_ply_err.c_str(); }
int orc_ply_open(const char* path, orc_ply_info* out) {
    PlyLayout L;
    if (!ply_open(path, L, g_ply_err)) return -1;
    out->num_points = (uint64_t)L.num_points;
    out->header_bytes = L.header.header_len;
    out->record_bytes = L.record_bytes;
    out->has_color = L.has_color;
    out->has_intensity = L.has_intensity;
    out->num_fields = (int32_t)L.fields.size();
    for (int a = 0; a < 3; ++a) out->offset[a] = L.header.offset[a];
    return 0;
}
// field i of the vertex record: role (PlyRole), type (PlyType), byte offset, bytes consumed
int orc_ply_field(const char* path, int i, int32_t* role, int32_t* type, uint32_t* offset, uint32_t* bytes) {
    PlyLayout L;
    if (!ply_open(path, L, g_ply_err) || i < 0 || i >= (int)L.fields.size()) return -1;
    *role = L.fields[i].role;
    *type = L.fields[i].type;
    *offset = L.fields[i].offset;
    *bytes = L.fields[i].bytes;
    return 0;
}
int orc_ply_read(const char* path, uint64_t first, uint64_t count, double* x, double* y, double* z, uint8_t* rgb, float* intensity) {
    PlyLayout L;
    if (!ply_open(path, L, g_ply_err)) return -1;
    return ply_read_range(path, L, first, count, x, y, z, L.has_color ? rgb : nullptr, L.has_intensity ? intensity : nullptr, g_ply_err) ? 0 : -1;
}
int orc_ply_find_bounding_box(const char* path, double* out6) {
    return ply_find_bounding_box(path, out6, out6 + 3, g_ply_err) ? 0 : -1;
}

}  // extern "C"
