// pcv.hpp — header-only C++ host layer over the C ABI (pcv.h), mirroring the names, argument meaning and error behaviour
// of the reference's Rust interface for this path, so that callers (and tests) read like the reference's own:
//
//   point_viewer::octree::build_octree                  src/octree/generation.rs:289-295   -> pcv::build_octree
//   point_viewer::octree::Octree::{from_data_provider, get_visible_nodes, get_node_data, nodes_in_location}
//                                                       src/octree/mod.rs:156,228,285,329  -> pcv::Octree
//   point_viewer::iterator::{PointQuery, PointLocation, ParallelIterator::try_for_each_batch}
//                                                       src/iterator.rs:13-20,66-72,255    -> pcv::PointQuery, pcv::ParallelIterator
//   point_viewer::{PointsBatch, NodeId}                 src/lib.rs:102-107, src/octree/node.rs:52-111
//   point_viewer::s2_cells::S2Cells, read_write::S2Splitter   src/s2_cells/mod.rs, src/read_write/s2.rs  -> pcv::S2Cells, pcv::s2_split
//
// Error behaviour: the reference panics (unwrap) in build_octree / get_visible_nodes and returns Result elsewhere; here
// every failure is a pcv::Error exception carrying the pcv_status and text (callers that want the panic semantics let it
// propagate).  A consumer callback returning false cancels the stream (== Err -> ErrorKind::Channel).
#pragma once
#include <array>
#include <cstdint>
#include <functional>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "pcv.h"

namespace pcv {

struct Error : std::runtime_error {
    int status;
    Error(int s, const std::string& m) : std::runtime_error(m), status(s) {}
};
inline void check(int rc) {
    if (rc != PCV_OK) throw Error(rc, pcv_last_error());
}

// NodeId: u128 = level << 120 | index (node.rs:52-111), Display "r" + octal path (node.rs:73-86)
struct NodeId {
    uint64_t high = 0, low = 0;
    int level() const { return (int)(high >> 56); }
    std::string to_string() const {
        unsigned __int128 v = ((unsigned __int128)high << 64) | low;
        std::string s(1, 'r');
        for (int i = level() - 1; i >= 0; --i) s.push_back((char)('0' + (int)((v >> (3 * i)) & 7)));
        return s;
    }
    bool operator==(const NodeId& o) const { return high == o.high && low == o.low; }
};

struct Aabb {  // Aabb::new takes inf/sup of the two corners (aabb.rs:19-24)
    std::array<double, 3> min, max;
    Aabb(std::array<double, 3> a, std::array<double, 3> b) {
        for (int i = 0; i < 3; ++i) {
            min[i] = a[i] < b[i] ? a[i] : b[i];
            max[i] = a[i] < b[i] ? b[i] : a[i];
        }
    }
};

// PointsBatch (lib.rs:102-107): AoS positions + colour (U8Vec3) and optional intensity (F32)
struct PointsBatch {
    std::vector<std::array<double, 3>> position;
    std::vector<std::array<uint8_t, 3>> color;
    std::vector<float> intensity;         // empty if absent
    std::vector<uint64_t> source_index;   // provenance (not in the reference)
};

// PointLocation (iterator.rs:13-20).  Frustum / Obb carry the fields the reference structs hold.
struct PointLocation {
    pcv_location raw{};
    static PointLocation AllPoints() {
        PointLocation l;
        l.raw.kind = PCV_LOC_ALL;
        return l;
    }
    static PointLocation from(const Aabb& b) {
        PointLocation l;
        l.raw.kind = PCV_LOC_AABB;
        for (int i = 0; i < 3; ++i) {
            l.raw.aabb_min[i] = b.min[i];
            l.raw.aabb_max[i] = b.max[i];
        }
        return l;
    }
    // Frustum{query_from_clip, clip_from_query}: column-major 4x4 (nalgebra storage)
    static PointLocation Frustum(const double clip_from_query[16], const double query_from_clip[16]) {
        PointLocation l;
        l.raw.kind = PCV_LOC_FRUSTUM;
        for (int i = 0; i < 16; ++i) {
            l.raw.clip_from_query[i] = clip_from_query[i];
            l.raw.query_from_clip[i] = query_from_clip[i];
        }
        return l;
    }
    // Obb{query_from_obb, obb_from_query, half_extent}: isometries as tx,ty,tz,qi,qj,qk,qw
    static PointLocation Obb(const double query_from_obb[7], const double obb_from_query[7], const double half_extent[3]) {
        PointLocation l;
        l.raw.kind = PCV_LOC_OBB;
        for (int i = 0; i < 7; ++i) {
            l.raw.query_from_obb[i] = query_from_obb[i];
            l.raw.obb_from_query[i] = obb_from_query[i];
        }
        for (int i = 0; i < 3; ++i) l.raw.half_extent[i] = half_extent[i];
        return l;
    }
    // WebMercatorRect::from_zoomed_coordinates(min, max, z) (web_mercator_rect.rs:40-53), map pixels at zoom z; throws
    // Error(PCV_ERR_INVALID) where the reference returns None.
    static PointLocation WebMercatorRect(const std::array<double, 2>& min, const std::array<double, 2>& max, uint32_t z) {
        PointLocation l;
        check(pcv_web_mercator_rect(min.data(), max.data(), z, &l.raw));
        return l;
    }
};

// WebMercatorCoord::from_lat_lng(ECEF -> WGS84).to_zoomed_coordinate(z): an ECEF point's map pixel at zoom z.
inline std::array<double, 2> web_mercator_coord(const std::array<double, 3>& ecef, uint32_t z) {
    std::array<double, 2> out{};
    check(pcv_web_mercator_coord(ecef.data(), z, out.data()));
    return out;
}

struct ClosedInterval {
    double lower_bound, upper_bound;
};
struct PointQuery {  // iterator.rs:66-72 (attributes: colour is always delivered, intensity when the octree has it)
    PointLocation location = PointLocation::AllPoints();
    std::vector<ClosedInterval> filter_intervals;  // on "intensity"
};

namespace detail {
// The tile callback of the X-ray quadtree entries over a C++ callable (level, index, RGBA, tile_px).
template <class F>
struct XrayThunk {
    F* f;
    static int call(void* user, uint8_t level, uint64_t index, const uint8_t* rgba, uint32_t tile_px) {
        (*static_cast<XrayThunk*>(user)->f)(level, index, rgba, tile_px);
        return 0;
    }
};
}  // namespace detail

class Context {
   public:
    explicit Context(int device = 0, uint64_t max_points_per_node = 0) {
        pcv_config cfg{max_points_per_node, 0, 0};
        check(pcv_create(device, &cfg, &h_));
    }
    ~Context() { pcv_destroy(h_); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    pcv_ctx* raw() const { return h_; }
    // build_xray_quadtree over the octree in `octree_dir` (build_quadtree.rs), streamed from disk window by window: what
    // Octree::build_xray_quadtree gives over the loaded directory.  `max_device_bytes` bounds everything the call allocates.
    template <class F>
    pcv_xray_quadtree_info build_xray_quadtree_from_dir(const std::string& octree_dir, const pcv_xray_quadtree_params& params, F&& on_tile,
                                                        uint64_t max_device_bytes = 0, pcv_xray_bounded_info* bounded_info = nullptr,
                                                        pcv_xray_dir_info* dir_info = nullptr) const {
        detail::XrayThunk<std::remove_reference_t<F>> th{&on_tile};
        pcv_xray_quadtree_info info{};
        check(pcv_xray_quadtree_from_dir(h_, octree_dir.c_str(), &params, max_device_bytes, &decltype(th)::call, &th, &info, bounded_info, dir_info));
        return info;
    }

   private:
    pcv_ctx* h_ = nullptr;
};

using CellID = uint64_t;                 // s2::cellid::CellID(u64)
using CellUnion = std::vector<CellID>;   // s2::cellunion::CellUnion(Vec<CellID>)

// The octree queries by cell union (PointLocation::S2Cells) shared by Octree and OctreeDir, over their pcv_* entry points.
namespace detail {
inline pcv_cell_union raw_union(const CellUnion& cu) { return pcv_cell_union{cu.data(), (uint32_t)cu.size(), 0}; }
inline std::vector<pcv_cell_union> raw_unions(const std::vector<CellUnion>& us) {
    std::vector<pcv_cell_union> raw;
    for (auto& u : us) raw.push_back(raw_union(u));
    return raw;
}
// A pcv_*_batch_points_device entry over raw locations or cell unions: offsets (one per location, plus one) on the host, the
// points to the device arrays.  Returns the total.
template <class Fn, class H, class Raw>
uint64_t batch_points(Fn fn, H h, const std::vector<Raw>& raw, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                      double* d_xyz, uint8_t* d_rgb, float* d_intensity, uint64_t* d_src, uint64_t cap) {
    std::vector<pcv_interval> f;
    for (auto& iv : filter_intervals) f.push_back(pcv_interval{iv.lower_bound, iv.upper_bound});
    offsets.assign(raw.size() + 1, 0);
    check(fn(h, raw.data(), (uint32_t)raw.size(), f.empty() ? nullptr : f.data(), (uint32_t)f.size(), offsets.data(), d_xyz, d_rgb, d_intensity, d_src, cap));
    return offsets.back();
}
}  // namespace detail

struct NodeData {  // octree/mod.rs:147-152
    pcv_node_meta meta;
    std::vector<uint8_t> position, color;
};

class Octree {
   public:
    Octree(pcv_octree* o) : o_(o) { load_table(); }
    // Octree::from_data_provider(OnDiskDataProvider{directory})
    static Octree from_directory(Context& ctx, const std::string& dir) {
        pcv_octree* o = nullptr;
        check(pcv_octree_load_dir(ctx.raw(), dir.c_str(), &o));
        return Octree(o);
    }
    Octree(Octree&& other) noexcept : o_(other.o_), nodes_(std::move(other.nodes_)) { other.o_ = nullptr; }
    Octree(const Octree&) = delete;
    ~Octree() {
        if (o_) pcv_octree_free(o_);
    }
    const std::vector<pcv_node_meta>& nodes() const { return nodes_; }
    int64_t num_points() const {
        int64_t n = 0;
        for (auto& m : nodes_) n += m.num_points;
        return n;
    }
    std::vector<NodeId> get_visible_nodes(const double projection_matrix[16]) const {  // mod.rs:228 (panics if singular)
        std::vector<uint64_t> ids(2 * nodes_.size() + 2);
        uint64_t n = 0;
        check(pcv_visible_nodes(o_, projection_matrix, ids.data(), nodes_.size(), &n));
        return to_ids(ids, n);
    }
    std::vector<NodeId> nodes_in_location(const PointLocation& loc) const {  // mod.rs:329-331
        std::vector<uint64_t> ids(2 * nodes_.size() + 2);
        uint64_t n = 0;
        check(pcv_nodes_in_location(o_, &loc.raw, ids.data(), nodes_.size(), &n));
        return to_ids(ids, n);
    }
    // PointLocation::S2Cells: every node that holds a point whose leaf cell the union contains, in BFS order
    std::vector<NodeId> nodes_in_location(const CellUnion& cell_union) const {
        std::vector<uint64_t> ids(2 * nodes_.size() + 2);
        uint64_t n = 0;
        const pcv_cell_union cu = detail::raw_union(cell_union);
        check(pcv_nodes_in_cell_union(o_, &cu, ids.data(), nodes_.size(), &n));
        return to_ids(ids, n);
    }
    // The points of PointLocation::S2Cells(cell_union) that pass the filter intervals, in batches of `batch_size` points (the
    // last one short), in AllPoints order; func returns false to stop.  Returns true if every batch was consumed.
    bool for_each_batch(const CellUnion& cell_union, const std::vector<ClosedInterval>& filter_intervals, size_t batch_size,
                        const std::function<bool(PointsBatch&&)>& func) const;
    // survivors and tested points of every cell union
    void query_batch(const std::vector<CellUnion>& unions, std::vector<uint64_t>& counts, std::vector<uint64_t>& tested) const {
        const std::vector<pcv_cell_union> raw = detail::raw_unions(unions);
        counts.assign(unions.size(), 0);
        tested.assign(unions.size(), 0);
        check(pcv_query_cell_unions_batch_device(o_, raw.data(), (uint32_t)raw.size(), nullptr, 0, counts.data(), tested.data()));
    }
    // The points of every location in device memory (pcv_query_batch_points_device): [offsets[i], offsets[i + 1]) of the device
    // arrays, which hold cap points, is what for_each_batch streams for locs[i].  d_xyz == nullptr: offsets only; d_rgb,
    // d_intensity and d_src may be nullptr.  Returns the total.
    uint64_t query_batch_points(const std::vector<PointLocation>& locs, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                                double* d_xyz = nullptr, uint8_t* d_rgb = nullptr, float* d_intensity = nullptr, uint64_t* d_src = nullptr,
                                uint64_t cap = 0) const {
        std::vector<pcv_location> raw;
        for (auto& l : locs) raw.push_back(l.raw);
        return detail::batch_points(pcv_query_batch_points_device, o_, raw, filter_intervals, offsets, d_xyz, d_rgb, d_intensity, d_src, cap);
    }
    uint64_t query_batch_points(const std::vector<CellUnion>& unions, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                                double* d_xyz = nullptr, uint8_t* d_rgb = nullptr, float* d_intensity = nullptr, uint64_t* d_src = nullptr,
                                uint64_t cap = 0) const {
        return detail::batch_points(pcv_query_cell_unions_batch_points_device, o_, detail::raw_unions(unions), filter_intervals, offsets, d_xyz, d_rgb,
                                    d_intensity, d_src, cap);
    }
    NodeData get_node_data(const NodeId& id) const {  // mod.rs:285-307
        for (auto& m : nodes_)
            if (m.id_high == id.high && m.id_low == id.low) {
                NodeData d;
                d.meta = m;
                const size_t bpc = m.position_encoding == 1 ? 1 : m.position_encoding == 2 ? 2 : m.position_encoding == 3 ? 4 : 8;
                d.position.resize((size_t)m.num_points * 3 * bpc);
                d.color.resize((size_t)m.num_points * 3);
                check(pcv_octree_node_data(o_, id.high, id.low, d.position.data(), d.color.data(), nullptr, nullptr));
                return d;
            }
        throw Error(PCV_ERR_NOT_FOUND, "node " + id.to_string() + " not found");
    }
    // The web viewer's /nodes_data reply for a list of nodes (octree_web_viewer/src/backend.rs:92-165), gathered on the GPU.
    std::vector<uint8_t> nodes_data_blob(const std::vector<NodeId>& ids) const {
        std::vector<uint64_t> hl;
        for (auto& id : ids) hl.push_back(id.high), hl.push_back(id.low);
        uint64_t size = 0;
        check(pcv_nodes_data_blob(o_, hl.data(), (uint32_t)ids.size(), nullptr, 0, &size));
        std::vector<uint8_t> blob(size);
        if (size) check(pcv_nodes_data_blob(o_, hl.data(), (uint32_t)ids.size(), blob.data(), size, &size));
        return blob;
    }
    // xray_from_points for one tile with ColoringStrategyKind::{Colored, ColoredWithIntensity, ColoredWithHeightStddev}
    // (xray/src/generation.rs:76-97); returns false for a tile without points (None in the reference).
    bool xray_tile_attr(const Aabb& tile, uint32_t w, uint32_t h, int strategy, float p0, float p1, int colormap, std::vector<uint8_t>& rgba,
                        const double* query_from_global7 = nullptr) const {
        rgba.assign((size_t)w * h * 4, 0);
        int any = 0;
        check(pcv_xray_tile_attr(o_, tile.min.data(), tile.max.data(), w, h, query_from_global7, strategy, p0, p1, colormap, rgba.data(), &any));
        return any != 0;
    }
    // ... with Binning = Some(("intensity", bin_size)) for the Colored / ColoredWithIntensity strategies (generation.rs:129-157)
    bool xray_tile_attr_binned(const Aabb& tile, uint32_t w, uint32_t h, int strategy, float p0, float p1, double bin_size, std::vector<uint8_t>& rgba,
                               const double* query_from_global7 = nullptr) const {
        rgba.assign((size_t)w * h * 4, 0);
        int any = 0;
        check(pcv_xray_tile_attr_binned(o_, tile.min.data(), tile.max.data(), w, h, query_from_global7, strategy, p0, p1, bin_size, rgba.data(), &any));
        return any != 0;
    }
    // build_xray_quadtree (xray/src/generation.rs:560-622): every tile of the quadtree through `on_tile` (level, index, RGBA
    // tile_size_px^2) in post-order - every tile after all of its children, the root last; returns what the reference writes
    // into the quadtree's meta.pb.  `max_device_bytes` bounds the driver's device memory (0: most of the free memory).
    template <class F>
    pcv_xray_quadtree_info build_xray_quadtree(const pcv_xray_quadtree_params& params, F&& on_tile, uint64_t max_device_bytes = 0,
                                               pcv_xray_bounded_info* bounded_info = nullptr) const {
        detail::XrayThunk<std::remove_reference_t<F>> th{&on_tile};
        pcv_xray_quadtree_info info{};
        check(pcv_xray_quadtree_bounded(o_, &params, max_device_bytes, &decltype(th)::call, &th, &info, bounded_info));
        return info;
    }
    void write_to_directory(const std::string& dir) const { check(pcv_octree_write_dir(o_, dir.c_str())); }
    pcv_octree* raw() const { return o_; }

   private:
    void load_table() {
        uint64_t nn = 0;
        check(pcv_octree_info(o_, &nn, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr));
        nodes_.resize(nn);
        check(pcv_octree_nodes(o_, nodes_.data(), nn));
    }
    static std::vector<NodeId> to_ids(const std::vector<uint64_t>& v, uint64_t n) {
        std::vector<NodeId> out(n);
        for (uint64_t i = 0; i < n; ++i) out[i] = NodeId{v[2 * i], v[2 * i + 1]};
        return out;
    }
    pcv_octree* o_;
    std::vector<pcv_node_meta> nodes_;
};

inline PointsBatch batch_from(const pcv_batch* b) {
    PointsBatch pb;
    pb.position.resize(b->n);
    if (b->rgb) pb.color.resize(b->n);  // an S2 cloud without colour delivers none
    for (uint64_t i = 0; i < b->n; ++i) {
        pb.position[i] = {b->xyz[3 * i], b->xyz[3 * i + 1], b->xyz[3 * i + 2]};
        if (b->rgb) pb.color[i] = {b->rgb[3 * i], b->rgb[3 * i + 1], b->rgb[3 * i + 2]};
    }
    if (b->intensity) pb.intensity.assign(b->intensity, b->intensity + b->n);
    pb.source_index.assign(b->src_index, b->src_index + b->n);
    return pb;
}

namespace detail {
// One streaming call (query(cb, user)) with `func` as the consumer: false if func stopped it.
template <class Q>
inline bool stream_batches(const std::function<bool(PointsBatch&&)>& func, Q&& query) {
    auto tramp = [](void* user, const pcv_batch* b) -> int { return (*(const std::function<bool(PointsBatch&&)>*)user)(batch_from(b)) ? 0 : 1; };
    const int rc = query(+tramp, (void*)&func);
    if (rc == PCV_ERR_CANCELLED) return false;
    check(rc);
    return true;
}
inline std::vector<pcv_interval> raw_intervals(const std::vector<ClosedInterval>& iv) {
    std::vector<pcv_interval> f;
    for (auto& i : iv) f.push_back(pcv_interval{i.lower_bound, i.upper_bound});
    return f;
}
}  // namespace detail

inline bool Octree::for_each_batch(const CellUnion& cell_union, const std::vector<ClosedInterval>& filter_intervals, size_t batch_size,
                                   const std::function<bool(PointsBatch&&)>& func) const {
    const pcv_cell_union cu = detail::raw_union(cell_union);
    const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
    return detail::stream_batches(func, [&](pcv_batch_cb cb, void* user) {
        return pcv_query_cell_union(o_, &cu, f.empty() ? nullptr : f.data(), (uint32_t)f.size(), batch_size, cb, user);
    });
}

// An octree directory queried where it lies (Octree over OnDiskDataProvider, octree/mod.rs:156-215, 337-352): the node table is
// on the device and every query reads only the nodes it selects, within `max_device_bytes`.  Results equal Octree::from_directory's;
// a batch's source_index is the point's slot in nodes() (point_offset + j of its node).
class OctreeDir {
   public:
    OctreeDir(Context& ctx, const std::string& dir, uint64_t max_device_bytes = 0) {
        check(pcv_octree_dir_open(ctx.raw(), dir.c_str(), max_device_bytes, &d_));
        uint64_t nn = 0;
        check(pcv_octree_dir_info(d_, &nn, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr));
        nodes_.resize(nn);
        check(pcv_octree_dir_nodes(d_, nodes_.data(), nn));
    }
    OctreeDir(const OctreeDir&) = delete;
    OctreeDir& operator=(const OctreeDir&) = delete;
    ~OctreeDir() { pcv_octree_dir_close(d_); }
    const std::vector<pcv_node_meta>& nodes() const { return nodes_; }
    std::vector<NodeId> get_visible_nodes(const double projection_matrix[16]) const {
        std::vector<uint64_t> ids(2 * nodes_.size() + 2);
        uint64_t n = 0;
        check(pcv_octree_dir_visible_nodes(d_, projection_matrix, ids.data(), nodes_.size(), &n));
        return to_ids(ids, n);
    }
    std::vector<NodeId> nodes_in_location(const PointLocation& loc) const {
        std::vector<uint64_t> ids(2 * nodes_.size() + 2);
        uint64_t n = 0;
        check(pcv_octree_dir_nodes_in_location(d_, &loc.raw, ids.data(), nodes_.size(), &n));
        return to_ids(ids, n);
    }
    // PointQuery streamed in batches of `batch_size` points (the last one short); func returns false to stop.  Returns true if
    // every batch was consumed.
    bool for_each_batch(const PointQuery& query, size_t batch_size, const std::function<bool(PointsBatch&&)>& func) const {
        auto tramp = [](void* user, const pcv_batch* b) -> int { return (*(const std::function<bool(PointsBatch&&)>*)user)(batch_from(b)) ? 0 : 1; };
        std::vector<pcv_interval> f;
        for (auto& iv : query.filter_intervals) f.push_back(pcv_interval{iv.lower_bound, iv.upper_bound});
        const int rc = pcv_octree_dir_query_points(d_, &query.location.raw, f.empty() ? nullptr : f.data(), (uint32_t)f.size(), batch_size, tramp,
                                                   (void*)&func);
        if (rc == PCV_ERR_CANCELLED) return false;
        check(rc);
        return true;
    }
    // survivors and tested points of every location, each visited node read once
    void query_batch(const std::vector<PointLocation>& locs, std::vector<uint64_t>& counts, std::vector<uint64_t>& tested) const {
        std::vector<pcv_location> raw;
        for (auto& l : locs) raw.push_back(l.raw);
        counts.assign(locs.size(), 0);
        tested.assign(locs.size(), 0);
        check(pcv_octree_dir_query_batch(d_, raw.data(), (uint32_t)raw.size(), nullptr, 0, counts.data(), tested.data()));
    }
    // The cell-union forms of Octree's, over the directory (source_index = slot)
    std::vector<NodeId> nodes_in_location(const CellUnion& cell_union) const {
        std::vector<uint64_t> ids(2 * nodes_.size() + 2);
        uint64_t n = 0;
        const pcv_cell_union cu = detail::raw_union(cell_union);
        check(pcv_octree_dir_nodes_in_cell_union(d_, &cu, ids.data(), nodes_.size(), &n));
        return to_ids(ids, n);
    }
    bool for_each_batch(const CellUnion& cell_union, const std::vector<ClosedInterval>& filter_intervals, size_t batch_size,
                        const std::function<bool(PointsBatch&&)>& func) const {
        const pcv_cell_union cu = detail::raw_union(cell_union);
        const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
        return detail::stream_batches(func, [&](pcv_batch_cb cb, void* user) {
            return pcv_octree_dir_query_cell_union(d_, &cu, f.empty() ? nullptr : f.data(), (uint32_t)f.size(), batch_size, cb, user);
        });
    }
    void query_batch(const std::vector<CellUnion>& unions, std::vector<uint64_t>& counts, std::vector<uint64_t>& tested) const {
        const std::vector<pcv_cell_union> raw = detail::raw_unions(unions);
        counts.assign(unions.size(), 0);
        tested.assign(unions.size(), 0);
        check(pcv_octree_dir_query_cell_unions_batch(d_, raw.data(), (uint32_t)raw.size(), nullptr, 0, counts.data(), tested.data()));
    }
    // Octree::query_batch_points over the directory (pcv_octree_dir_query_batch_points_device): [offsets[i], offsets[i + 1]) of the
    // device arrays is what for_each_batch streams for locs[i] (source_index = slot).  Returns the total.
    uint64_t query_batch_points(const std::vector<PointLocation>& locs, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                                double* d_xyz = nullptr, uint8_t* d_rgb = nullptr, float* d_intensity = nullptr, uint64_t* d_src = nullptr,
                                uint64_t cap = 0) const {
        std::vector<pcv_location> raw;
        for (auto& l : locs) raw.push_back(l.raw);
        return detail::batch_points(pcv_octree_dir_query_batch_points_device, d_, raw, filter_intervals, offsets, d_xyz, d_rgb, d_intensity, d_src, cap);
    }
    uint64_t query_batch_points(const std::vector<CellUnion>& unions, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                                double* d_xyz = nullptr, uint8_t* d_rgb = nullptr, float* d_intensity = nullptr, uint64_t* d_src = nullptr,
                                uint64_t cap = 0) const {
        return detail::batch_points(pcv_octree_dir_query_cell_unions_batch_points_device, d_, detail::raw_unions(unions), filter_intervals, offsets, d_xyz,
                                    d_rgb, d_intensity, d_src, cap);
    }
    std::vector<uint8_t> nodes_data_blob(const std::vector<NodeId>& ids) const {
        std::vector<uint64_t> hl;
        for (auto& id : ids) hl.push_back(id.high), hl.push_back(id.low);
        uint64_t size = 0;
        check(pcv_octree_dir_nodes_data_blob(d_, hl.data(), (uint32_t)ids.size(), nullptr, 0, &size));
        std::vector<uint8_t> blob(size);
        if (size) check(pcv_octree_dir_nodes_data_blob(d_, hl.data(), (uint32_t)ids.size(), blob.data(), size, &size));
        return blob;
    }
    pcv_dir_query_stats last_stats() const {
        pcv_dir_query_stats s{};
        check(pcv_octree_dir_last_stats(d_, &s));
        return s;
    }
    pcv_octree_dir* raw() const { return d_; }

   private:
    static std::vector<NodeId> to_ids(const std::vector<uint64_t>& v, uint64_t n) {
        std::vector<NodeId> out(n);
        for (uint64_t i = 0; i < n; ++i) out[i] = NodeId{v[2 * i], v[2 * i + 1]};
        return out;
    }
    pcv_octree_dir* d_ = nullptr;
    std::vector<pcv_node_meta> nodes_;
};

// build_octree(output_directory, resolution, bounding_box, input, attributes) — generation.rs:289-295.  `input` is drained on
// the calling thread; colour is mandatory; attributes selects whether intensity is carried.  Returns the GPU-resident
// octree as well (the reference returns ()).
template <class BatchIterator>
inline Octree build_octree(Context& ctx, const std::string& output_directory, double resolution, const Aabb& bounding_box, BatchIterator begin,
                           BatchIterator end, const std::vector<std::string>& attributes = {"color"}) {
    std::vector<std::array<double, 3>> pos;
    std::vector<std::array<uint8_t, 3>> col;
    std::vector<float> inten;
    bool want_i = false;
    for (auto& a : attributes) want_i = want_i || a == "intensity";
    for (BatchIterator it = begin; it != end; ++it) {
        const PointsBatch& b = *it;
        if (b.color.size() != b.position.size()) throw Error(PCV_ERR_INVALID, "color is mandatory (on_disk.rs:23-33)");
        pos.insert(pos.end(), b.position.begin(), b.position.end());
        col.insert(col.end(), b.color.begin(), b.color.end());
        if (want_i && !b.intensity.empty()) inten.insert(inten.end(), b.intensity.begin(), b.intensity.end());
    }
    pcv_points pts{};
    const double* base = pos.empty() ? nullptr : pos[0].data();
    pts.x = base;
    pts.y = base ? base + 1 : nullptr;
    pts.z = base ? base + 2 : nullptr;
    pts.stride = 3;  // AoS Point3<f64>, no transpose
    pts.rgb = col.empty() ? nullptr : col[0].data();
    pts.intensity = (want_i && inten.size() == pos.size() && !inten.empty()) ? inten.data() : nullptr;
    pts.n = pos.size();
    pcv_octree* o = nullptr;
    check(pcv_build_octree(ctx.raw(), &pts, resolution, bounding_box.min.data(), bounding_box.max.data(), &o));
    Octree tree(o);
    if (!output_directory.empty()) tree.write_to_directory(output_directory);
    return tree;
}

// build_octree_from_file(output_directory, resolution, filename, attributes) — generation.rs:272-287: the PLY body goes to the
// GPU as raw records, the bounding-box pass is fused into the unpack kernel.
inline Octree build_octree_from_file(Context& ctx, const std::string& output_directory, double resolution, const std::string& filename,
                                     const std::vector<std::string>& attributes = {"color"}) {
    bool want_i = false;
    for (auto& a : attributes) want_i = want_i || a == "intensity";
    pcv_octree* o = nullptr;
    check(pcv_build_octree_from_file(ctx.raw(), filename.c_str(), resolution, want_i ? 1 : 0, &o));
    Octree tree(o);
    if (!output_directory.empty()) tree.write_to_directory(output_directory);
    return tree;
}

// ---- the S2-cell point cloud: point_viewer::s2_cells::S2Cells + read_write::S2Splitter (src/s2_cells/mod.rs, src/read_write/s2.rs) ----

// CellID::to_token (the per-cell file stem of the S2 directory layout)
inline std::string cell_token(CellID id) {
    if (id == 0) return "X";
    static const char* hex = "0123456789abcdef";
    std::string s;
    for (int k = 15; k >= 0; --k) s.push_back(hex[(id >> (4 * k)) & 15]);
    while (!s.empty() && s.back() == '0') s.pop_back();
    return s;
}

class S2Cells {
   public:
    explicit S2Cells(pcv_s2cloud* s) : s_(s) {}
    // S2Cells::from_data_provider over an on-disk directory (mod.rs:203-216)
    static S2Cells from_directory(Context& ctx, const std::string& directory) {
        pcv_s2cloud* s = nullptr;
        check(pcv_s2_load_dir(ctx.raw(), directory.c_str(), &s));
        return S2Cells(s);
    }
    // S2Splitter<RawNodeWriter>::write batch by batch + get_meta, straight to `directory` in bounded device memory: the files
    // pcv_s2_build + pcv_s2_write_dir would write (pcv_s2_build_to_dir).  Load them with from_directory.
    static pcv_s2_dir_build_info build_to_directory(Context& ctx, const pcv_points& host_points, const std::string& directory,
                                                    uint32_t split_level = 20, uint64_t max_device_bytes = 0) {
        pcv_s2_dir_build_info info{};
        check(pcv_s2_build_to_dir(ctx.raw(), &host_points, split_level, max_device_bytes, directory.c_str(), &info));
        return info;
    }
    static pcv_s2_dir_build_info build_file_to_directory(Context& ctx, const std::string& ply_path, const std::string& directory,
                                                         uint32_t split_level = 20, uint64_t max_device_bytes = 0) {
        pcv_s2_dir_build_info info{};
        check(pcv_s2_build_from_file_to_dir(ctx.raw(), ply_path.c_str(), split_level, max_device_bytes, directory.c_str(), &info));
        return info;
    }
    ~S2Cells() {
        if (s_) pcv_s2_free(s_);
    }
    S2Cells(S2Cells&& o) noexcept : s_(o.s_) { o.s_ = nullptr; }
    S2Cells(const S2Cells&) = delete;
    S2Cells& operator=(const S2Cells&) = delete;

    uint64_t num_points() const {
        uint64_t n = 0;
        check(pcv_s2_info(s_, nullptr, &n, nullptr, nullptr, nullptr, nullptr, nullptr));
        return n;
    }
    Aabb bounding_box() const {  // PointCloud::bounding_box (mod.rs:192-194)
        std::array<double, 3> mn{}, mx{};
        check(pcv_s2_info(s_, nullptr, nullptr, nullptr, mn.data(), mx.data(), nullptr, nullptr));
        return Aabb(mn, mx);
    }
    // S2Meta::get_cells: (cell id, num_points), in id order
    std::vector<std::pair<CellID, uint64_t>> cells() const {
        uint64_t nc = 0;
        check(pcv_s2_info(s_, &nc, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr));
        std::vector<uint64_t> ids(nc), cnt(nc);
        check(pcv_s2_cells(s_, ids.data(), cnt.data()));
        std::vector<std::pair<CellID, uint64_t>> out(nc);
        for (uint64_t k = 0; k < nc; ++k) out[k] = {ids[k], cnt[k]};
        return out;
    }
    // PointCloud::nodes_in_location for PointLocation::AllPoints (nullptr) and PointLocation::S2Cells (mod.rs:157-168)
    std::vector<CellID> nodes_in_location(const CellUnion* cell_union) const {
        uint64_t n = 0;
        const uint64_t* u = cell_union ? cell_union->data() : nullptr;
        const uint32_t nu = cell_union ? (uint32_t)cell_union->size() : 0;
        check(pcv_s2_cells_in_union(s_, u, nu, nullptr, 0, &n));
        std::vector<CellID> out(n);
        check(pcv_s2_cells_in_union(s_, u, nu, out.data(), n, &n));
        return out;
    }
    // points_in_node (mod.rs:174-190) as one batch
    PointsBatch points_in_node(CellID id) const {
        PointsBatch b;
        for (auto& c : cells())
            if (c.first == id) {
                int hc = 0, hi = 0;
                check(pcv_s2_info(s_, nullptr, nullptr, nullptr, nullptr, nullptr, &hc, &hi));
                b.position.resize(c.second);
                if (hc) b.color.resize(c.second);
                if (hi) b.intensity.resize(c.second);
                check(pcv_s2_cell_data(s_, id, c.second ? b.position[0].data() : nullptr, hc && c.second ? b.color[0].data() : nullptr,
                                       hi && c.second ? b.intensity.data() : nullptr, nullptr));
                return b;
            }
        throw Error(PCV_ERR_NOT_FOUND, "cell " + cell_token(id) + " not found");
    }
    // the filtered point stream of PointLocation::AllPoints / S2Cells (iterator.rs:96-119 with the CellUnion as PointCulling)
    PointsBatch query(const CellUnion* cell_union) const {
        const uint64_t* u = cell_union ? cell_union->data() : nullptr;
        const uint32_t nu = cell_union ? (uint32_t)cell_union->size() : 0;
        uint64_t n = 0;
        check(pcv_s2_query_union(s_, u, nu, nullptr, nullptr, nullptr, nullptr, 0, &n, nullptr));
        int hc = 0, hi = 0;
        check(pcv_s2_info(s_, nullptr, nullptr, nullptr, nullptr, nullptr, &hc, &hi));
        PointsBatch b;
        b.position.resize(n);
        if (hc) b.color.resize(n);
        if (hi) b.intensity.resize(n);
        if (n)
            check(pcv_s2_query_union(s_, u, nu, b.position[0].data(), hc ? b.color[0].data() : nullptr, hi ? b.intensity.data() : nullptr, nullptr, n, &n,
                                     nullptr));
        return b;
    }
    // PointCloud::nodes_in_location for AllPoints, Aabb, Obb and Frustum: the cells whose point box the location's separating-axis
    // test does not call Out, in id order (not the reference's rectangle-based list; see pcv_s2_cells_in_location)
    std::vector<CellID> nodes_in_location(const PointLocation& loc) const {
        uint64_t n = 0;
        check(pcv_s2_cells_in_location(s_, &loc.raw, nullptr, 0, &n));
        std::vector<CellID> out(n);
        check(pcv_s2_cells_in_location(s_, &loc.raw, out.data(), n, &n));
        return out;
    }
    // PointQuery streamed in batches of `batch_size` points (the last one short), in cell order; func returns false to stop.
    // Returns true if every batch was consumed.  `color` is empty for a cloud without colour.
    bool for_each_batch(const PointQuery& query, size_t batch_size, const std::function<bool(PointsBatch&&)>& func) const;
    // The points of PointLocation::S2Cells(cell_union) that pass the filter intervals, in cell order
    bool for_each_batch(const CellUnion& cell_union, const std::vector<ClosedInterval>& filter_intervals, size_t batch_size,
                        const std::function<bool(PointsBatch&&)>& func) const;
    // survivors and tested points of every location / cell union
    void query_batch(const std::vector<PointLocation>& locs, std::vector<uint64_t>& counts, std::vector<uint64_t>& tested) const {
        std::vector<pcv_location> raw;
        for (auto& l : locs) raw.push_back(l.raw);
        counts.assign(locs.size(), 0);
        tested.assign(locs.size(), 0);
        check(pcv_s2_query_batch_device(s_, raw.data(), (uint32_t)raw.size(), nullptr, 0, counts.data(), tested.data()));
    }
    void query_batch(const std::vector<CellUnion>& unions, std::vector<uint64_t>& counts, std::vector<uint64_t>& tested) const {
        const std::vector<pcv_cell_union> raw = detail::raw_unions(unions);
        counts.assign(unions.size(), 0);
        tested.assign(unions.size(), 0);
        check(pcv_s2_query_cell_unions_batch_device(s_, raw.data(), (uint32_t)raw.size(), nullptr, 0, counts.data(), tested.data()));
    }
    // Octree::query_batch_points over the cloud (pcv_s2_query_batch_points_device)
    uint64_t query_batch_points(const std::vector<PointLocation>& locs, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                                double* d_xyz = nullptr, uint8_t* d_rgb = nullptr, float* d_intensity = nullptr, uint64_t* d_src = nullptr,
                                uint64_t cap = 0) const {
        std::vector<pcv_location> raw;
        for (auto& l : locs) raw.push_back(l.raw);
        return detail::batch_points(pcv_s2_query_batch_points_device, s_, raw, filter_intervals, offsets, d_xyz, d_rgb, d_intensity, d_src, cap);
    }
    uint64_t query_batch_points(const std::vector<CellUnion>& unions, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                                double* d_xyz = nullptr, uint8_t* d_rgb = nullptr, float* d_intensity = nullptr, uint64_t* d_src = nullptr,
                                uint64_t cap = 0) const {
        return detail::batch_points(pcv_s2_query_cell_unions_batch_points_device, s_, detail::raw_unions(unions), filter_intervals, offsets, d_xyz, d_rgb,
                                    d_intensity, d_src, cap);
    }
    // build_xray_quadtree (xray/src/build_quadtree.rs) over the cloud, with the leaf queries' filter intervals: every tile through
    // `on_tile` in post-order, as Octree::build_xray_quadtree delivers it.  `max_device_bytes` bounds the call's device memory.
    template <class F>
    pcv_xray_quadtree_info xray_quadtree(const pcv_xray_quadtree_params& params, const std::vector<ClosedInterval>& filter_intervals, F&& on_tile,
                                         uint64_t max_device_bytes = 0, pcv_xray_bounded_info* bounded_info = nullptr) const {
        detail::XrayThunk<std::remove_reference_t<F>> th{&on_tile};
        const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
        pcv_xray_quadtree_info info{};
        check(pcv_s2_xray_quadtree(s_, &params, f.data(), (uint32_t)f.size(), max_device_bytes, &decltype(th)::call, &th, &info, bounded_info));
        return info;
    }
    void write_to_directory(const std::string& dir) const { check(pcv_s2_write_dir(s_, dir.c_str())); }
    pcv_s2cloud* raw() const { return s_; }

   private:
    pcv_s2cloud* s_;
};

// S2Cells over an OnDiskDataProvider (mod.rs:203-216): the directory queried where it lies (pcv_s2_dir).  Every call reads only
// the cells it selects, within `max_device_bytes`, and returns what S2Cells::from_directory's does (source_index = slot).
class S2CellsDir {
   public:
    S2CellsDir(Context& ctx, const std::string& dir, uint64_t max_device_bytes = 0) { check(pcv_s2_dir_open(ctx.raw(), dir.c_str(), max_device_bytes, &d_)); }
    S2CellsDir(const S2CellsDir&) = delete;
    S2CellsDir& operator=(const S2CellsDir&) = delete;
    ~S2CellsDir() { pcv_s2_dir_close(d_); }
    // AllPoints (nullptr) / S2Cells(cell_union): the cells whose id range intersects it, no file read
    std::vector<CellID> nodes_in_location(const CellUnion* cell_union) const {
        uint64_t n = 0;
        const uint64_t* u = cell_union ? cell_union->data() : nullptr;
        const uint32_t nu = cell_union ? (uint32_t)cell_union->size() : 0;
        check(pcv_s2_dir_cells_in_union(d_, u, nu, nullptr, 0, &n));
        std::vector<CellID> out(n);
        check(pcv_s2_dir_cells_in_union(d_, u, nu, out.data(), n, &n));
        return out;
    }
    // S2Cells::nodes_in_location over the directory (the first polyhedral call reads every position once for the point boxes)
    std::vector<CellID> nodes_in_location(const PointLocation& loc) const {
        uint64_t n = 0;
        check(pcv_s2_dir_cells_in_location(d_, &loc.raw, nullptr, 0, &n));
        std::vector<CellID> out(n);
        check(pcv_s2_dir_cells_in_location(d_, &loc.raw, out.data(), n, &n));
        return out;
    }
    bool for_each_batch(const PointQuery& query, size_t batch_size, const std::function<bool(PointsBatch&&)>& func) const {
        const std::vector<pcv_interval> f = detail::raw_intervals(query.filter_intervals);
        return detail::stream_batches(func, [&](pcv_batch_cb cb, void* user) {
            return pcv_s2_dir_query_points(d_, &query.location.raw, f.empty() ? nullptr : f.data(), (uint32_t)f.size(), batch_size, cb, user);
        });
    }
    bool for_each_batch(const CellUnion& cell_union, const std::vector<ClosedInterval>& filter_intervals, size_t batch_size,
                        const std::function<bool(PointsBatch&&)>& func) const {
        const pcv_cell_union cu = detail::raw_union(cell_union);
        const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
        return detail::stream_batches(func, [&](pcv_batch_cb cb, void* user) {
            return pcv_s2_dir_query_cell_union(d_, &cu, f.empty() ? nullptr : f.data(), (uint32_t)f.size(), batch_size, cb, user);
        });
    }
    // survivors and tested points of every location / cell union, each selected cell read once
    void query_batch(const std::vector<PointLocation>& locs, std::vector<uint64_t>& counts, std::vector<uint64_t>& tested) const {
        std::vector<pcv_location> raw;
        for (auto& l : locs) raw.push_back(l.raw);
        counts.assign(locs.size(), 0);
        tested.assign(locs.size(), 0);
        check(pcv_s2_dir_query_batch(d_, raw.data(), (uint32_t)raw.size(), nullptr, 0, counts.data(), tested.data()));
    }
    void query_batch(const std::vector<CellUnion>& unions, std::vector<uint64_t>& counts, std::vector<uint64_t>& tested) const {
        const std::vector<pcv_cell_union> raw = detail::raw_unions(unions);
        counts.assign(unions.size(), 0);
        tested.assign(unions.size(), 0);
        check(pcv_s2_dir_query_cell_unions_batch(d_, raw.data(), (uint32_t)raw.size(), nullptr, 0, counts.data(), tested.data()));
    }
    // Octree::query_batch_points over the directory's cells (pcv_s2_dir_query_batch_points_device; source_index = slot)
    uint64_t query_batch_points(const std::vector<PointLocation>& locs, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                                double* d_xyz = nullptr, uint8_t* d_rgb = nullptr, float* d_intensity = nullptr, uint64_t* d_src = nullptr,
                                uint64_t cap = 0) const {
        std::vector<pcv_location> raw;
        for (auto& l : locs) raw.push_back(l.raw);
        return detail::batch_points(pcv_s2_dir_query_batch_points_device, d_, raw, filter_intervals, offsets, d_xyz, d_rgb, d_intensity, d_src, cap);
    }
    uint64_t query_batch_points(const std::vector<CellUnion>& unions, const std::vector<ClosedInterval>& filter_intervals, std::vector<uint64_t>& offsets,
                                double* d_xyz = nullptr, uint8_t* d_rgb = nullptr, float* d_intensity = nullptr, uint64_t* d_src = nullptr,
                                uint64_t cap = 0) const {
        return detail::batch_points(pcv_s2_dir_query_cell_unions_batch_points_device, d_, detail::raw_unions(unions), filter_intervals, offsets, d_xyz, d_rgb,
                                    d_intensity, d_src, cap);
    }
    pcv_dir_query_stats last_stats() const {
        pcv_dir_query_stats st{};
        check(pcv_s2_dir_last_stats(d_, &st));
        return st;
    }
    pcv_s2_dir* raw() const { return d_; }

   private:
    pcv_s2_dir* d_ = nullptr;
};

// build_xray_quadtree over several resident octrees at once (point_cloud_client/src/lib.rs:118-141): the quadtree over the union
// of their boxes, every leaf made of the points of all of them that its location contains and that pass `filter_intervals`.
// Tiles through `on_tile` in post-order, as Octree::build_xray_quadtree delivers them (pcv_xray_quadtree_clouds).
template <class F>
pcv_xray_quadtree_info build_xray_quadtree(const std::vector<const Octree*>& clouds, const pcv_xray_quadtree_params& params,
                                           const std::vector<ClosedInterval>& filter_intervals, F&& on_tile, uint64_t max_device_bytes = 0,
                                           pcv_xray_bounded_info* bounded_info = nullptr) {
    std::vector<const pcv_octree*> raw;
    for (const Octree* o : clouds) raw.push_back(o ? o->raw() : nullptr);
    const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
    detail::XrayThunk<std::remove_reference_t<F>> th{&on_tile};
    pcv_xray_quadtree_info info{};
    check(pcv_xray_quadtree_clouds(raw.data(), (uint32_t)raw.size(), &params, f.data(), (uint32_t)f.size(), max_device_bytes, &decltype(th)::call, &th, &info,
                                   bounded_info));
    return info;
}
// ... over several resident S2 clouds at once (pcv_s2_xray_quadtree_clouds).
template <class F>
pcv_xray_quadtree_info build_xray_quadtree(const std::vector<const S2Cells*>& clouds, const pcv_xray_quadtree_params& params,
                                           const std::vector<ClosedInterval>& filter_intervals, F&& on_tile, uint64_t max_device_bytes = 0,
                                           pcv_xray_bounded_info* bounded_info = nullptr) {
    std::vector<const pcv_s2cloud*> raw;
    for (const S2Cells* s : clouds) raw.push_back(s ? s->raw() : nullptr);
    const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
    detail::XrayThunk<std::remove_reference_t<F>> th{&on_tile};
    pcv_xray_quadtree_info info{};
    check(pcv_s2_xray_quadtree_clouds(raw.data(), (uint32_t)raw.size(), &params, f.data(), (uint32_t)f.size(), max_device_bytes, &decltype(th)::call, &th, &info,
                                      bounded_info));
    return info;
}
// Context::build_xray_quadtree_from_dir with filter intervals (pcv_xray_quadtree_from_dir_filtered).
template <class F>
pcv_xray_quadtree_info build_xray_quadtree_from_dir(const Context& ctx, const std::string& octree_dir, const pcv_xray_quadtree_params& params,
                                                    const std::vector<ClosedInterval>& filter_intervals, F&& on_tile, uint64_t max_device_bytes = 0,
                                                    pcv_xray_bounded_info* bounded_info = nullptr, pcv_xray_dir_info* dir_info = nullptr) {
    const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
    detail::XrayThunk<std::remove_reference_t<F>> th{&on_tile};
    pcv_xray_quadtree_info info{};
    check(pcv_xray_quadtree_from_dir_filtered(ctx.raw(), octree_dir.c_str(), &params, f.data(), (uint32_t)f.size(), max_device_bytes, &decltype(th)::call, &th,
                                              &info, bounded_info, dir_info));
    return info;
}
// build_xray_quadtree over the octree directories `dirs` streamed from disk, none of them ever resident as a whole: the tiles of
// build_xray_quadtree over Octrees loaded from each of them, in the same order (pcv_xray_quadtree_from_dirs).
template <class F>
pcv_xray_quadtree_info build_xray_quadtree_from_dirs(const Context& ctx, const std::vector<std::string>& dirs, const pcv_xray_quadtree_params& params,
                                                     const std::vector<ClosedInterval>& filter_intervals, F&& on_tile, uint64_t max_device_bytes = 0,
                                                     pcv_xray_bounded_info* bounded_info = nullptr, pcv_xray_dir_info* dir_info = nullptr) {
    std::vector<const char*> raw;
    for (const std::string& d : dirs) raw.push_back(d.c_str());
    const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
    detail::XrayThunk<std::remove_reference_t<F>> th{&on_tile};
    pcv_xray_quadtree_info info{};
    check(pcv_xray_quadtree_from_dirs(ctx.raw(), raw.data(), (uint32_t)raw.size(), &params, f.data(), (uint32_t)f.size(), max_device_bytes, &decltype(th)::call,
                                      &th, &info, bounded_info, dir_info));
    return info;
}
// merge_xray_quadtrees: the sub-root builds in `input_dirs` joined into one quadtree in `output_dir` (pcv_xray_merge_quadtrees).
inline pcv_xray_merge_info merge_xray_quadtrees(const Context& ctx, const std::vector<std::string>& input_dirs, const std::string& output_dir,
                                                const std::array<uint8_t, 4>& background = {255, 255, 255, 255}, uint64_t max_device_bytes = 0) {
    std::vector<const char*> raw;
    for (const std::string& d : input_dirs) raw.push_back(d.c_str());
    pcv_xray_merge_info info{};
    check(pcv_xray_merge_quadtrees(ctx.raw(), raw.data(), (uint32_t)raw.size(), output_dir.c_str(), background.data(), max_device_bytes, &info));
    return info;
}
// inpaint_xray_quadtree: the leaves of the quadtree with root (root_level, root_index) in `input_dir` inpainted into
// `output_dir`, their background assigned and the parents rebuilt (pcv_xray_inpaint_quadtree).
inline pcv_xray_inpaint_info inpaint_xray_quadtree(const Context& ctx, const std::string& input_dir, const std::string& output_dir, uint32_t inpaint_distance_px,
                                                   const std::array<uint8_t, 4>& background = {255, 255, 255, 255}, uint8_t root_level = 0,
                                                   uint64_t root_index = 0, uint64_t max_device_bytes = 0) {
    pcv_xray_inpaint_info info{};
    check(pcv_xray_inpaint_quadtree(ctx.raw(), input_dir.c_str(), output_dir.c_str(), root_level, root_index, inpaint_distance_px, background.data(),
                                    max_device_bytes, &info));
    return info;
}
// build_xray_quadtree over the S2 directories `dirs` streamed from disk, none of them ever resident as a whole: the tiles of
// build_xray_quadtree over S2Cells loaded from each of them, in the same order (pcv_s2_xray_quadtree_from_dirs).
template <class F>
pcv_xray_quadtree_info build_xray_quadtree_from_s2_dirs(const Context& ctx, const std::vector<std::string>& dirs, const pcv_xray_quadtree_params& params,
                                                        const std::vector<ClosedInterval>& filter_intervals, F&& on_tile, uint64_t max_device_bytes = 0,
                                                        pcv_xray_bounded_info* bounded_info = nullptr, pcv_xray_dir_info* dir_info = nullptr) {
    std::vector<const char*> raw;
    for (const std::string& d : dirs) raw.push_back(d.c_str());
    const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
    detail::XrayThunk<std::remove_reference_t<F>> th{&on_tile};
    pcv_xray_quadtree_info info{};
    check(pcv_s2_xray_quadtree_from_dirs(ctx.raw(), raw.data(), (uint32_t)raw.size(), &params, f.data(), (uint32_t)f.size(), max_device_bytes,
                                         &decltype(th)::call, &th, &info, bounded_info, dir_info));
    return info;
}

inline bool S2Cells::for_each_batch(const PointQuery& query, size_t batch_size, const std::function<bool(PointsBatch&&)>& func) const {
    const std::vector<pcv_interval> f = detail::raw_intervals(query.filter_intervals);
    return detail::stream_batches(func, [&](pcv_batch_cb cb, void* user) {
        return pcv_s2_query_points(s_, &query.location.raw, f.empty() ? nullptr : f.data(), (uint32_t)f.size(), batch_size, cb, user);
    });
}
inline bool S2Cells::for_each_batch(const CellUnion& cell_union, const std::vector<ClosedInterval>& filter_intervals, size_t batch_size,
                                    const std::function<bool(PointsBatch&&)>& func) const {
    const pcv_cell_union cu = detail::raw_union(cell_union);
    const std::vector<pcv_interval> f = detail::raw_intervals(filter_intervals);
    return detail::stream_batches(func, [&](pcv_batch_cb cb, void* user) {
        return pcv_s2_query_cell_union(s_, &cu, f.empty() ? nullptr : f.data(), (uint32_t)f.size(), batch_size, cb, user);
    });
}

// S2Splitter::with_split_level(level, path, Encoding::Plain, ..) + write(batch)... + get_meta (read_write/s2.rs:33-50,59-125,165-173):
// the batches of one cloud, split by S2 cell on the GPU; throws ("... is not a valid ECEF point") like the writer's Err.
template <class BatchIterator>
inline S2Cells s2_split(Context& ctx, const std::string& output_directory, BatchIterator begin, BatchIterator end, uint32_t split_level = 20) {
    std::vector<std::array<double, 3>> pos;
    std::vector<std::array<uint8_t, 3>> col;
    std::vector<float> inten;
    for (BatchIterator it = begin; it != end; ++it) {
        const PointsBatch& b = *it;
        pos.insert(pos.end(), b.position.begin(), b.position.end());
        col.insert(col.end(), b.color.begin(), b.color.end());
        inten.insert(inten.end(), b.intensity.begin(), b.intensity.end());
    }
    pcv_points pts{};
    const double* base = pos.empty() ? nullptr : pos[0].data();
    pts.x = base;
    pts.y = base ? base + 1 : nullptr;
    pts.z = base ? base + 2 : nullptr;
    pts.stride = 3;
    pts.rgb = col.size() == pos.size() && !col.empty() ? col[0].data() : nullptr;
    pts.intensity = inten.size() == pos.size() && !inten.empty() ? inten.data() : nullptr;
    pts.n = pos.size();
    pcv_s2cloud* s = nullptr;
    check(pcv_s2_build(ctx.raw(), &pts, split_level, &s));
    S2Cells cloud(s);
    if (!output_directory.empty()) cloud.write_to_directory(output_directory);
    return cloud;
}

// ParallelIterator::new(point_clouds, query, batch_size, num_threads, buffer_size).try_for_each_batch(func) — iterator.rs:238-257.
// num_threads / buffer_size are accepted for signature parity; the GPU path streams on the caller's thread.
class ParallelIterator {
   public:
    ParallelIterator(const std::vector<const Octree*>& point_clouds, const PointQuery& query, size_t batch_size, size_t /*num_threads*/ = 1,
                     size_t /*buffer_size*/ = 4)
        : clouds_(point_clouds), query_(query), batch_size_(batch_size) {}
    // func returns true to continue, false to stop (== Err).  Returns true if every batch was consumed.
    bool try_for_each_batch(const std::function<bool(PointsBatch&&)>& func) {
        struct State {
            const std::function<bool(PointsBatch&&)>* f;
        } st{&func};
        auto tramp = [](void* user, const pcv_batch* b) -> int {
            State* s = (State*)user;
            return (*s->f)(batch_from(b)) ? 0 : 1;
        };
        std::vector<pcv_interval> f;
        for (auto& iv : query_.filter_intervals) f.push_back(pcv_interval{iv.lower_bound, iv.upper_bound});
        for (const Octree* o : clouds_) {
            const int rc = pcv_query_points(o->raw(), &query_.location.raw, f.empty() ? nullptr : f.data(), (uint32_t)f.size(), batch_size_, tramp, &st);
            if (rc == PCV_ERR_CANCELLED) return false;
            check(rc);
        }
        return true;
    }

   private:
    std::vector<const Octree*> clouds_;
    PointQuery query_;
    size_t batch_size_;
};

}  // namespace pcv
