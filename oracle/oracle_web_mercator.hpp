// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_core.hpp header).
//
// PointLocation::WebMercatorRect restated from src/math/web_mercator.rs and src/geometry/web_mercator_rect.rs: the constructor,
// the ECEF -> WGS84 -> map point test, the extruded polyhedron, node selection and the filtered point query of one octree.
// The reference converts through the un-vendored nav-types crate; here ECEF -> WGS84 is Heikkinen's closed form and WGS84 ->
// ECEF the textbook prime-vertical form over WGS84's a and 1/f, in the operation order of the product (csrc/geometry_host.hpp),
// so that both give the same doubles with the same libm.
#pragma once
#include <cmath>
#include <deque>

#include "oracle_query.hpp"

namespace orc {
namespace wm {

const double A = 6378137.0;  // WGS84 semi-major axis and flattening
const double F = 1.0 / 298.257223563;
const double B = A * (1.0 - F);
const double E2 = 1.0 - (B * B) / (A * A);
const double PI = 3.14159265358979323846;
const double FRAC_1_PI = 0.31830988618379067153776752674503;
const double LAT_BOUND_RAD = 1.4844222297453324;  // web_mercator.rs:9-13
const double LAT_BOUND_SIN = 0.99627207622075;
const unsigned MAX_ZOOM = 23;
const double MIN_ELEVATION_M = -500.0;  // web_mercator_rect.rs:11-26
const double MAX_ELEVATION_M = 10000.0;

inline double clamp(double v, double lo, double hi) { return v > lo ? (v < hi ? v : hi) : lo; }  // nalgebra::clamp

struct LatLng {
    double lat, lng;
};

// ECEF -> WGS84 (height dropped): Heikkinen 1982.
inline LatLng from_ecef(Vec3 p) {
    const double a2 = A * A, b2 = B * B, ep2 = (a2 - b2) / b2;
    const double r2 = p.x * p.x + p.y * p.y, r = std::sqrt(r2), z2 = p.z * p.z;
    const double f = 54.0 * b2 * z2;
    const double g = r2 + (1.0 - E2) * z2 - E2 * (a2 - b2);
    const double c = E2 * E2 * f * r2 / (g * g * g);
    const double s = std::cbrt(1.0 + c + std::sqrt(c * c + 2.0 * c));
    const double k = s + 1.0 / s + 1.0;
    const double pp = f / (3.0 * k * k * g * g);
    const double q = std::sqrt(1.0 + 2.0 * E2 * E2 * pp);
    // the radicand is 0 on the polar axis in exact arithmetic and may round below it there
    const double r0 = -(pp * E2 * r) / (1.0 + q) + std::sqrt(std::fmax(0.5 * a2 * (1.0 + 1.0 / q) - pp * (1.0 - E2) * z2 / (q * (1.0 + q)) - 0.5 * pp * r2, 0.0));
    const double t = r - E2 * r0;
    const double v = std::sqrt(t * t + (1.0 - E2) * z2);
    const double z0 = b2 * p.z / (A * v);
    return {std::atan((p.z + ep2 * z0) / r), std::atan2(p.y, p.x)};
}

// WGS84 -> ECEF
inline Vec3 to_ecef(double lat, double lng, double h) {
    const double sl = std::sin(lat), cl = std::cos(lat);
    const double n = A / std::sqrt(1.0 - E2 * sl * sl);
    return {(n + h) * cl * std::cos(lng), (n + h) * cl * std::sin(lng), (n * (1.0 - E2) + h) * sl};
}

struct Coord {  // WebMercatorCoord: normalised to [0, 1)
    double x, y;
};

inline Coord from_lat_lng(LatLng ll) {  // web_mercator.rs:38-50
    const double lat = clamp(ll.lat, -LAT_BOUND_RAD, LAT_BOUND_RAD);
    const double sin_y = std::sin(lat);
    return {0.5 + ll.lng / (2.0 * PI), 0.5 - std::log((1.0 + sin_y) / (1.0 - sin_y)) * (0.25 * FRAC_1_PI)};
}

inline LatLng to_lat_lng(Coord c) {  // web_mercator.rs:55-64
    const double cx = c.x - 0.5, cy = c.y - 0.5;
    const double sin_term = std::exp(-cy * (4.0 * PI));
    const double one_over_sin_y = (sin_term + 1.0) * -0.5;
    double sin_y = (1.0 / one_over_sin_y) + 1.0;
    sin_y = clamp(sin_y, -LAT_BOUND_SIN, LAT_BOUND_SIN);
    const double lng = clamp(cx * (2.0 * PI), -PI, PI);
    return {std::asin(sin_y), lng};
}

inline bool from_zoomed_coordinate(double x, double y, unsigned z, Coord& out) {  // web_mercator.rs:84-97
    if (z > MAX_ZOOM || std::fmin(x, y) < 0.0) return false;
    const double zoom = (double)(256u << z);
    if (!(std::fmax(x, y) < zoom)) return false;
    out = {x / zoom, y / zoom};
    return true;
}

struct Rect {
    Coord north_west, south_east;

    // web_mercator_rect.rs:40-53; non-finite input is rejected too (nalgebra's min / max would skip a NaN)
    static bool from_zoomed_coordinates(const double mn[2], const double mx[2], unsigned z, Rect& out) {
        for (int i = 0; i < 2; ++i)
            if (!std::isfinite(mn[i]) || !std::isfinite(mx[i])) return false;
        Rect r;
        if (!from_zoomed_coordinate(mn[0], mn[1], z, r.north_west) || !from_zoomed_coordinate(mx[0], mx[1], z, r.south_east)) return false;
        const double div = (double)(1u << z);
        const double dx = (mx[0] - mn[0]) / div, dy = (mx[1] - mn[1]) / div;
        double rx = std::fmod(dx, 256.0);  // rem_euclid
        if (rx < 0.0) rx += 256.0;
        if (rx > 1.0 || dy > 1.0 || dy < 0.0) return false;
        out = r;
        return true;
    }

    bool contains(Vec3 p) const {  // web_mercator_rect.rs:121-127, component-wise partial_le / partial_lt
        const Coord w = from_lat_lng(from_ecef(p));
        return north_west.x <= w.x && north_west.y <= w.y && w.x < south_east.x && w.y < south_east.y;
    }

    Intersector intersector() const {  // web_mercator_rect.rs:60-119
        const LatLng nw = to_lat_lng(north_west), se = to_lat_lng(south_east);
        Intersector r;
        r.corners[0] = to_ecef(nw.lat, nw.lng, MIN_ELEVATION_M);  // NW down
        r.corners[1] = to_ecef(nw.lat, se.lng, MIN_ELEVATION_M);  // NE down
        r.corners[2] = to_ecef(se.lat, se.lng, MIN_ELEVATION_M);  // SE down
        r.corners[3] = to_ecef(se.lat, nw.lng, MIN_ELEVATION_M);  // SW down
        r.corners[4] = to_ecef(nw.lat, nw.lng, MAX_ELEVATION_M);  // NW up
        r.corners[5] = to_ecef(nw.lat, se.lng, MAX_ELEVATION_M);  // NE up
        r.corners[6] = to_ecef(se.lat, se.lng, MAX_ELEVATION_M);  // SE up
        r.corners[7] = to_ecef(se.lat, nw.lng, MAX_ELEVATION_M);  // SW up
        const Vec3* c = r.corners;
        r.edges = {normalize(c[1] - c[0]), normalize(c[2] - c[1]), normalize(c[3] - c[2]), normalize(c[0] - c[3]),
                   normalize(c[5] - c[4]), normalize(c[6] - c[5]), normalize(c[7] - c[6]), normalize(c[4] - c[7]),
                   normalize(c[4] - c[0]), normalize(c[5] - c[1]), normalize(c[6] - c[2]), normalize(c[7] - c[3])};
        const std::vector<Vec3>& e = r.edges;
        r.face_normals = {normalize(cross(e[0], e[8])), normalize(cross(e[1], e[9])), normalize(cross(e[2], e[10])),
                          normalize(cross(e[3], e[11])), normalize(cross(e[1], e[0])), normalize(cross(e[5], e[4]))};
        return r;
    }
};

// Intersector::intersect (sat.rs:146-152): how `b` relates to `a`.
inline Relation intersect(const Intersector& a, const Intersector& b) {
    return sat(separating_axes(a, b.edges, b.face_normals), a.corners, 8, b.corners, 8);
}

// nodes_in_location (octree/mod.rs:309-323, octree_iterator.rs:30-43) with the rect's cached axes.
inline std::vector<NodeId> nodes_in_rect(const Octree& oct, const Rect& rect) {
    const CachedAxesIntersector isec = cache_separating_axes_for_aabb(rect.intersector());
    std::vector<NodeId> out;
    std::deque<NodeId> q;
    q.push_back(NodeId());
    while (!q.empty()) {
        NodeId cur = q.front();
        q.pop_front();
        auto it = oct.nodes.find(cur);
        if (it == oct.nodes.end()) continue;
        Vec3 c[8];
        it->second.cube.to_aabb().corners(c);
        if (isec.intersect(c, 8) != REL_OUT) {
            for (unsigned k = 0; k < 8; ++k) {
                NodeId ch = cur.child(k);
                if (oct.nodes.count(ch)) q.push_back(ch);
            }
            out.push_back(cur);
        }
    }
    return out;
}

// FilteredIterator (iterator.rs:96-119) over one node: query_node of oracle_query.hpp with the rect as PointCulling.
inline void query_node_rect(const Octree& oct, NodeId id, const Rect& rect, const std::vector<Interval>& filters, QueryOut& out) {
    auto it = oct.files.find(id);
    if (it == oct.files.end()) return;
    const NodeFile& f = it->second;
    const size_t n = (size_t)f.num_points();
    for (size_t i = 0; i < n; ++i) {
        Point pt = node_read(f, i, oct.with_intensity);
        bool keep = rect.contains(pt.p);
        for (auto& fi : filters) {
            const double v = (double)pt.intensity;
            keep = keep && (fi.lo <= v && v <= fi.hi);
        }
        if (!keep) continue;
        out.xyz.insert(out.xyz.end(), {pt.p.x, pt.p.y, pt.p.z});
        out.rgb.insert(out.rgb.end(), {pt.rgb[0], pt.rgb[1], pt.rgb[2]});
        if (oct.with_intensity) out.intensity.push_back(pt.intensity);
        out.src.push_back(pt.src);
    }
}

}  // namespace wm
}  // namespace orc
