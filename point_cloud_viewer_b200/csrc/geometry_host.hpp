// geometry_host.hpp — per-query setup of the culling geometry (host, runs once per location):
// corners, edges, face normals and the cached, de-duplicated separating axes that the CUDA SAT
// kernel then applies to every octree node.
//   Frustum corners/edges/normals   src/geometry/frustum.rs:129-166
//   Obb corners/edges               src/geometry/obb.rs:49-78
//   Aabb fast path (3 unit axes)    src/geometry/aabb.rs:103-111
//   WebMercatorRect                 src/geometry/web_mercator_rect.rs:40-127, src/math/web_mercator.rs:38-97
//   axis generation + O(n^2) dedup  src/math/sat.rs:80-143
//   Matrix4::transform_point        nalgebra 0.22 (column-by-column accumulation, divide by w if != 0)
#pragma once
#include <cmath>
#include <cstring>
#include <limits>
#include <stdexcept>

#include "../../include/pcv.h"
#include "s2.h"

namespace pcv {

struct V3 {
    double x, y, z;
};
#if defined(__CUDACC__)
#define PCV_GHD __host__ __device__ inline
#else
#define PCV_GHD inline
#endif

PCV_GHD V3 v3sub(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
PCV_GHD V3 v3add(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
PCV_GHD double v3dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
PCV_GHD V3 v3cross(V3 a, V3 b) { return V3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

// m: column-major 4x4.  (M3x3 * p + t) / (r3 . p + m33) unless the normaliser is exactly zero.
PCV_GHD V3 mat4_transform_point(const double* m, V3 p) {
    double n = m[3] * p.x;
    n = n + m[7] * p.y;
    n = n + m[11] * p.z;
    n = n + m[15];
    double r[3];
    for (int i = 0; i < 3; ++i) {
        double a = m[i] * p.x;
        a = m[4 + i] * p.y + a;
        a = m[8 + i] * p.z + a;
        r[i] = a + m[12 + i];
    }
    if (n != 0.0) return V3{r[0] / n, r[1] / n, r[2] / n};
    return V3{r[0], r[1], r[2]};
}

// UnitQuaternion * Vector3 and Isometry3 * Point3 (iso = tx,ty,tz,qi,qj,qk,qw)
PCV_GHD V3 quat_rot(const double* iso7, V3 p) {
    const V3 qv{iso7[3], iso7[4], iso7[5]};
    V3 t = v3cross(qv, p);
    t = V3{t.x * 2.0, t.y * 2.0, t.z * 2.0};
    const V3 c = v3cross(qv, t);
    const double w = iso7[6];
    return V3{t.x * w + c.x + p.x, t.y * w + c.y + p.y, t.z * w + c.z + p.z};
}
PCV_GHD V3 iso_apply(const double* iso7, V3 p) {
    const V3 r = quat_rot(iso7, p);
    return V3{r.x + iso7[0], r.y + iso7[1], r.z + iso7[2]};
}

// ---- Web Mercator (src/math/web_mercator.rs) over the WGS84 ellipsoid ----------------------------------------------------
// WGS84's defining semi-major axis and flattening; the semi-minor axis and the first eccentricity squared follow from them.
constexpr double kWgs84A = 6378137.0;
constexpr double kWgs84F = 1.0 / 298.257223563;
constexpr double kWgs84B = kWgs84A * (1.0 - kWgs84F);
constexpr double kWgs84E2 = 1.0 - (kWgs84B * kWgs84B) / (kWgs84A * kWgs84A);
constexpr double kPi = 3.14159265358979323846;                // std::f64::consts::PI
constexpr double kFrac1Pi = 0.31830988618379067153776752674503; // std::f64::consts::FRAC_1_PI
constexpr double kWmLatBoundRad = 1.4844222297453324;          // LAT_BOUND_RAD: 2 atan(e^pi) - pi/2, 85.051129 degrees
constexpr double kWmLatBoundSin = 0.99627207622075;            // LAT_BOUND_SIN = sin(LAT_BOUND_RAD)
constexpr uint32_t kWmMaxZoom = 23;                            // MAX_ZOOM: 256 << z fits a u32
constexpr double kWmMinElevation = -500.0;                     // the rect's extrusion, web_mercator_rect.rs:11-26
constexpr double kWmMaxElevation = 10000.0;

// nalgebra::clamp: min for NaN.
PCV_GHD double wm_clamp(double v, double lo, double hi) { return v > lo ? (v < hi ? v : hi) : lo; }

// ECEF -> WGS84 latitude and longitude (radians), the closed form of Heikkinen (1982) that the conversion literature calls
// "Ferrari's solution"; the height is not needed.  Shared by the cull kernels and the host.
PCV_GHD void ecef_to_lat_lng(double x, double y, double z, double& lat, double& lng) {
    const double a2 = kWgs84A * kWgs84A, b2 = kWgs84B * kWgs84B, e2 = kWgs84E2, ep2 = (a2 - b2) / b2;
    const double r2 = x * x + y * y, r = sqrt(r2), z2 = z * z;
    const double f = 54.0 * b2 * z2;
    const double g = r2 + (1.0 - e2) * z2 - e2 * (a2 - b2);
    const double c = e2 * e2 * f * r2 / (g * g * g);
    const double s = cbrt(1.0 + c + sqrt(c * c + 2.0 * c));
    const double k = s + 1.0 / s + 1.0;
    const double p = f / (3.0 * k * k * g * g);
    const double q = sqrt(1.0 + 2.0 * e2 * e2 * p);
    // the radicand is 0 on the polar axis in exact arithmetic and may round below it there
    const double r0 = -(p * e2 * r) / (1.0 + q) + sqrt(fmax(0.5 * a2 * (1.0 + 1.0 / q) - p * (1.0 - e2) * z2 / (q * (1.0 + q)) - 0.5 * p * r2, 0.0));
    const double t = r - e2 * r0;
    const double v = sqrt(t * t + (1.0 - e2) * z2);
    const double z0 = b2 * z / (kWgs84A * v);
    lat = atan((z + ep2 * z0) / r);
    lng = atan2(y, x);
}

// WebMercatorCoord::from_lat_lng (web_mercator.rs:38-50): the normalised map position in [0, 1)^2 (x east, y south).
PCV_GHD void web_mercator_from_lat_lng(double lat, double lng, double w[2]) {
    const double sin_y = sin(wm_clamp(lat, -kWmLatBoundRad, kWmLatBoundRad));
    w[0] = 0.5 + lng / (2.0 * kPi);
    w[1] = 0.5 - log((1.0 + sin_y) / (1.0 - sin_y)) * (0.25 * kFrac1Pi);
}

// WebMercatorRect::contains (web_mercator_rect.rs:121-127): the point's map position lies in [nw, se) component by component,
// so a rect that wraps the antimeridian (nw.x > se.x) holds no point.  The point's altitude plays no part.
PCV_GHD bool web_mercator_rect_contains(const double nw[2], const double se[2], double x, double y, double z) {
    double lat, lng, w[2];
    ecef_to_lat_lng(x, y, z, lat, lng);
    web_mercator_from_lat_lng(lat, lng, w);
    return nw[0] <= w[0] && nw[1] <= w[1] && w[0] < se[0] && w[1] < se[1];
}

// The kind of a QueryGeom built from a cell union (PointLocation::S2Cells, src/iterator.rs:13-20).  Internal: pcv_location has no
// such kind; the cell-union entry points build the geometry themselves.
constexpr int32_t kLocCellUnion = 16;

// The most separating axes a location caches against an Aabb (sat.rs:111-142): 6 face normals, the 3 unit axes and the 12 x 3
// edge cross products of a polyhedron with 12 edges (the Web Mercator rect's extrusion).
constexpr int kMaxAxes = 6 + 3 + 12 * 3;
// The axes a QueryGeom holds itself: every Aabb, Obb and Frustum (at most 5 + 3 + 6 x 3).  A Web Mercator rect's axes past these
// live in a table its record points to (like a cell union's ids), so the record - one per location in every selection, X-ray
// leaves included - keeps its size, and so do the projection tables (LocProj) and the kernels' shared-memory copies of them.
constexpr int kInlineAxes = 26;
struct MoreAxes {
    double a[kMaxAxes - kInlineAxes][3];
    double proj[kMaxAxes - kInlineAxes][2];  // the location's own projections on them (project_location_axis)
};

// What the device needs per location.
struct QueryGeom {
    int32_t kind;
    int32_t naxes;       // cached separating axes (<= kMaxAxes; past kInlineAxes in more_axes); 0 for AllPoints and cell unions
    double axes[kInlineAxes][3];
    double corners[8][3];
    double aabb_min[3], aabb_max[3];  // Web Mercator rect: north_west in aabb_min[0..1], south_east in aabb_max[0..1], as given
    double clip_from_query[16];
    double obb_from_query[7];
    double half_extent[3];
    union {
        const uint64_t* cells;      // cell union: its normalised ids (device) ...
        const MoreAxes* more_axes;  // Web Mercator rect: its axes kInlineAxes.. (device for the kernels, host on the host)
    };
    const S2Square* squares;   // ... and each one's face and square of leaf cells (device)
    uint32_t ncells, pad;
};

// Cached axis k of a location.
PCV_GHD const double* geom_axis(const QueryGeom& g, int k) { return k < kInlineAxes ? g.axes[k] : g.more_axes->a[k - kInlineAxes]; }
// The location's own projection on its axis k (project_location of query.cuh, one axis).
PCV_GHD void project_location_axis(const QueryGeom& g, int k, double& lo, double& hi) {
    const double* ax = geom_axis(g, k);
    lo = 1.7976931348623157e308;
    hi = -1.7976931348623157e308;
    for (int i = 0; i < 8; ++i) {
        const double p = g.corners[i][0] * ax[0] + g.corners[i][1] * ax[1] + g.corners[i][2] * ax[2];
        lo = fmin(lo, p);
        hi = fmax(hi, p);
    }
}

inline V3 unit(V3 v) {
    const double n = std::sqrt(v3dot(v, v));
    return V3{v.x / n, v.y / n, v.z / n};
}

struct PolyIntersector {
    V3 corners[8];
    V3 edges[12];
    int nedges = 0;
    V3 normals[6];
    int nnormals = 0;
};

inline PolyIntersector frustum_intersector(const double* query_from_clip) {
    PolyIntersector r;
    int i = 0;
    for (int sx = -1; sx <= 1; sx += 2)
        for (int sy = -1; sy <= 1; sy += 2)
            for (int sz = -1; sz <= 1; sz += 2) r.corners[i++] = mat4_transform_point(query_from_clip, V3{(double)sx, (double)sy, (double)sz});
    const V3* c = r.corners;
    r.edges[0] = unit(v3sub(c[4], c[0]));
    r.edges[1] = unit(v3sub(c[2], c[0]));
    r.edges[2] = unit(v3sub(c[1], c[0]));
    r.edges[3] = unit(v3sub(c[3], c[2]));
    r.edges[4] = unit(v3sub(c[5], c[4]));
    r.edges[5] = unit(v3sub(c[7], c[6]));
    r.nedges = 6;
    r.normals[0] = unit(v3cross(r.edges[0], r.edges[1]));
    r.normals[1] = unit(v3cross(r.edges[0], r.edges[2]));
    r.normals[2] = unit(v3cross(r.edges[0], r.edges[3]));
    r.normals[3] = unit(v3cross(r.edges[1], r.edges[2]));
    r.normals[4] = unit(v3cross(r.edges[1], r.edges[4]));
    r.nnormals = 5;
    return r;
}

inline PolyIntersector obb_intersector(const double* query_from_obb, const double* h) {
    PolyIntersector r;
    for (int i = 0; i < 8; ++i) {
        const V3 l{(i & 1) ? h[0] : -h[0], (i & 2) ? h[1] : -h[1], (i & 4) ? h[2] : -h[2]};
        r.corners[i] = iso_apply(query_from_obb, l);
    }
    r.edges[0] = unit(quat_rot(query_from_obb, V3{1, 0, 0}));
    r.edges[1] = unit(quat_rot(query_from_obb, V3{0, 1, 0}));
    r.edges[2] = unit(quat_rot(query_from_obb, V3{0, 0, 1}));
    r.nedges = 3;
    for (int i = 0; i < 3; ++i) r.normals[i] = r.edges[i];
    r.nnormals = 3;
    return r;
}

// WebMercatorCoord::to_lat_lng (web_mercator.rs:55-64).
inline void web_mercator_to_lat_lng(const double w[2], double& lat, double& lng) {
    const double cx = w[0] - 0.5, cy = w[1] - 0.5;
    const double sin_term = std::exp(-cy * (4.0 * kPi));
    const double one_over_sin_y = (sin_term + 1.0) * -0.5;
    const double sin_y = wm_clamp(1.0 / one_over_sin_y + 1.0, -kWmLatBoundSin, kWmLatBoundSin);
    lng = wm_clamp(cx * (2.0 * kPi), -kPi, kPi);
    lat = std::asin(sin_y);
}

// WGS84 (latitude, longitude, height) -> ECEF.
inline V3 wgs84_to_ecef(double lat, double lng, double h) {
    const double sl = std::sin(lat), cl = std::cos(lat);
    const double n = kWgs84A / std::sqrt(1.0 - kWgs84E2 * sl * sl);
    return V3{(n + h) * cl * std::cos(lng), (n + h) * cl * std::sin(lng), (n * (1.0 - kWgs84E2) + h) * sl};
}

// A Web Mercator rect as the constructor leaves it (web_mercator_rect.rs:40-53, web_mercator.rs:84-97): both corners in
// [0, 1), se.y >= nw.y, and at most one zoom-0 pixel across, where x may wrap around the antimeridian.  NaN fails.
inline bool web_mercator_rect_valid(const double nw[2], const double se[2]) {
    for (int i = 0; i < 2; ++i)
        if (!(nw[i] >= 0.0 && nw[i] < 1.0 && se[i] >= 0.0 && se[i] < 1.0)) return false;
    // (max - min) / 2^z of the constructor, exactly: its corners are these times 256 * 2^z
    const double dx = (se[0] - nw[0]) * 256.0, dy = (se[1] - nw[1]) * 256.0;
    double rx = std::fmod(dx, 256.0);  // f64::rem_euclid
    if (rx < 0.0) rx += 256.0;
    return !(rx > 1.0 || dy > 1.0 || dy < 0.0);
}

// WebMercatorRect::from_zoomed_coordinates: false where the reference returns None, and for non-finite input.
inline bool web_mercator_rect_from_zoomed(const double mn[2], const double mx[2], uint32_t z, double nw[2], double se[2]) {
    if (z > kWmMaxZoom) return false;
    const double zoom = (double)(256u << z);
    for (int i = 0; i < 2; ++i) {
        nw[i] = mn[i] / zoom;  // powers of two: exact
        se[i] = mx[i] / zoom;
    }
    return web_mercator_rect_valid(nw, se);
}

// WebMercatorRect::intersector (web_mercator_rect.rs:60-119): the rect's corners extruded from -500 m to 10 km, NW NE SE SW down,
// then up; 12 edges and 6 face normals.
inline PolyIntersector web_mercator_intersector(const double nw[2], const double se[2]) {
    PolyIntersector r;
    double nlat, nlng, slat, slng;
    web_mercator_to_lat_lng(nw, nlat, nlng);
    web_mercator_to_lat_lng(se, slat, slng);
    for (int u = 0; u < 2; ++u) {
        const double h = u ? kWmMaxElevation : kWmMinElevation;
        r.corners[4 * u + 0] = wgs84_to_ecef(nlat, nlng, h);
        r.corners[4 * u + 1] = wgs84_to_ecef(nlat, slng, h);
        r.corners[4 * u + 2] = wgs84_to_ecef(slat, slng, h);
        r.corners[4 * u + 3] = wgs84_to_ecef(slat, nlng, h);
    }
    const V3* c = r.corners;
    for (int u = 0; u < 2; ++u)
        for (int i = 0; i < 4; ++i) r.edges[4 * u + i] = unit(v3sub(c[4 * u + (i + 1) % 4], c[4 * u + i]));  // N E S W, down then up
    for (int i = 0; i < 4; ++i) r.edges[8 + i] = unit(v3sub(c[4 + i], c[i]));                             // NW NE SE SW, upward
    r.nedges = 12;
    const V3* e = r.edges;
    for (int i = 0; i < 4; ++i) r.normals[i] = unit(v3cross(e[i], e[8 + i]));  // N E S W faces
    r.normals[4] = unit(v3cross(e[1], e[0]));                                  // down
    r.normals[5] = unit(v3cross(e[5], e[4]));                                  // up
    r.nnormals = 6;
    return r;
}

// Intersector::cache_separating_axes_for_aabb: [own normals, x,y,z, normalize(edge_i x unit_j) if finite], then dedup.
// Axes past kInlineAxes go to `more` (g.more_axes points to it); only a Web Mercator rect has them.
inline void cache_axes_for_aabb(const PolyIntersector& p, QueryGeom& g, MoreAxes* more = nullptr) {
    V3 all[6 + 3 + 36];
    int n = 0;
    const V3 units[3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int i = 0; i < p.nnormals; ++i) all[n++] = p.normals[i];
    for (int j = 0; j < 3; ++j) all[n++] = units[j];
    for (int i = 0; i < p.nedges; ++i)
        for (int j = 0; j < 3; ++j) {
            const V3 c = unit(v3cross(p.edges[i], units[j]));
            if (std::isfinite(c.x) && std::isfinite(c.y) && std::isfinite(c.z)) all[n++] = c;
        }
    g.naxes = 0;
    g.more_axes = more;
    for (int i = 0; i < n; ++i) {
        bool dupe = false;
        for (int k = 0; k < g.naxes && !dupe; ++k) {
            const double* a = geom_axis(g, k);
            const V3 o{a[0], a[1], a[2]};
            const V3 dm = v3sub(all[i], o), dp = v3add(all[i], o);
            dupe = std::fmin(v3dot(dm, dm), v3dot(dp, dp)) < std::numeric_limits<double>::epsilon();
        }
        if (!dupe) {
            if (g.naxes >= kInlineAxes && !more) throw std::logic_error("a location with more than kInlineAxes axes and no table for them");
            double* a = g.naxes < kInlineAxes ? g.axes[g.naxes] : more->a[g.naxes - kInlineAxes];
            a[0] = all[i].x;
            a[1] = all[i].y;
            a[2] = all[i].z;
            ++g.naxes;
        }
    }
    for (int i = 0; i < 8; ++i) {
        g.corners[i][0] = p.corners[i].x;
        g.corners[i][1] = p.corners[i].y;
        g.corners[i][2] = p.corners[i].z;
    }
    for (int k = kInlineAxes; k < g.naxes; ++k) project_location_axis(g, k, more->proj[k - kInlineAxes][0], more->proj[k - kInlineAxes][1]);
}

// `more` holds a Web Mercator rect's axes past kInlineAxes (required for that kind, unused for the others).
inline QueryGeom make_query_geom(const pcv_location& loc, MoreAxes* more = nullptr) {
    QueryGeom g;
    std::memset(&g, 0, sizeof g);
    g.kind = loc.kind;
    for (int a = 0; a < 3; ++a) {
        g.aabb_min[a] = std::fmin(loc.aabb_min[a], loc.aabb_max[a]);
        g.aabb_max[a] = std::fmax(loc.aabb_min[a], loc.aabb_max[a]);
        g.half_extent[a] = loc.half_extent[a];
    }
    std::memcpy(g.clip_from_query, loc.clip_from_query, sizeof g.clip_from_query);
    std::memcpy(g.obb_from_query, loc.obb_from_query, sizeof g.obb_from_query);
    if (loc.kind == PCV_LOC_AABB) {
        g.naxes = 3;
        for (int j = 0; j < 3; ++j) g.axes[j][j] = 1.0;
        for (int i = 0; i < 8; ++i) {  // aabb.rs:114-125: x fastest
            g.corners[i][0] = (i & 1) ? g.aabb_max[0] : g.aabb_min[0];
            g.corners[i][1] = (i & 2) ? g.aabb_max[1] : g.aabb_min[1];
            g.corners[i][2] = (i & 4) ? g.aabb_max[2] : g.aabb_min[2];
        }
    } else if (loc.kind == PCV_LOC_FRUSTUM) {
        cache_axes_for_aabb(frustum_intersector(loc.query_from_clip), g);
    } else if (loc.kind == PCV_LOC_OBB) {
        cache_axes_for_aabb(obb_intersector(loc.query_from_obb, loc.half_extent), g);
    } else if (loc.kind == PCV_LOC_WEB_MERCATOR_RECT) {
        for (int a = 0; a < 3; ++a) {  // unsorted: a rect that wraps the antimeridian stays wrapped
            g.aabb_min[a] = loc.aabb_min[a];
            g.aabb_max[a] = loc.aabb_max[a];
        }
        cache_axes_for_aabb(web_mercator_intersector(loc.aabb_min, loc.aabb_max), g, more);
    }
    return g;
}

// The separating-axis test of a location against an arbitrary box [mn, mx] (the point box of an S2 cell, s2_api.inl): sat()
// of sat.rs:174-194 over the location's cached axes, the box's 8 corners in the Aabb order (x fastest, aabb.rs:114-125), exactly
// as sat_cube (query.cuh) tests a node cube, whose max is min + edge.  Shared by the device kernels and the test backend.
PCV_GHD void project_box(const double mn[3], const double mx[3], const double ax[3], double& lo, double& hi) {
    lo = 1.7976931348623157e308;
    hi = -1.7976931348623157e308;
    for (int i = 0; i < 8; ++i) {
        const double cx = (i & 1) ? mx[0] : mn[0], cy = (i & 2) ? mx[1] : mn[1], cz = (i & 4) ? mx[2] : mn[2];
        const double p = cx * ax[0] + cy * ax[1] + cz * ax[2];
        lo = fmin(lo, p);
        hi = fmax(hi, p);
    }
}
// kS2RelIn / kS2RelCross / kS2RelOut; aproj[k] = project_location_axis(g, k) for k < kInlineAxes, a Web Mercator rect's table
// holds the projections on its further axes.  The relation does not depend on the order of the axes.
PCV_GHD int sat_box(const QueryGeom& g, const double (*aproj)[2], const double mn[3], const double mx[3]) {
    int rel = kS2RelIn;
    const int ni = g.naxes < kInlineAxes ? g.naxes : kInlineAxes;
    for (int k = 0; k < ni; ++k) {
        double bmin, bmax;
        project_box(mn, mx, g.axes[k], bmin, bmax);
        const double amin = aproj[k][0], amax = aproj[k][1];
        if (bmin > amax || bmax < amin) return kS2RelOut;
        if (amin > bmin || bmax > amax) rel = kS2RelCross;
    }
    for (int k = 0; k < g.naxes - kInlineAxes; ++k) {
        double bmin, bmax;
        project_box(mn, mx, g.more_axes->a[k], bmin, bmax);
        const double amin = g.more_axes->proj[k][0], amax = g.more_axes->proj[k][1];
        if (bmin > amax || bmax < amin) return kS2RelOut;
        if (amin > bmin || bmax > amax) rel = kS2RelCross;
    }
    return rel;
}

// The location of an X-ray tile with box [tmin, tmax]: Aabb(bbox), or Obb::from(bbox).transformed(query_from_global.inverse())
// (xray generation.rs:471-477).
inline pcv_location xray_location(const double tmin[3], const double tmax[3], const double* qfg) {
    pcv_location loc{};
    double bmin[3], bmax[3];
    for (int a = 0; a < 3; ++a) {
        bmin[a] = std::fmin(tmin[a], tmax[a]);
        bmax[a] = std::fmax(tmin[a], tmax[a]);
    }
    if (qfg) {
        loc.kind = PCV_LOC_OBB;
        double ginv[7];  // global_from_query = query_from_global.inverse(): conjugate, t' = rot_inv * (-t)
        ginv[3] = -qfg[3];
        ginv[4] = -qfg[4];
        ginv[5] = -qfg[5];
        ginv[6] = qfg[6];
        const V3 nt = quat_rot(ginv, V3{-qfg[0], -qfg[1], -qfg[2]});
        ginv[0] = nt.x;
        ginv[1] = nt.y;
        ginv[2] = nt.z;
        // Obb::from(&aabb): centre = (min+max)*0.5, half = diag*0.5 (obb.rs:19-26); composed with the identity rotation
        const V3 centre{(bmin[0] + bmax[0]) * 0.5, (bmin[1] + bmax[1]) * 0.5, (bmin[2] + bmax[2]) * 0.5};
        const V3 sh = quat_rot(ginv, centre);
        double* q = loc.query_from_obb;
        q[0] = ginv[0] + sh.x;
        q[1] = ginv[1] + sh.y;
        q[2] = ginv[2] + sh.z;
        q[3] = ginv[3];
        q[4] = ginv[4];
        q[5] = ginv[5];
        q[6] = ginv[6];
        double* qi = loc.obb_from_query;
        qi[3] = -q[3];
        qi[4] = -q[4];
        qi[5] = -q[5];
        qi[6] = q[6];
        const V3 it = quat_rot(qi, V3{-q[0], -q[1], -q[2]});
        qi[0] = it.x;
        qi[1] = it.y;
        qi[2] = it.z;
        for (int a = 0; a < 3; ++a) loc.half_extent[a] = (bmax[a] - bmin[a]) * 0.5;
    } else {
        loc.kind = PCV_LOC_AABB;
        for (int a = 0; a < 3; ++a) {
            loc.aabb_min[a] = bmin[a];
            loc.aabb_max[a] = bmax[a];
        }
    }
    return loc;
}

// 4x4 inverse by cofactors (the formula nalgebra's try_inverse uses for 4x4); false if det == 0.
inline bool mat4_try_inverse(const double* m, double* out) {
    double inv[16];
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const double det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    if (det == 0.0) return false;
    const double inv_det = 1.0 / det;
    for (int i = 0; i < 16; ++i) out[i] = inv[i] * inv_det;
    return true;
}

}  // namespace pcv
