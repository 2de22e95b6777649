// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_core.hpp header).
// C interface of oracle_web_mercator.hpp for tests/ (ctypes), built by the tests into liboracle_wm.so.  It compiles the oracle's
// own C interface too, so an octree handle of liboracle.so (same sources, same flags) is a Handle here.
// A rect is passed as nw_se[4] = north_west.x, north_west.y, south_east.x, south_east.y (normalised), as the constructor
// leaves it or set by hand.
#include "oracle_capi.cpp"
#include "oracle_web_mercator.hpp"

using namespace orc;

static wm::Rect rect_of(const double* nw_se) { return wm::Rect{{nw_se[0], nw_se[1]}, {nw_se[2], nw_se[3]}}; }

extern "C" {

// WebMercatorRect::from_zoomed_coordinates: 1 and nw_se_out, or 0 where the reference returns None.
int orc_wm_rect(const double* mn, const double* mx, uint32_t z, double* nw_se_out) {
    wm::Rect r;
    if (!wm::Rect::from_zoomed_coordinates(mn, mx, z, r)) return 0;
    nw_se_out[0] = r.north_west.x, nw_se_out[1] = r.north_west.y, nw_se_out[2] = r.south_east.x, nw_se_out[3] = r.south_east.y;
    return 1;
}

// The normalised map position of n ECEF points (xyz: n x 3) into out[2n], and their WGS84 latitude / longitude into ll[2n].
void orc_wm_coords(const double* xyz, uint64_t n, double* out, double* ll) {
    for (uint64_t i = 0; i < n; ++i) {
        const wm::LatLng g = wm::from_ecef({xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]});
        const wm::Coord c = wm::from_lat_lng(g);
        out[2 * i] = c.x, out[2 * i + 1] = c.y;
        if (ll) ll[2 * i] = g.lat, ll[2 * i + 1] = g.lng;
    }
}
// WebMercatorCoord::from_lat_lng and to_lat_lng of n values (radians / normalised)
void orc_wm_from_lat_lng(const double* ll, uint64_t n, double* out) {
    for (uint64_t i = 0; i < n; ++i) {
        const wm::Coord c = wm::from_lat_lng({ll[2 * i], ll[2 * i + 1]});
        out[2 * i] = c.x, out[2 * i + 1] = c.y;
    }
}
void orc_wm_to_lat_lng(const double* w, uint64_t n, double* out) {
    for (uint64_t i = 0; i < n; ++i) {
        const wm::LatLng g = wm::to_lat_lng({w[2 * i], w[2 * i + 1]});
        out[2 * i] = g.lat, out[2 * i + 1] = g.lng;
    }
}
// WGS84 (lat, lng radians, height m: n x 3) -> ECEF (n x 3)
void orc_wm_to_ecef(const double* llh, uint64_t n, double* out) {
    for (uint64_t i = 0; i < n; ++i) {
        const Vec3 p = wm::to_ecef(llh[3 * i], llh[3 * i + 1], llh[3 * i + 2]);
        out[3 * i] = p.x, out[3 * i + 1] = p.y, out[3 * i + 2] = p.z;
    }
}

void orc_wm_contains_n(const double* nw_se, const double* xyz, uint64_t n, uint8_t* out) {
    const wm::Rect r = rect_of(nw_se);
    for (uint64_t i = 0; i < n; ++i) out[i] = r.contains({xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]}) ? 1 : 0;
}

// contains through SAT with the face normals only against each point (point_cloud_test/tests/main.rs:104-127): 1 if In
void orc_wm_contains_sat_n(const double* nw_se, const double* xyz, uint64_t n, uint8_t* out) {
    const Intersector a = rect_of(nw_se).intersector();
    for (uint64_t i = 0; i < n; ++i) {
        const Vec3 p{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
        out[i] = sat(a.face_normals, a.corners, 8, &p, 1) == REL_IN ? 1 : 0;
    }
}

// The polyhedron's corners (out24) and its axes cached for an Aabb (cache_separating_axes_for_aabb): returns their count.
int orc_wm_geometry(const double* nw_se, double* corners24, double* axes_out, int cap) {
    const CachedAxesIntersector c = cache_separating_axes_for_aabb(rect_of(nw_se).intersector());
    for (int i = 0; i < 8; ++i) corners24[3 * i] = c.corners[i].x, corners24[3 * i + 1] = c.corners[i].y, corners24[3 * i + 2] = c.corners[i].z;
    for (int i = 0; i < (int)c.axes.size() && i < cap; ++i) axes_out[3 * i] = c.axes[i].x, axes_out[3 * i + 1] = c.axes[i].y, axes_out[3 * i + 2] = c.axes[i].z;
    return (int)c.axes.size();
}

// rect_a.intersector().intersect(&rect_b.intersector()): 0 In, 1 Cross, 2 Out
int orc_wm_intersect(const double* nw_se_a, const double* nw_se_b) { return wm::intersect(rect_of(nw_se_a).intersector(), rect_of(nw_se_b).intersector()); }

// The cached-axes relation of the rect to each box [mn[3k..], mx[3k..]]: 0 In, 1 Cross, 2 Out
void orc_wm_intersect_boxes(const double* nw_se, const double* mn, const double* mx, uint64_t n, int32_t* rel_out) {
    const CachedAxesIntersector isec = cache_separating_axes_for_aabb(rect_of(nw_se).intersector());
    for (uint64_t k = 0; k < n; ++k) {
        Vec3 c[8];
        Aabb::make({mn[3 * k], mn[3 * k + 1], mn[3 * k + 2]}, {mx[3 * k], mx[3 * k + 1], mx[3 * k + 2]}).corners(c);
        rel_out[k] = isec.intersect(c, 8);
    }
}

// nodes_in_location of an octree handle (orc_build / orc_load_dir of liboracle.so), BFS order
int64_t orc_wm_nodes(void* hp, const double* nw_se, uint64_t* hi_lo_out, int64_t cap) {
    const std::vector<NodeId> ids = wm::nodes_in_rect(((Handle*)hp)->oct, rect_of(nw_se));
    for (int64_t i = 0; i < (int64_t)ids.size() && i < cap; ++i) hi_lo_out[2 * i] = ids[i].high(), hi_lo_out[2 * i + 1] = ids[i].low();
    return (int64_t)ids.size();
}

// orc_query with the rect: survivors in node (BFS) order, file order inside a node; call with null outputs to count.
int64_t orc_wm_query(void* hp, const double* nw_se, const double* filters, int nfilt, double* xyz, uint64_t* src, int64_t cap) {
    Handle* h = (Handle*)hp;
    const wm::Rect r = rect_of(nw_se);
    std::vector<Interval> fi;
    for (int i = 0; i < nfilt; ++i) fi.push_back({0, filters[2 * i], filters[2 * i + 1]});
    QueryOut out;
    for (NodeId id : wm::nodes_in_rect(h->oct, r)) wm::query_node_rect(h->oct, id, r, fi, out);
    const int64_t n = (int64_t)out.src.size();
    if (xyz && n <= cap) {
        std::memcpy(xyz, out.xyz.data(), out.xyz.size() * 8);
        std::memcpy(src, out.src.data(), out.src.size() * 8);
    }
    return n;
}

}  // extern "C"
