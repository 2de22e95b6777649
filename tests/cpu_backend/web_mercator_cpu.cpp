// TEST-ONLY: sequential driver of the Web Mercator rect (csrc/geometry_host.hpp): the constructor and its validation, the
// PCV_GHD point test the cull kernels call, and the host geometry the node and cell selections use.  NOT part of the shipped
// library.  A rect is nw_se[4] = north_west.x, north_west.y, south_east.x, south_east.y (normalised).
#include "../../point_cloud_viewer_b200/csrc/geometry_host.hpp"

using namespace pcv;

static pcv_location rect_loc(const double* nw_se) {
    pcv_location loc{};
    loc.kind = PCV_LOC_WEB_MERCATOR_RECT;
    loc.aabb_min[0] = nw_se[0], loc.aabb_min[1] = nw_se[1];
    loc.aabb_max[0] = nw_se[2], loc.aabb_max[1] = nw_se[3];
    return loc;
}

extern "C" {
// web_mercator_rect_from_zoomed: 1 and nw_se_out, or 0
int tbw_rect(const double* mn, const double* mx, uint32_t z, double* nw_se_out) {
    double nw[2], se[2];
    if (!web_mercator_rect_from_zoomed(mn, mx, z, nw, se)) return 0;
    nw_se_out[0] = nw[0], nw_se_out[1] = nw[1], nw_se_out[2] = se[0], nw_se_out[3] = se[1];
    return 1;
}
int tbw_valid(const double* nw_se) { return web_mercator_rect_valid(nw_se, nw_se + 2) ? 1 : 0; }

// the point test's map position of n ECEF points (n x 3) into out[2n], and their latitude / longitude into ll[2n]
void tbw_coords(const double* xyz, uint64_t n, double* out, double* ll) {
    for (uint64_t i = 0; i < n; ++i) {
        double lat, lng;
        ecef_to_lat_lng(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], lat, lng);
        web_mercator_from_lat_lng(lat, lng, out + 2 * i);
        if (ll) ll[2 * i] = lat, ll[2 * i + 1] = lng;
    }
}
void tbw_to_lat_lng(const double* w, uint64_t n, double* out) {
    for (uint64_t i = 0; i < n; ++i) web_mercator_to_lat_lng(w + 2 * i, out[2 * i], out[2 * i + 1]);
}
void tbw_to_ecef(const double* llh, uint64_t n, double* out) {
    for (uint64_t i = 0; i < n; ++i) {
        const V3 p = wgs84_to_ecef(llh[3 * i], llh[3 * i + 1], llh[3 * i + 2]);
        out[3 * i] = p.x, out[3 * i + 1] = p.y, out[3 * i + 2] = p.z;
    }
}

void tbw_contains_n(const double* nw_se, const double* xyz, uint64_t n, uint8_t* out) {
    MoreAxes more;
    const QueryGeom g = make_query_geom(rect_loc(nw_se), &more);
    for (uint64_t i = 0; i < n; ++i) out[i] = web_mercator_rect_contains(g.aabb_min, g.aabb_max, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]) ? 1 : 0;
}

// make_query_geom of the kind-4 location: its corners (out24) and cached axes; returns naxes
int tbw_geometry(const double* nw_se, double* corners24, double* axes_out, int cap) {
    MoreAxes more;
    const QueryGeom g = make_query_geom(rect_loc(nw_se), &more);
    for (int i = 0; i < 8; ++i)
        for (int a = 0; a < 3; ++a) corners24[3 * i + a] = g.corners[i][a];
    for (int k = 0; k < g.naxes && k < cap; ++k)
        for (int a = 0; a < 3; ++a) axes_out[3 * k + a] = geom_axis(g, k)[a];
    return g.naxes;
}

// sat_box of the rect against every box [mn[3k..], mx[3k..]] (the S2 cloud's cell test): 0 In, 1 Cross, 2 Out
void tbw_sat_box(const double* nw_se, const double* mn, const double* mx, uint64_t nboxes, int32_t* rel_out) {
    MoreAxes more;
    const QueryGeom g = make_query_geom(rect_loc(nw_se), &more);
    double aproj[kInlineAxes][2];
    for (int k = 0; k < g.naxes && k < kInlineAxes; ++k) project_location_axis(g, k, aproj[k][0], aproj[k][1]);
    for (uint64_t k = 0; k < nboxes; ++k) rel_out[k] = sat_box(g, aproj, mn + 3 * k, mx + 3 * k);
}
}

extern "C" {
// The axes of any polyhedron (corners24, edges36 = 12 edges, normals18 = 6 face normals) cached against an Aabb, past
// kInlineAxes included (axes_out: up to kMaxAxes x 3; returns naxes), and sat_box against every box: the table path that a
// Web Mercator rect's record uses when it has more axes than the record holds.
int tbw_poly_sat_box(const double* corners24, const double* edges36, const double* normals18, double* axes_out, const double* mn, const double* mx,
                     uint64_t nboxes, int32_t* rel_out) {
    PolyIntersector p;
    for (int i = 0; i < 8; ++i) p.corners[i] = V3{corners24[3 * i], corners24[3 * i + 1], corners24[3 * i + 2]};
    for (int i = 0; i < 12; ++i) p.edges[i] = V3{edges36[3 * i], edges36[3 * i + 1], edges36[3 * i + 2]};
    for (int i = 0; i < 6; ++i) p.normals[i] = V3{normals18[3 * i], normals18[3 * i + 1], normals18[3 * i + 2]};
    p.nedges = 12;
    p.nnormals = 6;
    QueryGeom g;
    std::memset(&g, 0, sizeof g);
    g.kind = PCV_LOC_WEB_MERCATOR_RECT;
    MoreAxes more;
    cache_axes_for_aabb(p, g, &more);
    for (int k = 0; k < g.naxes; ++k)
        for (int a = 0; a < 3; ++a) axes_out[3 * k + a] = geom_axis(g, k)[a];
    double aproj[kInlineAxes][2];
    for (int k = 0; k < g.naxes && k < kInlineAxes; ++k) project_location_axis(g, k, aproj[k][0], aproj[k][1]);
    for (uint64_t k = 0; k < nboxes; ++k) rel_out[k] = sat_box(g, aproj, mn + 3 * k, mx + 3 * k);
    return g.naxes;
}
}
