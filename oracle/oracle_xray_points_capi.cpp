// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_core.hpp header).
// C interface of oracle_xray_points.hpp for tests/ (ctypes): the X-ray tiles and quadtree of a point list.  Built on its own
// (tests/test_s2_xray_oracle_points.py, with the flags of oracle/Makefile) into liboracle_points.so.
#include <cstring>

#include "oracle_xray_points.hpp"

using namespace orc;

extern "C" {

// Same layout as the product's pcv_xray_quadtree_params and oracle_capi.cpp's orc_xray_quadtree_params.
struct orc_points_quadtree_params {
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

}  // extern "C"

static Iso3 iso_from7(const double* v) {
    Iso3 r;
    r.t = {v[0], v[1], v[2]};
    for (int k = 0; k < 4; ++k) r.q[k] = v[3 + k];
    return r;
}

// n stored positions (xyz, n * 3), optional colour and intensity, filter intervals on the intensity ([lo, hi] pairs), the box
// the quadtree is laid over (bbox6 = min xyz, max xyz) and the frame of the grid that narrows the candidates (null: global).
static PointList point_list(const double* xyz, const uint8_t* rgb, const float* intensity, uint64_t n, const double* bbox6, const double* filters,
                            uint32_t nfilt, const double* query_from_global7) {
    PointList pl;
    pl.xyz = xyz;
    pl.rgb = rgb;
    pl.intensity = intensity;
    pl.n = (size_t)n;
    for (uint32_t f = 0; f < nfilt; ++f) pl.filters.push_back(Interval{0, filters[2 * f], filters[2 * f + 1]});
    pl.bbox = Aabb::make({bbox6[0], bbox6[1], bbox6[2]}, {bbox6[3], bbox6[4], bbox6[5]});
    pl.has_frame = query_from_global7 != nullptr;
    if (pl.has_frame) pl.frame = iso_from7(query_from_global7);
    pl.index();
    return pl;
}

extern "C" {

// xray_tile (mode 0) or xray_tile_attr (modes 1-3) of one tile over a point list; returns whether a point passed.
int orc_xray_tile_points(const double* xyz, const uint8_t* rgb, const float* intensity, uint64_t n, const double* filters, uint32_t nfilt,
                         const double* bbox_min, const double* bbox_max, uint32_t w, uint32_t hgt, const double* query_from_global7, int mode, float p0,
                         float p1, int colormap, uint8_t* rgba_out) {
    const double b6[6] = {bbox_min[0], bbox_min[1], bbox_min[2], bbox_max[0], bbox_max[1], bbox_max[2]};
    const PointList pl = point_list(xyz, rgb, intensity, n, b6, filters, nfilt, query_from_global7);
    const Aabb bb = pl.bbox;
    Iso3 q{};
    if (query_from_global7) q = iso_from7(query_from_global7);
    std::vector<uint8_t> rgba;
    const bool any = mode == 0 ? xray_tile_points(pl, bb, w, hgt, query_from_global7 != nullptr, q, rgba)
                               : xray_tile_attr_points(pl, bb, w, hgt, query_from_global7 != nullptr, q, mode, p0, p1, colormap, rgba);
    std::memcpy(rgba_out, rgba.data(), rgba.size());
    return any ? 1 : 0;
}

void* orc_xray_quadtree_build_points(const double* xyz, const uint8_t* rgb, const float* intensity, uint64_t n, const double* bbox6, const double* filters,
                                     uint32_t nfilt, const orc_points_quadtree_params* p) {
    const PointList pl = point_list(xyz, rgb, intensity, n, bbox6, filters, nfilt, p->has_query_from_global ? p->query_from_global : nullptr);
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
    if (!build_xray_quadtree_points(pl, pr, *q)) {
        delete q;
        return nullptr;
    }
    return q;
}
void orc_points_quadtree_info(void* qp, double* rect3, int* deepest, uint64_t* ntiles) {
    XrayQuadtree* q = (XrayQuadtree*)qp;
    rect3[0] = q->bounding_rect.min_x, rect3[1] = q->bounding_rect.min_y, rect3[2] = q->bounding_rect.edge;
    *deepest = q->deepest_level;
    *ntiles = q->tiles.size();
}
void orc_points_quadtree_ids(void* qp, uint8_t* levels, uint64_t* indices) {
    size_t k = 0;
    for (auto& kv : ((XrayQuadtree*)qp)->tiles) levels[k] = kv.first.level, indices[k] = kv.first.index, ++k;
}
int orc_points_quadtree_tile(void* qp, uint8_t level, uint64_t index, uint8_t* rgba_out) {
    XrayQuadtree* q = (XrayQuadtree*)qp;
    auto it = q->tiles.find(QuadId{level, index});
    if (it == q->tiles.end()) return -1;
    std::memcpy(rgba_out, it->second.px.data(), it->second.px.size());
    return 0;
}
void orc_points_quadtree_free(void* qp) { delete (XrayQuadtree*)qp; }

}  // extern "C"
