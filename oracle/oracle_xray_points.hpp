// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle_core.hpp header).  Never linked into, imported by or executed from the
// product; only tests/ may use it.
//
// The X-ray leaf tiles and build_xray_quadtree over a list of points instead of an octree: what the reference computes when
// PointCloudClientBuilder opens an S2-cell directory (point_cloud_client/src/lib.rs:108-133) and the leaf queries carry
// filter_intervals (xray/src/generation.rs:464-513, FilteredIterator in src/iterator.rs:76-125), with the reference's
// latitude / longitude pre-selection of cells replaced by nothing: a leaf's points are every listed point its location
// contains that passes every interval.  The per-point arithmetic is xray_tile / xray_tile_attr of oracle_query.hpp restated
// over a point list; tests/test_s2_xray_oracle_points.py pins both forms to each other bit for bit, fed the decoded points of
// an oracle octree.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <set>
#include <vector>

#include "oracle_query.hpp"
#include "oracle_xray_pyramid.hpp"

namespace orc {

// Stored f64 positions, optional colour and intensity, filter intervals on the intensity, and the box the quadtree is laid
// over.  Points are visited in list order.  A uniform grid over (x, y) of the points in `frame` (the quadtree's
// query_from_global, if any) only narrows which points get tested: the location's eight corners (an Aabb's, or an Obb's
// through query_from_obb) are taken into the frame, and their box, widened far beyond the rounding of these transforms (1e-7
// of the largest coordinate), holds every point the location contains; every candidate then takes the exact test.
struct PointList {
    const double* xyz = nullptr;  // n * 3
    const uint8_t* rgb = nullptr;
    const float* intensity = nullptr;
    size_t n = 0;
    std::vector<Interval> filters;
    Aabb bbox{};
    bool has_frame = false;
    Iso3 frame{};
    double gx = 0.0, gy = 0.0, cell = 1.0;
    int64_t side = 1;
    std::vector<uint32_t> first, idx;  // grid cell c holds idx[first[c] .. first[c + 1])

    Vec3 in_frame(Vec3 p) const { return has_frame ? iso_transform_point(frame, p) : p; }
    int64_t cell_of(double v, double v0) const {
        const double f = std::floor((v - v0) / cell);
        return !(f >= 0.0) ? 0 : (f >= (double)(side - 1) ? side - 1 : (int64_t)f);
    }
    void index() {
        double lo[2] = {0, 0}, hi[2] = {0, 0};
        std::vector<double> fx(n), fy(n);
        for (size_t i = 0; i < n; ++i) {
            const Vec3 q = in_frame(Vec3{xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]});
            fx[i] = q.x, fy[i] = q.y;
            lo[0] = i == 0 ? q.x : std::fmin(lo[0], q.x), hi[0] = i == 0 ? q.x : std::fmax(hi[0], q.x);
            lo[1] = i == 0 ? q.y : std::fmin(lo[1], q.y), hi[1] = i == 0 ? q.y : std::fmax(hi[1], q.y);
        }
        side = std::max<int64_t>(1, std::min<int64_t>(1024, (int64_t)std::sqrt((double)n / 32.0)));
        gx = lo[0], gy = lo[1];
        cell = std::fmax(hi[0] - lo[0], hi[1] - lo[1]) / (double)side;
        if (!(cell > 0.0)) cell = 1.0;
        first.assign((size_t)(side * side + 1), 0);
        std::vector<uint32_t> key(n);
        for (size_t i = 0; i < n; ++i) first[(key[i] = (uint32_t)(cell_of(fy[i], gy) * side + cell_of(fx[i], gx))) + 1]++;
        for (size_t c = 1; c < first.size(); ++c) first[c] += first[c - 1];
        idx.resize(n);
        std::vector<uint32_t> cur(first.begin(), first.end() - 1);
        for (size_t i = 0; i < n; ++i) idx[cur[key[i]]++] = (uint32_t)i;  // ascending inside every cell
    }
    // the indices of the points that can pass `loc`, ascending
    std::vector<uint32_t> candidates(const Location& loc) const {
        std::vector<uint32_t> out;
        if (loc.kind != LOC_AABB && loc.kind != LOC_OBB) {
            for (uint32_t i = 0; i < (uint32_t)n; ++i) out.push_back(i);
            return out;
        }
        double lo[2] = {0, 0}, hi[2] = {0, 0}, big = 0.0;
        for (int k = 0; k < 8; ++k) {
            Vec3 c;
            if (loc.kind == LOC_AABB) {
                c = Vec3{(k & 1) ? loc.aabb.maxs.x : loc.aabb.mins.x, (k & 2) ? loc.aabb.maxs.y : loc.aabb.mins.y, (k & 4) ? loc.aabb.maxs.z : loc.aabb.mins.z};
            } else {
                const Vec3 h = loc.obb.half_extent;
                c = iso_transform_point(loc.obb.query_from_obb, Vec3{(k & 1) ? h.x : -h.x, (k & 2) ? h.y : -h.y, (k & 4) ? h.z : -h.z});
            }
            big = std::fmax(big, std::fmax(std::fabs(c.x), std::fmax(std::fabs(c.y), std::fabs(c.z))));
            c = in_frame(c);
            big = std::fmax(big, std::fmax(std::fabs(c.x), std::fabs(c.y)));
            lo[0] = k == 0 ? c.x : std::fmin(lo[0], c.x), hi[0] = k == 0 ? c.x : std::fmax(hi[0], c.x);
            lo[1] = k == 0 ? c.y : std::fmin(lo[1], c.y), hi[1] = k == 0 ? c.y : std::fmax(hi[1], c.y);
        }
        const double widen = 1e-7 * big + 1e-9;
        lo[0] -= widen, lo[1] -= widen, hi[0] += widen, hi[1] += widen;
        if (!(lo[0] <= hi[0]) || !(lo[1] <= hi[1])) return out;
        for (int64_t cy = cell_of(lo[1], gy); cy <= cell_of(hi[1], gy); ++cy)
            for (int64_t cx = cell_of(lo[0], gx); cx <= cell_of(hi[0], gx); ++cx) {
                const size_t c = (size_t)(cy * side + cx);
                out.insert(out.end(), idx.begin() + first[c], idx.begin() + first[c + 1]);
            }
        std::sort(out.begin(), out.end());
        return out;
    }
    // FilteredIterator over the list: every point `loc` contains that passes every interval (intensity as f64, closed;
    // math/mod.rs:87-89), in list order, as one batch
    QueryOut query(const Location& loc) const {
        QueryOut q;
        for (uint32_t i : candidates(loc)) {
            const Vec3 p{xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]};
            bool keep = loc.contains(p);
            for (const Interval& fi : filters) {
                const double v = intensity ? (double)intensity[i] : 0.0;
                keep = keep && (fi.lo <= v && v <= fi.hi);
            }
            if (!keep) continue;
            q.xyz.push_back(p.x);
            q.xyz.push_back(p.y);
            q.xyz.push_back(p.z);
            for (int k = 0; k < 3; ++k) q.rgb.push_back(rgb ? rgb[3 * (size_t)i + k] : 0);
            if (intensity) q.intensity.push_back(intensity[i]);
            q.src.push_back(i);
        }
        return q;
    }
};

// xray_tile (oracle_query.hpp) over the points of a list: the XRay strategy, 1024 z buckets per pixel.
inline bool xray_tile_points(const PointList& pl, const Aabb& bbox, uint32_t w, uint32_t h, bool has_q, const Iso3& query_from_global,
                             std::vector<uint8_t>& rgba) {
    const QueryOut q = pl.query(xray_location(bbox, has_q, query_from_global));
    std::vector<uint32_t> zbits((size_t)w * h * 32, 0u);
    std::vector<uint8_t> zover((size_t)w * h, 0);
    const Vec3 mn = bbox.mins, dg = bbox.diag();
    for (size_t i = 0; i < q.src.size(); ++i) {
        Vec3 p{q.xyz[3 * i], q.xyz[3 * i + 1], q.xyz[3 * i + 2]};
        if (has_q) p = iso_transform_point(query_from_global, p);
        const uint32_t x = rust_f64_as_u32(((p.x - mn.x) / dg.x) * (double)w);
        const uint32_t y = rust_f64_as_u32((1. - ((p.y - mn.y) / dg.y)) * (double)h);
        const uint32_t z = rust_f64_as_u32(((p.z - mn.z) / dg.z) * 1024.);
        if (x < w && y < h) {
            if (z < 1024)
                zbits[((size_t)y * w + x) * 32 + (z >> 5)] |= 1u << (z & 31);
            else
                zover[(size_t)y * w + x] = 1;
        }
    }
    fill_transparent(rgba, (size_t)w * h);
    if (q.src.empty()) return false;
    const double max_sat = std::log(1024.);
    for (size_t px = 0; px < (size_t)w * h; ++px) {
        uint32_t cnt = zover[px];
        for (int k = 0; k < 32; ++k) cnt += (uint32_t)__builtin_popcount(zbits[px * 32 + k]);
        if (cnt == 0) continue;
        const uint32_t v = rust_f64_as_u32((1. - std::log((double)cnt) / max_sat) * 255.);
        const uint8_t g = (uint8_t)(v > 255 ? 255 : v);
        rgba[px * 4 + 0] = rgba[px * 4 + 1] = rgba[px * 4 + 2] = g;
        rgba[px * 4 + 3] = 255;
    }
    return true;
}

// xray_tile_attr (oracle_query.hpp) over the points of a list: modes 1-3, Binning = None.
inline bool xray_tile_attr_points(const PointList& pl, const Aabb& bbox, uint32_t w, uint32_t h, bool has_q, const Iso3& query_from_global, int mode,
                                  float p0, float p1, int colormap, std::vector<uint8_t>& rgba) {
    const QueryOut q = pl.query(xray_location(bbox, has_q, query_from_global));
    const size_t npix = (size_t)w * h;
    std::vector<float> sum(npix * 4, 0.f);
    std::vector<uint64_t> count(npix, 0);
    std::vector<double> mean(npix, 0.0), variance(npix, 0.0);  // OnlineStats
    const Vec3 mn = bbox.mins, dg = bbox.diag();
    for (size_t i = 0; i < q.src.size(); ++i) {
        Vec3 p{q.xyz[3 * i], q.xyz[3 * i + 1], q.xyz[3 * i + 2]};
        if (has_q) p = iso_transform_point(query_from_global, p);
        const uint32_t x = rust_f64_as_u32(((p.x - mn.x) / dg.x) * (double)w);
        const uint32_t y = rust_f64_as_u32((1. - ((p.y - mn.y) / dg.y)) * (double)h);
        if (!(x < w && y < h)) continue;
        const size_t px = (size_t)y * w + x;
        if (mode == 1) {
            sum[px * 4 + 0] += (float)q.rgb[3 * i] / 255.f;
            sum[px * 4 + 1] += (float)q.rgb[3 * i + 1] / 255.f;
            sum[px * 4 + 2] += (float)q.rgb[3 * i + 2] / 255.f;
            sum[px * 4 + 3] += 255.f / 255.f;
            count[px]++;
        } else if (mode == 2) {
            const float v = q.intensity.empty() ? 0.f : q.intensity[i];
            if (v < 0.f) continue;  // see oracle_query.hpp: "negative intensities are skipped"
            sum[px * 4] += v;
            count[px]++;
        } else {
            const double sample = p.z, oldmean = mean[px], prevq = variance[px] * (double)count[px];
            count[px]++;
            mean[px] += (sample - oldmean) / (double)count[px];
            variance[px] = (prevq + (sample - oldmean) * (sample - mean[px])) / (double)count[px];
        }
    }
    fill_transparent(rgba, npix);
    if (q.src.empty()) return false;
    for (size_t px = 0; px < npix; ++px) {
        if (count[px] == 0) continue;
        uint8_t* o = &rgba[px * 4];
        if (mode == 1) {
            for (int k = 0; k < 4; ++k) o[k] = f32_to_u8((0.f + sum[px * 4 + k] / (float)count[px]) / 1.f);
        } else if (mode == 2) {
            float m = (0.f + sum[px * 4] / (float)count[px]) / 1.f;
            m = std::fmin(std::fmax(m, p0), p1);
            o[0] = o[1] = o[2] = f32_to_u8(std::log(m - p0) / std::log(p1 - p0));
            o[3] = f32_to_u8(1.f);
        } else {
            float sd = (float)std::sqrt(variance[px]);
            sd = sd < 0.f ? 0.f : (sd > p0 ? p0 : sd);
            colormap_u8(colormap, sd / p0, o);
        }
    }
    return true;
}

// build_xray_quadtree (oracle_xray_pyramid.hpp) over a point list, laid over pl.bbox; Binning = None only.
inline bool build_xray_quadtree_points(const PointList& pl, const XrayQuadtreeParams& pr, XrayQuadtree& out) {
    const Aabb bounding_box = pr.has_q ? aabb_transform(pl.bbox, pr.query_from_global) : pl.bbox;
    QuadRect rect;
    uint8_t deepest = 0;
    find_quadtree_bounding_rect_and_levels(bounding_box, pr.tile_size_px, pr.pixel_size_m, rect, deepest);
    if (pr.root.level > deepest) return false;
    out.deepest_level = deepest;
    out.bounding_rect = quad_rect_of(pr.root, rect);
    std::vector<QuadId> leaves{pr.root};
    for (int l = pr.root.level; l < deepest; ++l) {
        std::vector<QuadId> next;
        for (const QuadId& n : leaves)
            for (int k = 0; k < 4; ++k) next.push_back(n.child(k));
        leaves.swap(next);
    }
    std::set<QuadId> current;
    for (const QuadId& id : leaves) {
        const QuadRect r = quad_rect_of(id, rect);
        const Aabb bb = Aabb::make({r.min_x, r.min_y, bounding_box.mins.z}, {r.min_x + r.edge, r.min_y + r.edge, bounding_box.maxs.z});
        Image img;
        img.w = img.h = pr.tile_size_px;
        const bool any = pr.strategy == 0 ? xray_tile_points(pl, bb, img.w, img.h, pr.has_q, pr.query_from_global, img.px)
                                          : xray_tile_attr_points(pl, bb, img.w, img.h, pr.has_q, pr.query_from_global, pr.strategy, pr.p0, pr.p1,
                                                                  pr.colormap, img.px);
        if (!any) continue;
        assign_background(img, pr.background);
        out.tiles[id] = std::move(img);
        current.insert(id);
    }
    for (int level = (int)deepest - 1; level >= (int)pr.root.level; --level) {
        std::set<QuadId> parents;
        for (const QuadId& id : current) parents.insert(id.parent());
        for (const QuadId& id : parents) {
            const Image* ch[4];
            for (int k = 0; k < 4; ++k) {
                auto it = out.tiles.find(id.child(k));
                ch[k] = it == out.tiles.end() ? nullptr : &it->second;
            }
            out.tiles[id] = resize_lanczos3(build_parent(ch, pr.background), pr.tile_size_px, pr.tile_size_px);
        }
        current.swap(parents);
    }
    return true;
}

}  // namespace orc
