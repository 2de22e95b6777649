// s2.h — the S2 cell arithmetic the S2-cell point cloud needs (SURVEY 8 f4), shared by the CUDA kernels (s2.cuh) and the
// sequential test backend.  Everything is integer or IEEE-754 binary64 (+, *, /, sqrt, floor): no libm, so host and device
// agree bit for bit.
//
// Reference call sites (file:line relative to the reference checkout):
//   CellID::from_point(p) = CellID::from(Point::from_coords(x, y, z))   src/math/mod.rs:119-131
//   S2Splitter::write: radius check, bounding box, from_point(p).parent(split_level), per-cell batches
//                                                                      src/read_write/s2.rs:14-17,59-125
//   CellUnion as PointCulling: contains_cellid(from_point(p))          src/geometry/s2_cell_union.rs:27-31
//   S2Cells::nodes_in_location (AllPoints, S2Cells)                     src/s2_cells/mod.rs:157-168,233-241
// THIRD-PARTY, UN-VENDORED: the arithmetic itself lives in the `s2` crate (0.0.10 in Cargo.lock, a port of golang/geo's s2
// package), which is not in /root/reference.  It is restated here from the published S2 algorithm (the same in the C++, Go and
// Rust libraries): point -> unit vector -> face and (u, v) by the largest component -> quadratic (s, t) -> (i, j) in
// [0, 2^30) -> position along the Hilbert curve of the face.  This header walks the curve level by level with the 4 x 4
// tables; the oracle (oracle/oracle_s2.hpp) uses the libraries' 1024-entry look-up tables - two formulations of one curve.
#pragma once
#include <stdint.h>

#include "chain.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

namespace pcv {

constexpr int kS2MaxLevel = 30;
constexpr double kEarthRadiusMinM = 6352800.0;  // src/math/mod.rs:30-35
constexpr double kEarthRadiusMaxM = 6384400.0;

// The orientation change after each curve position (the libraries' posToOrientation; swapMask = 1, invertMask = 2).
PCV_HD int s2_pos_to_orientation(int pos) { return pos == 0 ? 1 : pos == 3 ? 3 : 0; }

// uv -> st (quadratic projection) and st -> ij
PCV_HD double s2_uv_to_st(double u) { return u >= 0.0 ? 0.5 * sqrt(1.0 + 3.0 * u) : 1.0 - 0.5 * sqrt(1.0 - 3.0 * u); }
PCV_HD int s2_st_to_ij(double s) {
    const double f = floor(1073741824.0 * s);  // maxSize = 2^30
    // clamp(int(f), 0, maxSize - 1); a NaN becomes 0 (Rust `as i32`; unreachable for points that pass the radius check)
    if (!(f >= 0.0)) return 0;
    return f >= 1073741823.0 ? 1073741823 : (int)f;
}

// Point::from_coords + xyz_to_face_uv: the unit vector, its face and (u, v).
PCV_HD int s2_face_uv(double x, double y, double z, double& u, double& v) {
    if (!(x == 0.0 && y == 0.0 && z == 0.0)) {  // Vector::normalize: v * (1 / |v|)
        const double inv = 1.0 / sqrt(x * x + y * y + z * z);
        x = x * inv, y = y * inv, z = z * inv;
    } else {  // Point::origin(): (-0.0099994664, 0.0025924542, 0.9999466403), already unit length in the libraries' eyes
        x = -0.0099994664350250197, y = 0.0025924542609324121, z = 0.99994664350250195;
    }
    const double ax = fabs(x), ay = fabs(y), az = fabs(z);
    int axis;  // largest_component: ties go to the later axis
    if (ax > ay)
        axis = ax > az ? 0 : 2;
    else
        axis = ay > az ? 1 : 2;
    const double c = axis == 0 ? x : axis == 1 ? y : z;
    const int face = c < 0.0 ? axis + 3 : axis;
    switch (face) {
        case 0: u = y / x, v = z / x; break;
        case 1: u = -x / y, v = z / y; break;
        case 2: u = -x / z, v = -y / z; break;
        case 3: u = z / x, v = y / x; break;
        case 4: u = z / y, v = -x / y; break;
        default: u = -y / z, v = -x / z; break;
    }
    return face;
}

// cellIDFromFaceIJ: the leaf cell (level 30) of (face, i, j), walking the Hilbert curve one level at a time.
PCV_HD uint64_t s2_from_face_ij(int face, int i, int j) {
    uint64_t n = (uint64_t)face << 60;
    int orientation = face & 1;
    for (int k = kS2MaxLevel - 1; k >= 0; --k) {
        const int ij = (((i >> k) & 1) << 1) | ((j >> k) & 1);
        // position of the sub-cell (i bit, j bit) along the curve in the current orientation
        int pos;
        switch (orientation) {
            case 0: pos = ij == 0 ? 0 : ij == 1 ? 1 : ij == 3 ? 2 : 3; break;  // posToIJ[0] = {0, 1, 3, 2}
            case 1: pos = ij == 0 ? 0 : ij == 2 ? 1 : ij == 3 ? 2 : 3; break;  // posToIJ[1] = {0, 2, 3, 1}
            case 2: pos = ij == 3 ? 0 : ij == 2 ? 1 : ij == 0 ? 2 : 3; break;  // posToIJ[2] = {3, 2, 0, 1}
            default: pos = ij == 3 ? 0 : ij == 1 ? 1 : ij == 0 ? 2 : 3; break; // posToIJ[3] = {3, 1, 0, 2}
        }
        n |= (uint64_t)pos << (2 * k);
        orientation ^= s2_pos_to_orientation(pos);
    }
    return n * 2 + 1;
}

PCV_HD uint64_t s2_cell_id_from_point(double x, double y, double z) {
    double u, v;
    const int face = s2_face_uv(x, y, z, u, v);
    return s2_from_face_ij(face, s2_st_to_ij(s2_uv_to_st(u)), s2_st_to_ij(s2_uv_to_st(v)));
}

PCV_HD uint64_t s2_lsb_for_level(int level) { return 1ull << (2 * (kS2MaxLevel - level)); }
PCV_HD uint64_t s2_lsb(uint64_t id) { return id & (0 - id); }
PCV_HD uint64_t s2_parent(uint64_t id, int level) {  // CellID::parent(level)
    const uint64_t lsb = s2_lsb_for_level(level);
    return (id & (0 - lsb)) | lsb;
}
PCV_HD uint64_t s2_range_min(uint64_t id) { return id - (s2_lsb(id) - 1); }
PCV_HD uint64_t s2_range_max(uint64_t id) { return id + (s2_lsb(id) - 1); }
PCV_HD int s2_level(uint64_t id) {  // 30 - (trailing zeros) / 2
    int tz = 0;
    while (tz < 64 && !((id >> tz) & 1)) ++tz;
    return kS2MaxLevel - tz / 2;
}
PCV_HD bool s2_is_valid(uint64_t id) { return (id >> 61) < 6 && (s2_lsb(id) & 0x1555555555555555ull) != 0; }

// CellUnion::contains_cellid / intersects_cellid over a NORMALISED union (sorted, no cell contains another):
// binary search for the first cell >= id, then the two range checks of the libraries.
PCV_HD uint32_t s2_lower_bound(const uint64_t* cells, uint32_t n, uint64_t id) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (cells[mid] < id)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}
PCV_HD bool s2_union_contains(const uint64_t* cells, uint32_t n, uint64_t id) {
    const uint32_t i = s2_lower_bound(cells, n, id);
    if (i < n && s2_range_min(cells[i]) <= id) return true;
    return i != 0 && s2_range_max(cells[i - 1]) >= id;
}
PCV_HD bool s2_union_intersects(const uint64_t* cells, uint32_t n, uint64_t id) {
    const uint32_t i = s2_lower_bound(cells, n, id);
    if (i < n && s2_range_min(cells[i]) <= s2_range_max(id)) return true;
    return i != 0 && s2_range_max(cells[i - 1]) >= s2_range_min(id);
}

// A cell as a face and the aligned square of leaf cells it covers: [i0, i0 + size) x [j0, j0 + size), size = 2^(30 - level).
// A leaf cell lies in a cell iff its (face, i, j) lies in the cell's square (the curve subdivides the face as a quadtree).
struct S2Square {
    int32_t face;
    uint32_t i0, j0, size;
};

// The inverse of s2_from_face_ij for a cell of any level: read its curve positions from the top, posToIJ per orientation.
PCV_HD S2Square s2_to_face_ij_level(uint64_t id) {
    S2Square q;
    q.face = (int32_t)(id >> 61);
    const int level = s2_level(id);
    int orientation = q.face & 1;
    uint32_t i = 0, j = 0;
    for (int k = kS2MaxLevel - 1; k >= kS2MaxLevel - level; --k) {
        const int pos = (int)((id >> (2 * k + 1)) & 3);
        int ij;
        switch (orientation) {
            case 0: ij = pos == 0 ? 0 : pos == 1 ? 1 : pos == 2 ? 3 : 2; break;  // posToIJ[0] = {0, 1, 3, 2}
            case 1: ij = pos == 0 ? 0 : pos == 1 ? 2 : pos == 2 ? 3 : 1; break;  // posToIJ[1] = {0, 2, 3, 1}
            case 2: ij = pos == 0 ? 3 : pos == 1 ? 2 : pos == 2 ? 0 : 1; break;  // posToIJ[2] = {3, 2, 0, 1}
            default: ij = pos == 0 ? 3 : pos == 1 ? 1 : pos == 2 ? 0 : 2; break; // posToIJ[3] = {3, 1, 0, 2}
        }
        i |= (uint32_t)(ij >> 1) << k;
        j |= (uint32_t)(ij & 1) << k;
        orientation ^= s2_pos_to_orientation(pos);
    }
    q.i0 = i;
    q.j0 = j;
    q.size = 1u << (kS2MaxLevel - level);
    return q;
}

// The node test of a cell union: where the leaf cells s2_cell_id_from_point computes for the points of the cube [m, m + e]^3 can
// lie, against the union's squares.  Out: no point's leaf cell is in the union; In: every point's is; Cross: otherwise.
// Same coding as the query kernels' Relation (query.cuh).
enum : int { kS2RelIn = 0, kS2RelCross = 1, kS2RelOut = 2 };

// Soundness.  A point p of the cube with |p_k| <= 1e150 for every k and max |p_k| >= 1e-150 is normalised without over- or
// underflow: x_n = RN(x * inv) with one inv for all three components, so the computed face has |p_a| >= |p_b| (1 - 2^-51) for its
// axis a, and its u = RN(y_n / x_n) equals (y / x)(1 + d) with |d| < 2^-51 (inv cancels; three roundings), up to an absolute
// 2^-1070 when y_n is subnormal.  The exact ratio of a cube point lies between the cube's extreme corner ratios, which are
// computed here with one rounding each.  Widening every bound by the relative kS2Widen = 2^-40 and the absolute 1e-300 therefore
// covers the point's computed u, v; s2_uv_to_st and s2_st_to_ij are monotone under correct rounding, so the widened bounds map to
// bounds of its (i, j).  The same margin admits every face whose axis can come within 2^-40 of the largest component.  Cubes
// outside that range (near the origin, huge or NaN corners) are Cross.  Decoded points lie in [m, RN(m + e)] (fma(t, e, m) with
// 0 <= t <= 1), the cube tested here.
constexpr double kS2Widen = 9.094947017729282e-13;  // 2^-40

// v[k] with selects rather than an indexed load (a small array indexed at run time goes to a kernel's local memory)
PCV_HD double s2_pick(const double v[3], int k) { return k == 0 ? v[0] : k == 1 ? v[1] : v[2]; }

// [lo, hi] of N / D over N in [nlo, nhi] and D in [dlo, dhi], 0 < dlo: the extremes lie at the corners.
PCV_HD void s2_ratio_bounds(double nlo, double nhi, double dlo, double dhi, double& lo, double& hi) {
    const double a = nlo / dlo, b = nlo / dhi, c = nhi / dlo, d = nhi / dhi;
    lo = a < b ? a : b;
    hi = c > d ? c : d;
    lo = lo - (fabs(lo) * kS2Widen + 1e-300);
    hi = hi + (fabs(hi) * kS2Widen + 1e-300);
    lo = lo < -1.0 ? -1.0 : lo;  // a computed u, v is in [-1, 1]: |y_n| <= |x_n| for the chosen face
    hi = hi > 1.0 ? 1.0 : hi;
}

PCV_HD int s2_cube_relation(const double m[3], double e, const S2Square* sq, uint32_t n) {
    if (n == 0) return kS2RelOut;
    double lo[3], hi[3], amin[3];
    bool near_origin = true;
    for (int k = 0; k < 3; ++k) {
        lo[k] = m[k];
        hi[k] = m[k] + e;
        if (!(fabs(lo[k]) <= 1e150 && fabs(hi[k]) <= 1e150 && lo[k] <= hi[k])) return kS2RelCross;
        near_origin = near_origin && lo[k] <= 1e-150 && hi[k] >= -1e-150;
        amin[k] = lo[k] > 0.0 ? lo[k] : hi[k] < 0.0 ? -hi[k] : 0.0;  // the smallest |p_k| over the cube
    }
    if (near_origin) return kS2RelCross;
    // (u, v) of face f as (+-p_b / |p_a|, +-p_c / |p_a|): s2_face_uv's table with the sign of p_a folded in.  Packed (a nibble per
    // face for b and c, a bit per face for a negative sign) so that no table lands in local memory:
    //   b = {1, 0, 0, 2, 2, 1}, u negated on faces 1-4;  c = {2, 2, 1, 1, 0, 0}, v negated on faces 2-3
    constexpr uint32_t kUAxis = 0x122001u, kUNeg = 0x1Eu, kVAxis = 0x001122u, kVNeg = 0x0Cu;
    bool hit = false, all_in = true;
    for (int f = 0; f < 6; ++f) {
        const int a = f % 3;
        const double dhi = f < 3 ? s2_pick(hi, a) : -s2_pick(lo, a);
        if (!(dhi > 0.0)) continue;  // the major component of a point of this face has the face's sign
        const double dl = f < 3 ? s2_pick(lo, a) : -s2_pick(hi, a), dlo = dl > 0.0 ? dl : 0.0;
        const double reach = dhi + dhi * kS2Widen;
        if (reach < s2_pick(amin, (a + 1) % 3) || reach < s2_pick(amin, (a + 2) % 3)) continue;  // p_a is never the largest component
        double ulo = -1.0, uhi = 1.0, vlo = -1.0, vhi = 1.0;
        if (dlo >= 1e-150) {
            const int b = (int)((kUAxis >> (4 * f)) & 15u), c = (int)((kVAxis >> (4 * f)) & 15u);
            const bool un = (kUNeg >> f) & 1u, vn = (kVNeg >> f) & 1u;
            const double blo = s2_pick(lo, b), bhi = s2_pick(hi, b), clo = s2_pick(lo, c), chi = s2_pick(hi, c);
            s2_ratio_bounds(un ? -bhi : blo, un ? -blo : bhi, dlo, dhi, ulo, uhi);
            s2_ratio_bounds(vn ? -chi : clo, vn ? -clo : chi, dlo, dhi, vlo, vhi);
        }
        const uint32_t i0 = (uint32_t)s2_st_to_ij(s2_uv_to_st(ulo)), i1 = (uint32_t)s2_st_to_ij(s2_uv_to_st(uhi));
        const uint32_t j0 = (uint32_t)s2_st_to_ij(s2_uv_to_st(vlo)), j1 = (uint32_t)s2_st_to_ij(s2_uv_to_st(vhi));
        bool face_hit = false, covered = false;
        for (uint32_t k = 0; k < n; ++k) {
            const S2Square s = sq[k];
            const uint32_t ie = s.i0 + (s.size - 1), je = s.j0 + (s.size - 1);  // last leaf row / column of the square
            if (s.face != f || i1 < s.i0 || i0 > ie || j1 < s.j0 || j0 > je) continue;
            face_hit = true;
            if (i0 >= s.i0 && i1 <= ie && j0 >= s.j0 && j1 <= je) {
                covered = true;
                break;
            }
        }
        hit = hit || face_hit;
        all_in = all_in && covered;
    }
    return !hit ? kS2RelOut : all_in ? kS2RelIn : kS2RelCross;
}

// The S2Splitter's validity rule (read_write/s2.rs:64-71): |p| outside [EARTH_RADIUS_MIN_M, EARTH_RADIUS_MAX_M] is an error.
// nalgebra's norm(): sqrt of the sum of squares in x, y, z order.
PCV_HD bool s2_valid_ecef(double x, double y, double z) {
    const double r = sqrt(x * x + y * y + z * z);
    return !(r > kEarthRadiusMaxM || r < kEarthRadiusMinM);
}

// ---- host helpers ------------------------------------------------------------------------------------------------
// CellID::to_token: the id in hex without its trailing zero digits; "X" for 0.
inline std::string s2_to_token(uint64_t id) {
    if (id == 0) return "X";
    char buf[17];
    snprintf(buf, sizeof buf, "%016llx", (unsigned long long)id);
    std::string s(buf);
    while (!s.empty() && s.back() == '0') s.pop_back();
    return s;
}
inline bool s2_from_token(const std::string& t, uint64_t& id) {
    if (t == "X") {
        id = 0;
        return true;
    }
    if (t.empty() || t.size() > 16) return false;
    uint64_t v = 0;
    for (char ch : t) {
        int d = ch >= '0' && ch <= '9' ? ch - '0' : ch >= 'a' && ch <= 'f' ? ch - 'a' + 10 : ch >= 'A' && ch <= 'F' ? ch - 'A' + 10 : -1;
        if (d < 0) return false;
        v = (v << 4) | (uint64_t)d;
    }
    id = v << (4 * (16 - t.size()));
    return true;
}
// CellUnion::normalize: sort, drop cells contained in an earlier one, replace four sibling cells by their parent.
inline void s2_normalize(std::vector<uint64_t>& cells) {
    std::sort(cells.begin(), cells.end());
    std::vector<uint64_t> out;
    for (uint64_t id : cells) {
        if (!out.empty() && s2_range_min(out.back()) <= id && id <= s2_range_max(out.back())) continue;  // contained in the previous cell
        while (!out.empty() && s2_range_min(id) <= out.back() && out.back() <= s2_range_max(id)) out.pop_back();  // contains previous cells
        while (out.size() >= 3 && s2_level(id) != 0) {  // the last three cells + id: the four children of one parent?  (areSiblings)
            const size_t m = out.size();
            const uint64_t a = out[m - 3], b = out[m - 2], c = out[m - 1];
            if ((a ^ b ^ c) != id) break;  // the libraries' fast reject: the XOR of four siblings is zero
            const uint64_t two = s2_lsb(id) << 1, mask = ~(two + (two << 1));  // everything above the two bits that number the children
            const uint64_t idm = id & mask;
            if ((a & mask) != idm || (b & mask) != idm || (c & mask) != idm) break;
            out.resize(m - 3);
            id = s2_parent(id, s2_level(id) - 1);
        }
        out.push_back(id);
    }
    cells.swap(out);
}

}  // namespace pcv
