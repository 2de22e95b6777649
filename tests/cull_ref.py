"""A plain numpy float64 restatement of the point culling of a query, and locations built to sit exactly on its edges.

`contains(loc, P)` is the point test of a location (`loc_contains` in csrc/query.cuh, the oracle's Location::contains), vectorised
over an (n, 3) array in the reference's operation order: every product and sum is a separate numpy operation, so nothing is fused.

  Aabb     half-open:  min <= p && p < max                                   (aabb.rs:46-48)
  Frustum  strict:     min(c) > -1 && max(c) < 1,  c = clip_from_query.transform_point(p), divided only when w != 0
                                                                              (frustum.rs:120-125)
  Obb      closed:     |q| <= half_extent,  q = obb_from_query * p            (obb.rs:83-90)

`keep_filters(intensity, intervals)` is the interval filter: the f32 attribute widened to f64, closed intervals, ANDed together
(iterator.rs:82-91, math/mod.rs:87-89).

The builders take the decoded positions of a tree (the oracle's query of all points, in node visit order) and return locations whose
faces or clip planes pass exactly through some of those points, with each designed point labelled by the outcome its class must
have (EXPECT).  The edge classes are what a subtly wrong comparison, decode or division would flip.
"""
import math

import numpy as np

LOC_ALL, LOC_AABB, LOC_FRUSTUM, LOC_OBB = 0, 1, 2, 3
ONE_MINUS = 1.0 - 2.0 ** -53  # the largest double below 1
T_FACTOR = 1.0 - 2.0 ** -52   # loc_contains' certainly-inside threshold is fl(|w| * T_FACTOR)

# the designed outcome of every label class: True = the point is in the location, False = out
EXPECT = {
    "aabb_min_face": True,       # p[k] == min[k], inside on the other axes
    "aabb_max_face": False,      # p[k] == max[k]
    "aabb_zero_thickness": False,  # min[k] == max[k] == p[k]
    "obb_face_in": True,         # |q[k]| == half_extent[k]
    "obb_face_out": False,       # half_extent[k] == nextafter(|q[k]|, 0)
    "frustum_r_eq_w": False,     # |r| == |w| with a normal w: fl(r / w) == +-1
    "frustum_band": True,        # T < |r| < |w|: the division decides, and never rounds to +-1
    "frustum_w_neg_in": True,    # w < 0, every |r| < |w|
    "frustum_w0_in": True,       # w == 0 and every |r| < 1: tested undivided
    "frustum_w0_edge": False,    # w == 0 and some r == +-1 exactly: tested undivided, strictly
    "frustum_tiny_w_edge": False,  # |w| < 1e-290 and |r| == |w|
    "frustum_tiny_w_in": True,   # |w| < 1e-290 and |r| < |w| in the band
    "frustum_huge_w_edge": False,  # |w| > 1e300 and |r| == |w|
    "frustum_huge_w_in": True,   # |w| > 1e300 and |r| < |w| in the band
}


def _col(loc, field, n):
    return np.array([getattr(loc, field)[i] for i in range(n)], np.float64)


# ---- the predicates ---------------------------------------------------------------------------------
def clip(m, P):
    """(r (n, 3), n (n,)) of clip_from_query (column-major m[c * 4 + r]) applied to P, in transform_point's order."""
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    w = m[3] * x
    w = w + m[7] * y
    w = w + m[11] * z
    w = w + m[15]
    r = np.empty_like(P)
    for i in range(3):
        a = m[i] * x
        a = m[4 + i] * y + a
        a = m[8 + i] * z + a
        r[:, i] = a + m[12 + i]
    return r, w


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)


def iso_apply(iso7, P):
    """Isometry3 * p: t = 2 (qv x p), (t w + qv x t) + p, then + translation (nalgebra 0.22)."""
    qv = np.broadcast_to(np.asarray(iso7[3:6], np.float64), P.shape)
    t = _cross(qv, P) * 2.0
    c = _cross(qv, t)
    q = t * iso7[6] + c
    q = q + P
    return q + np.asarray(iso7[:3], np.float64)


def contains(loc, P):
    P = np.asarray(P, np.float64).reshape(-1, 3)
    if loc.kind == LOC_AABB:
        mn, mx = _col(loc, "aabb_min", 3), _col(loc, "aabb_max", 3)
        return np.all(mn <= P, 1) & np.all(P < mx, 1)
    if loc.kind == LOC_FRUSTUM:
        r, w = clip(_col(loc, "clip_from_query", 16), P)
        c = r.copy()
        nz = w != 0.0
        with np.errstate(divide="ignore", invalid="ignore", over="ignore", under="ignore"):
            c[nz] = r[nz] / w[nz, None]
        mn = np.fmin(np.fmin(c[:, 0], c[:, 1]), c[:, 2])
        mx = np.fmax(np.fmax(c[:, 0], c[:, 1]), c[:, 2])
        return (mn > -1.0) & (mx < 1.0)
    if loc.kind == LOC_OBB:
        q = iso_apply(_col(loc, "obb_from_query", 7), P)
        return np.all(np.abs(q) <= _col(loc, "half_extent", 3), 1)
    return np.ones(len(P), bool)


def keep_filters(intensity, intervals):
    """intervals: [(lo, hi), ...] (f64).  NaN fails every comparison, so it is never kept when there is an interval."""
    v = np.asarray(intensity, np.float32).astype(np.float64)
    keep = np.ones(len(v), bool)
    for lo, hi in intervals:
        keep &= (lo <= v) & (v <= hi)
    return keep


# ---- the cloud --------------------------------------------------------------------------------------
# Intensities that sit on the edges of FILTERS: interval ends, -0.0 against lo = 0.0, NaN, +-inf, an f32 subnormal and f32 0.1
# (0.100000001490116..., above the f64 bound 0.1 although equal to it in f32).
SUBNORMAL_F32 = float(np.float32(1e-40))
SPECIAL_INTENSITY = np.array([0.25, 0.75, -0.0, 0.0, np.nan, np.inf, -np.inf, SUBNORMAL_F32, 0.1, 0.5, 1.0, -1.0], np.float32)
FILTERS = [
    [(0.25, 0.75)],                    # values equal to lo and hi are kept
    [(0.0, 0.5)],                      # -0.0 and the subnormal are kept, NaN is not
    [(-math.inf, math.inf)],           # +-inf are kept, NaN is not
    [(0.0, 0.1)],                      # f32 0.1 is above 0.1: dropped (kept if compared in f32)
    [(SUBNORMAL_F32, 0.5)],            # the subnormal is lo itself; +-0 are below it
    [(0.0, 0.6), (0.25, 1.0)],         # two intervals at once: [0.25, 0.6]
]


def edge_cloud(big=False, seed=5):
    """Six clusters near (4.1e6, 6.6e5, 4.7e6) with per-point spreads from 1e-6 to 1 m and a block of 3000 identical points: at
    resolution 1e-7 and max_points_per_node=200 the octree is 30 levels deep and holds Float64, Float32, Uint16 and Uint8 nodes.
    big=True adds four uniform blocks of 24 000 points with edges of 8 m, 0.4 m, 4 mm and 16 um, so that with a larger
    max_points_per_node every encoding has nodes of several cull tiles (2048 points).
    Returns x, y, z, rgb (n, 3) u8, intensity f32 (a special value on every 5th point)."""
    rng = np.random.default_rng(seed)
    n = 60000
    cen = rng.random((6, 3)) * 100.0 + [4.1e6, 6.6e5, 4.7e6]
    k = rng.integers(0, 6, n)
    P = cen[k] + rng.normal(0, 1, (n, 3)) * 10.0 ** rng.uniform(-6, 0, (n, 1))
    P[:3000] = P[0]
    if big:
        blocks = [cen[1] + [13.3, -7.1, 5.9] + (rng.random((24000, 3)) - 0.5) * e for e in (8.0, 0.4, 4e-3, 1.6e-5)]
        P = np.concatenate([P] + blocks)
    n = len(P)
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    inten = rng.random(n).astype(np.float32)
    inten[::5] = SPECIAL_INTENSITY[(np.arange(n)[::5] // 5) % len(SPECIAL_INTENSITY)]
    return np.ascontiguousarray(P[:, 0]), np.ascontiguousarray(P[:, 1]), np.ascontiguousarray(P[:, 2]), rgb, inten


# ---- boundary locations -----------------------------------------------------------------------------
def _aabb(Loc, mn, mx):
    loc = Loc()
    loc.kind = LOC_AABB
    loc.aabb_min[:] = [float(v) for v in mn]
    loc.aabb_max[:] = [float(v) for v in mx]
    return loc


def _aabb_labels(loc, P):
    mn, mx = _col(loc, "aabb_min", 3), _col(loc, "aabb_max", 3)
    lab = {}
    inside_closed = np.all(mn <= P, 1) & np.all(P <= mx, 1)
    on_max = inside_closed & np.any(P == mx, 1)
    on_min = inside_closed & np.any(P == mn, 1) & ~on_max
    if np.any(mn == mx):
        lab["aabb_zero_thickness"] = np.flatnonzero(on_max)
    else:
        lab["aabb_max_face"] = np.flatnonzero(on_max)
        lab["aabb_min_face"] = np.flatnonzero(on_min)
    return lab


def _common_value(v):
    """The most frequent value of v (coarse encodings share coordinates between many points)."""
    u, c = np.unique(v, return_counts=True)
    return u[np.argmax(c)]


def anchors(tree_nodes, order, P):
    """One node of each encoding that holds the most points, as (enc, first, count, cube) with `first` its first point in P
    (P: the points of `order`'s nodes, concatenated)."""
    best = {}
    first = 0
    for nm in order:
        m = tree_nodes[nm]
        cnt = m["num_points"]
        if cnt and (m["enc"] not in best or cnt > best[m["enc"]][2]):
            best[m["enc"]] = (m["enc"], first, cnt, m["cube"])
        first += cnt
    assert first == len(P)
    return [best[e] for e in sorted(best)]


def aabb_cases(Loc, nodes, P):
    """Boxes with faces through decoded points, boxes on octree cube planes and zero-thickness boxes."""
    out = []
    for enc, first, cnt, cube in nodes:
        Q = P[first:first + cnt]
        a = np.array([_common_value(Q[:, k]) for k in range(3)])
        e = cube[3]
        out.append(("aabb_min_faces_enc%d" % enc, _aabb(Loc, a, a + e)))   # the shared coordinates are min faces: in
        out.append(("aabb_max_faces_enc%d" % enc, _aabb(Loc, a - e, a)))   # ... and max faces: out
        cm = np.array(cube[:3])
        out.append(("aabb_below_cube_enc%d" % enc, _aabb(Loc, cm - e, cm)))          # touches the node's cube at its min corner
        out.append(("aabb_above_cube_enc%d" % enc, _aabb(Loc, cm + e, cm + 2 * e)))  # ... and at its max corner
        out.append(("aabb_on_cube_enc%d" % enc, _aabb(Loc, cm, cm + e)))             # the node's cube itself
        flat = np.arange(3) == enc % 3
        out.append(("aabb_flat_enc%d" % enc, _aabb(Loc, np.where(flat, a, a - e), np.where(flat, a, a + e))))  # zero thickness: empty
    return [(nm, loc, _aabb_labels(loc, P)) for nm, loc in out]


def _obb(Loc, iso7, inv7, h):
    loc = Loc()
    loc.kind = LOC_OBB
    loc.query_from_obb[:] = [float(v) for v in iso7]
    loc.obb_from_query[:] = [float(v) for v in inv7]
    loc.half_extent[:] = [float(v) for v in h]
    return loc


def _iso_inverse(iso7):
    qi = np.array([-iso7[3], -iso7[4], -iso7[5], iso7[6]])
    t = iso_apply([0.0, 0.0, 0.0, qi[0], qi[1], qi[2], qi[3]], -np.asarray(iso7[:3], np.float64).reshape(1, 3))[0]
    return [t[0], t[1], t[2], qi[0], qi[1], qi[2], qi[3]]


def obb_cases(Loc, nodes, P):
    """Axis-aligned and rotated boxes whose half extent on one axis is |q| of a chosen point (in) or one ulp less (out)."""
    out = []
    for enc, first, cnt, cube in nodes:
        Q = P[first:first + cnt]
        centre = Q[len(Q) // 3] + cube[3] * np.array([0.11, -0.07, 0.05])
        s, c = math.sin(0.3 + 0.2 * enc), math.cos(0.3 + 0.2 * enc)
        ax = np.array([1.0, -2.0, 0.5 + enc]) / np.linalg.norm([1.0, -2.0, 0.5 + enc])
        for rot, quat in (("aligned", [0.0, 0.0, 0.0, 1.0]), ("rotated", [ax[0] * s, ax[1] * s, ax[2] * s, c])):
            iso = [centre[0], centre[1], centre[2]] + list(quat)
            inv = _iso_inverse(iso)
            q = np.abs(iso_apply(inv, Q))
            k = (enc + (rot == "rotated")) % 3
            j = int(np.argsort(q[:, k])[len(Q) // 2])  # a point half way out on axis k
            wide = np.full(3, 4.0 * cube[3])
            for label, hk in (("in", q[j, k]), ("out", np.nextafter(q[j, k], 0.0))):
                h = wide.copy()
                h[k] = hk
                loc = _obb(Loc, iso, inv, h)
                qa = np.abs(iso_apply(inv, P))
                others = np.all(np.delete(qa <= h, k, 1), 1)
                if label == "in":
                    lab = {"obb_face_in": np.flatnonzero(others & (qa[:, k] == h[k]))}
                else:
                    lab = {"obb_face_out": np.flatnonzero(others & (qa[:, k] == q[j, k]))}
                out.append(("obb_%s_%s_enc%d" % (rot, label, enc), loc, lab))
    return out


def _binade_scale(v):
    """2^-e with every |v| * 2^-e in [0.5, 1), so that v * 2^-e is exact and its ulp is 2^-53."""
    e = math.frexp(float(np.max(np.abs(v))))[1]
    s = 2.0 ** -e
    assert np.all(np.abs(v) * s >= 0.5), "the cloud spans more than one binade on an axis"
    return s


def frustum_loc(Loc, M):
    """geometry.frustum_from_matrix4 on this module's Location type: clip_from_query = M, query_from_clip = inverse(M)."""
    M = np.asarray(M, np.float64)
    loc = Loc()
    loc.kind = LOC_FRUSTUM
    loc.clip_from_query[:] = [float(v) for v in M.T.reshape(-1)]
    loc.query_from_clip[:] = [float(v) for v in np.linalg.inv(M).T.reshape(-1)]
    return loc


def frustum_labels(loc, P):
    r, w = clip(_col(loc, "clip_from_query", 16), P)
    aw, ar = np.abs(w), np.abs(r)
    T = aw * T_FACTOR
    lab = {}
    normal = (aw > 1e-290) & (aw < 1e300)
    tiny, huge = (aw > 0) & (aw <= 1e-290), aw >= 1e300
    inside = np.all(ar < aw[:, None], 1)
    edge = inside | np.all(ar <= aw[:, None], 1) & np.any(ar == aw[:, None], 1)
    on_w = edge & ~inside  # some |r| == |w|, the rest within
    band = inside & np.any(ar > T[:, None], 1)
    lab["frustum_r_eq_w"] = np.flatnonzero(normal & on_w)
    lab["frustum_band"] = np.flatnonzero(normal & band)
    lab["frustum_w_neg_in"] = np.flatnonzero(normal & (w < 0) & inside)
    lab["frustum_tiny_w_edge"] = np.flatnonzero(tiny & on_w)
    lab["frustum_tiny_w_in"] = np.flatnonzero(tiny & band)
    lab["frustum_huge_w_edge"] = np.flatnonzero(huge & on_w)
    lab["frustum_huge_w_in"] = np.flatnonzero(huge & band)
    w0 = w == 0.0
    lab["frustum_w0_in"] = np.flatnonzero(w0 & np.all(ar < 1.0, 1))
    lab["frustum_w0_edge"] = np.flatnonzero(w0 & np.all(ar <= 1.0, 1) & np.any(ar == 1.0, 1))
    return {k: v for k, v in lab.items() if len(v)}


def frustum_cases(Loc, nodes, P, perspective=()):
    """Orthographic-like clip matrices whose plane on one axis passes exactly through a chosen point (r == +-w, or one double
    inside: the band), with w = +-1, scaled by 2^-980 and 2^1000 (tiny / huge w: the divisions decide), and a matrix whose w
    row vanishes on a plane of points (w == 0: r is tested undivided) with r == +-1 on some of them."""
    scale = [_binade_scale(P[:, k]) for k in range(3)]
    out = []
    for enc, first, cnt, cube in nodes:
        Q = P[first:first + cnt]
        j = first + len(Q) // 2
        p = P[j]
        k = enc % 3
        for target, sign in ((1.0, 1.0), (-1.0, -1.0), (ONE_MINUS, 1.0), (-ONE_MINUS, -1.0)):
            M = np.zeros((4, 4))
            for i in range(3):
                if i == k:
                    M[i, i] = sign * scale[i]
                    M[i, 3] = target - sign * scale[i] * p[i]  # exact: Sterbenz
                else:  # the other axes: (x - p) 2^-e, far inside for every point of the cloud
                    M[i, i] = scale[i]
                    M[i, 3] = -scale[i] * p[i]
            for wname, wv in (("w+", 1.0), ("w-", -1.0)):
                Mw = M.copy() * wv
                Mw[3, 3] = wv
                base = "frustum_enc%d_t%+.0f%s_%s" % (enc, target, "" if abs(target) == 1.0 else "band", wname)
                out.append((base, frustum_loc(Loc, Mw)))
                if wname == "w+":
                    out.append((base + "_tiny", frustum_loc(Loc, Mw * 2.0 ** -980)))
                    out.append((base + "_huge", frustum_loc(Loc, Mw * 2.0 ** 1000)))
        # w == 0 on the plane x[a] == p[a]: w = (x[a] - p[a]) 2^-e exactly, r tested undivided.  The corners put the location on both
        # sides of the plane, and at w == 0 it spans |r0| < 0.9: centred (r0 = 0 at p) the plane's points are in nodes the location
        # visits; with r0 = +-1 exactly at a second point of the plane they are not (the point test alone sees them).
        a = (k + 1) % 3
        b, c = (a + 1) % 3, (a + 2) % 3
        plane = np.flatnonzero(Q[:, a] == _common_value(Q[:, a]))
        p = Q[plane[0]]
        vals = Q[plane, b]
        kk = plane[np.argmax(vals)] if vals.max() > vals.min() else plane[0]
        for target, sign in ((0.0, 1.0), (1.0, 1.0), (-1.0, -1.0)):
            M = np.zeros((4, 4))
            M[3, a] = scale[a]
            M[3, 3] = -scale[a] * p[a]
            M[0, b] = sign * scale[b]
            M[0, 3] = target - sign * scale[b] * (Q[kk, b] if target else p[b])
            M[1, c] = scale[c]
            M[1, 3] = -scale[c] * p[c]
            M[2, a] = -0.1 * scale[a]
            M[2, c] = scale[c]
            M[2, 3] = 0.9 + 0.1 * scale[a] * p[a] - scale[c] * p[c]
            out.append(("frustum_enc%d_w0_r%+.0f" % (enc, target), frustum_loc(Loc, M)))
    out += list(perspective)
    return [(nm, loc, frustum_labels(loc, P)) for nm, loc in out]


def perspective_frusta(G, Loc, nodes, P):
    """Perspective frusta looking at the anchor nodes (geometry.frustum), copied into `Loc`."""
    out = []
    for enc, first, cnt, cube in nodes:
        e = cube[3]
        target = P[first + cnt // 2]
        eye = target + np.array([0.3, -0.2, 3.0]) * 4 * e
        q = G.quat_from_axis_angle([1.0, 0.2, 0.0], 0.1)
        loc = G.frustum(G.Isometry(eye, q), G.Perspective.new_fov(1.3, 1.1, 0.5 * e, 40 * e))
        o = Loc()
        for f, _ in Loc._fields_:
            setattr(o, f, getattr(loc, f))
        out.append(("perspective_enc%d" % enc, o))
    return out


def edge_locations(Loc, tree_nodes, order, P, G=None):
    """Every boundary location of the tree: [(name, loc, {label class: point indices into P})]."""
    nodes = anchors(tree_nodes, order, P)
    persp = perspective_frusta(G, Loc, nodes, P) if G is not None else ()
    return aabb_cases(Loc, nodes, P) + obb_cases(Loc, nodes, P) + frustum_cases(Loc, nodes, P, persp)
