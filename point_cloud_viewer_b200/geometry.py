"""Host-side constructors of the culling geometries, mirroring the reference's public constructors
(setup code that runs once per query on the host; the per-node / per-point work runs in CUDA).

  Aabb::new                src/geometry/aabb.rs:19-24
  Perspective::new/inverse src/geometry/frustum.rs:17-78   (and Perspective3 via new_fov, :185-203)
  Frustum::new             src/geometry/frustum.rs:101-108
  Frustum::from_matrix4    src/geometry/frustum.rs:111-117
  Obb::new / From<&Aabb> / transformed   src/geometry/obb.rs:19-45
  WebMercatorRect::from_zoomed_coordinates   src/geometry/web_mercator_rect.rs:40-53 (in the library: pcv_web_mercator_rect)
  Isometry3 (translation + unit quaternion i,j,k,w) algebra as in nalgebra 0.22.

Matrices are numpy (4,4) row/col indexed [r, c]; they are flattened column-major (nalgebra storage)
when written into a Location.
"""
import ctypes as C
import math

import numpy as np

from . import _native as _N
from ._native import CellUnion as _NativeCellUnion
from ._native import Location

LOC_ALL, LOC_AABB, LOC_FRUSTUM, LOC_OBB, LOC_WEB_MERCATOR_RECT = 0, 1, 2, 3, 4


# ---- isometries ---------------------------------------------------------------------------------
def quat_from_axis_angle(axis, angle):
    axis = np.asarray(axis, np.float64)
    axis = axis / math.sqrt(float(axis @ axis))
    s, c = math.sin(angle / 2.0), math.cos(angle / 2.0)
    return np.array([axis[0] * s, axis[1] * s, axis[2] * s, c])


def quat_mul(a, b):
    ai, aj, ak, aw = a
    bi, bj, bk, bw = b
    return np.array(
        [
            aw * bi + ai * bw + aj * bk - ak * bj,
            aw * bj - ai * bk + aj * bw + ak * bi,
            aw * bk + ai * bj - aj * bi + ak * bw,
            aw * bw - ai * bi - aj * bj - ak * bk,
        ]
    )


def quat_rotate(q, p):
    qv = np.asarray(q[:3], np.float64)
    p = np.asarray(p, np.float64)
    t = np.cross(qv, p) * 2.0
    return t * q[3] + np.cross(qv, t) + p


class Isometry:
    """translation + unit quaternion (i, j, k, w)."""

    def __init__(self, translation=(0.0, 0.0, 0.0), quaternion=(0.0, 0.0, 0.0, 1.0)):
        self.t = np.asarray(translation, np.float64).copy()
        self.q = np.asarray(quaternion, np.float64).copy()

    def inverse(self):
        qi = np.array([-self.q[0], -self.q[1], -self.q[2], self.q[3]])
        return Isometry(quat_rotate(qi, -self.t), qi)

    def __mul__(self, other):
        return Isometry(self.t + quat_rotate(self.q, other.t), quat_mul(self.q, other.q))

    def transform_point(self, p):
        return quat_rotate(self.q, p) + self.t

    def to_homogeneous(self):
        i, j, k, w = self.q
        ww, ii, jj, kk = w * w, i * i, j * j, k * k
        ij, wk, wj, ik, jk, wi = i * j * 2.0, w * k * 2.0, w * j * 2.0, i * k * 2.0, j * k * 2.0, w * i * 2.0
        m = np.eye(4)
        m[:3, :3] = [
            [ww + ii - jj - kk, ij - wk, wj + ik],
            [wk + ij, ww - ii + jj - kk, jk - wi],
            [ik - wj, wi + jk, ww - ii - jj + kk],
        ]
        m[:3, 3] = self.t
        return m

    def as7(self):
        return [self.t[0], self.t[1], self.t[2], self.q[0], self.q[1], self.q[2], self.q[3]]


# ---- perspective --------------------------------------------------------------------------------
class Perspective:
    def __init__(self, left, right, bottom, top, near, far):
        assert left < right and bottom < top and near > 0.0 and near < far
        m = np.zeros((4, 4))
        m[0, 0] = (2.0 * near) / (right - left)
        m[0, 2] = (right + left) / (right - left)
        m[1, 1] = (2.0 * near) / (top - bottom)
        m[1, 2] = (top + bottom) / (top - bottom)
        m[2, 2] = -(far + near) / (far - near)
        m[2, 3] = -(2.0 * far * near) / (far - near)
        m[3, 2] = -1.0
        self.matrix = m

    @classmethod
    def new_fov(cls, aspect, fovy, near, far):
        ymax = near * math.tan(fovy * 0.5)
        xmax = ymax * aspect
        return cls(-xmax, xmax, -ymax, ymax, near, far)

    def inverse(self):
        m = self.matrix
        r = np.zeros((4, 4))
        r[0, 0] = 1.0 / m[0, 0]
        r[0, 3] = m[0, 2] / m[0, 0]
        r[1, 1] = 1.0 / m[1, 1]
        r[1, 3] = m[1, 2] / m[1, 1]
        r[2, 3] = -1.0
        r[3, 2] = 1.0 / m[2, 3]
        r[3, 3] = m[2, 2] / m[2, 3]
        return r


def _colmajor(m):
    return [float(v) for v in np.asarray(m, np.float64).T.reshape(-1)]


# ---- locations ------------------------------------------------------------------------------------
def all_points():
    loc = Location()
    loc.kind = LOC_ALL
    return loc


def aabb(mins, maxs):
    a, b = np.asarray(mins, np.float64), np.asarray(maxs, np.float64)
    loc = Location()
    loc.kind = LOC_AABB
    loc.aabb_min[:] = list(np.minimum(a, b))
    loc.aabb_max[:] = list(np.maximum(a, b))
    return loc


def frustum(query_from_eye, clip_from_eye):
    """Frustum::new(query_from_eye: Isometry3, clip_from_eye: Perspective)."""
    clip_from_query = clip_from_eye.matrix @ query_from_eye.inverse().to_homogeneous()
    query_from_clip = query_from_eye.to_homogeneous() @ clip_from_eye.inverse()
    loc = Location()
    loc.kind = LOC_FRUSTUM
    loc.clip_from_query[:] = _colmajor(clip_from_query)
    loc.query_from_clip[:] = _colmajor(query_from_clip)
    return loc


def frustum_from_matrix4(clip_from_query):
    m = np.asarray(clip_from_query, np.float64)
    inv = np.linalg.inv(m)
    loc = Location()
    loc.kind = LOC_FRUSTUM
    loc.clip_from_query[:] = _colmajor(m)
    loc.query_from_clip[:] = _colmajor(inv)
    return loc


def obb(query_from_obb, half_extent):
    loc = Location()
    loc.kind = LOC_OBB
    loc.query_from_obb[:] = query_from_obb.as7()
    loc.obb_from_query[:] = query_from_obb.inverse().as7()
    loc.half_extent[:] = [float(v) for v in half_extent]
    return loc


def web_mercator_rect(min_xy, max_xy, z):
    """WebMercatorRect::from_zoomed_coordinates(min, max, z): the points whose map position at zoom z lies in [min, max), in
    pixels of the 256 * 2^z map (x east, y south).  x may wrap around the antimeridian (min.x > max.x), which selects nodes but no
    point.  ValueError where the reference returns None: z > 23, a corner outside [0, 256 * 2^z), max.y < min.y, more than one
    zoom-0 pixel across, or a non-finite value."""
    mn = (C.c_double * 2)(*[float(v) for v in min_xy])
    mx = (C.c_double * 2)(*[float(v) for v in max_xy])
    loc = Location()
    try:
        _N.check(_N.lib().pcv_web_mercator_rect(mn, mx, int(z), C.byref(loc)))
    except _N.PcvError as e:
        raise ValueError(str(e)) from None
    return loc


def web_mercator_coord(ecef, z):
    """WebMercatorCoord::from_lat_lng(ECEF -> WGS84).to_zoomed_coordinate(z): the map position (x, y) of an ECEF point at zoom z,
    in [0, 256 * 2^z).  ValueError for z > 23."""
    p = (C.c_double * 3)(*[float(v) for v in ecef])
    out = (C.c_double * 2)()
    try:
        _N.check(_N.lib().pcv_web_mercator_coord(p, int(z), out))
    except _N.PcvError as e:
        raise ValueError(str(e)) from None
    return out[0], out[1]


class CellUnion:
    """PointLocation::S2Cells (src/iterator.rs:13-20): the points whose leaf cell the union of S2 cells `ids` contains.  Not a
    pcv_location: Octree / OctreeDir queries dispatch it to the pcv_*cell_union* entry points, which validate and normalise the
    ids."""

    def __init__(self, ids):
        self.ids = np.ascontiguousarray(np.asarray(ids, np.uint64).reshape(-1))

    def struct(self):
        """The pcv_cell_union view of the ids (valid while this object lives)."""
        return _NativeCellUnion(self.ids.ctypes.data if len(self.ids) else None, len(self.ids), 0)


def cell_union(ids):
    return CellUnion(ids)


def obb_from_aabb(mins, maxs):
    a, b = np.asarray(mins, np.float64), np.asarray(maxs, np.float64)
    return Isometry((a + b) * 0.5), (b - a) * 0.5


def obb_from_aabb_transformed(mins, maxs, global_from_query):
    iso, half = obb_from_aabb(mins, maxs)
    return obb(global_from_query * iso, half)
