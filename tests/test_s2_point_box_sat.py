"""The cell test of the S2 cloud's location queries (csrc/geometry_host.hpp: sat_box, the separating-axis test of a location
against a cell's point box), through the TEST-ONLY sequential driver tests/cpu_backend/s2_box_cpu.cpp (built into
_build/libtbb.so), against the oracle's cache_separating_axes_for_aabb + intersect (orc_cached_intersect_aabb): equal for every
box.  The locations are the point_cloud_test queries at the slab pose plus random OBBs and frusta at ECEF scale; the boxes are
random, touch a face or a corner of the location exactly, are flat or a single point, or contain the location."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

import oracle_api as O

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpu_backend", "_build", "libtbb.so")
_tbb = None


def _tb():
    global _tbb
    if _tbb is None:
        L = C.CDLL(_SO)
        L.tbb_sat_box.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        _tbb = L
    return _tbb


def _oloc(loc):
    o = O.Location()
    for f, _ in O.Location._fields_:
        setattr(o, f, getattr(loc, f))
    return o


def sat_box(loc, mn, mx):
    mn = np.ascontiguousarray(mn, np.float64).reshape(-1, 3)
    mx = np.ascontiguousarray(mx, np.float64).reshape(-1, 3)
    out = np.zeros(len(mn), np.int32)
    o = _oloc(loc)
    _tb().tbb_sat_box(C.addressof(o), mn.ctypes.data, mx.ctypes.data, len(mn), out.ctypes.data)
    return out


def oracle(loc, mn, mx):
    L, o = O.lib(), _oloc(loc)
    return np.array([L.orc_cached_intersect_aabb(C.byref(o), O._d(a), O._d(b)) for a, b in zip(mn, mx)], np.int32)


def corners(loc):
    out = (C.c_double * 24)()
    O.lib().orc_location_corners(C.byref(_oloc(loc)), out)
    return np.array(out).reshape(8, 3)


def _locations():
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    bmin, bmax, _ = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    bmin, bmax = np.asarray(bmin, np.float64), np.asarray(bmax, np.float64)
    d = bmax - bmin
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    ecef_from_local = G.Isometry((4157222.543, 664789.307, 4774952.099), q)
    locs = {  # point_cloud_test/src/queries.rs at the slab pose, as in test_query_gpu.py
        "aabb": G.aabb(bmin + 0.2 * d, bmin + 0.8 * d),
        "obb": G.obb(ecef_from_local, (50.0, 50.0, 5.0)),
        "frustum": G.frustum(ecef_from_local, G.Perspective.new_fov(1.0, 1.2, 0.1, 10.0)),
        "frustum_far": G.frustum(ecef_from_local * G.Isometry((0, 0, 0), G.quat_from_axis_angle([1, 0.3, 0], 1.3)), G.Perspective.new_fov(1.3, 0.9, 0.5, 150.0)),
    }
    rng = np.random.default_rng(20261016)
    for k in range(6):  # random poses on the Earth's surface
        lat, lon = rng.uniform(-1.4, 1.4), rng.uniform(-3.1, 3.1)
        t = 6371000.0 * np.array([np.cos(lat) * np.cos(lon), np.cos(lat) * np.sin(lon), np.sin(lat)])
        pose = G.Isometry(tuple(t), G.quat_from_axis_angle(rng.normal(size=3), rng.uniform(0, np.pi)))
        locs["obb_%d" % k] = G.obb(pose, tuple(rng.uniform(0.5, 200.0, 3)))
        locs["frustum_%d" % k] = G.frustum(pose, G.Perspective.new_fov(rng.uniform(0.5, 2.0), rng.uniform(0.3, 1.5), rng.uniform(0.05, 2.0), rng.uniform(5.0, 500.0)))
    return locs


def _boxes(loc, rng):
    """(mn, mx) pairs around the location: random, touching its faces / corners exactly, flat, single points, containing it."""
    c = corners(loc)
    lo, hi = c.min(0), c.max(0)
    span = float(np.max(hi - lo))
    mn, mx = [], []

    def add(a, b):
        mn.append(np.minimum(a, b))
        mx.append(np.maximum(a, b))

    for _ in range(400):  # random boxes of every size near the location
        p = lo + rng.uniform(-0.5, 1.5, 3) * (hi - lo)
        add(p, p + rng.uniform(0, 1, 3) * span * rng.choice([1e-3, 0.1, 1.0]))
    for k in range(8):  # a box with its max (or min) corner exactly at a location corner, and a point box there
        add(c[k], c[k] + span * 0.1)
        add(c[k] - span * 0.1, c[k])
        add(c[k], c[k])
    for a in range(3):  # boxes whose face lies exactly on the location's extreme coordinate on each axis
        for side, v in ((0, lo[a]), (1, hi[a])):
            b0, b1 = lo.copy() - span, hi.copy() + span
            if side == 0:
                b1[a] = v
            else:
                b0[a] = v
            add(b0, b1)
            flat0, flat1 = b0.copy(), b1.copy()
            flat0[a] = flat1[a] = v  # flat box in the plane of that coordinate
            add(flat0, flat1)
    for _ in range(50):  # flat and point boxes inside / around the location
        p = lo + rng.uniform(0, 1, 3) * (hi - lo)
        q = p + rng.uniform(0, 1, 3) * span * 0.2
        q[rng.integers(3)] = p[rng.integers(3)] if rng.random() < 0.5 else q[0]
        add(p, q)
        add(p, p)
    add(lo - span, hi + span)  # contains the location
    add(lo, hi)  # the location's own bounding box
    add(lo - 1e7, hi + 1e7)
    return np.array(mn), np.array(mx)


@pytest.mark.parametrize("name", list(_locations()))
def test_sat_box_equals_oracle(name):
    loc = _locations()[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    mn, mx = _boxes(loc, rng)
    got, want = sat_box(loc, mn, mx), oracle(loc, mn, mx)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, (name, len(bad), mn[bad[:3]], mx[bad[:3]], got[bad[:3]], want[bad[:3]])
    assert set(want.tolist()) >= {1, 2}, (name, np.bincount(want))  # the fuzz reaches Cross and Out


def test_sat_box_all_points_and_aabb_faces():
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    assert sat_box(G.all_points(), [[0, 0, 0]], [[1, 1, 1]]).tolist() == [0]
    a = G.aabb((1.0, 2.0, 3.0), (4.0, 5.0, 6.0))
    mn = np.array([[4.0, 2.0, 3.0], [0.0, 0.0, 0.0], [2.0, 3.0, 4.0], [0.0, 0.0, 0.0], [np.nextafter(4.0, 5.0), 2.0, 3.0], [1.0, 2.0, 3.0]])
    mx = np.array([[5.0, 3.0, 4.0], [1.0, 2.0, 3.0], [3.0, 4.0, 5.0], [9.0, 9.0, 9.0], [5.0, 3.0, 4.0], [4.0, 5.0, 6.0]])
    got = sat_box(a, mn, mx)
    assert got.tolist() == oracle(a, mn, mx).tolist()
    assert got.tolist() == [1, 1, 0, 1, 2, 0]  # touching faces and a touching corner cross, a box just past a face is out
