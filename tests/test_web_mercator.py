"""PointLocation::WebMercatorRect on the CPU: the shared code of csrc/geometry_host.hpp (compiled by g++ into
tests/cpu_backend/_build/libtbw.so, the same PCV_GHD point test the cull kernels run) against the oracle
(oracle/oracle_web_mercator.hpp, built here into liboracle_wm.so).
- the reference's unit-test facts (tests/golden/web_mercator_facts.json) hold for both;
- ECEF -> WGS84 -> ECEF round trips within 1e-6 m from -500 m to 10 km over all latitudes;
- the constructor rejects what the reference's returns None for, and the product's constructor, validation and geometry equal
  the oracle's bit for bit;
- the point test equals the oracle's bit for bit on 1e6 points, edges at a point's own coordinate included;
- point_cloud_test's check_web_mercator_rect_point_culling_equality on the 1e6-point slab.  No GPU."""
import ctypes as C
import json
import math
import os
import sys

import numpy as np
import pytest

import oracle_api as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_wm.so")
_TBW = os.path.join(ROOT, "tests", "cpu_backend", "_build", "libtbw.so")
FACTS = json.load(open(os.path.join(ROOT, "tests", "golden", "web_mercator_facts.json")))
SEED, N = 80293751232, 1_000_000
SLAB_CENTRE = (4157222.543, 664789.307, 4774952.099)  # the translation of point_cloud_test's ecef_from_local
_libs = {}


def oracle():
    """liboracle_wm.so, built by __graft_entry__.build_oracle (rebuilt here when an oracle source is newer than it)."""
    if "o" not in _libs:
        import __graft_entry__

        __graft_entry__.build_oracle()
        L = C.CDLL(_SO)
        L.orc_load_dir.restype = C.c_void_p
        L.orc_load_dir.argtypes = [C.c_char_p]
        L.orc_num_nodes.restype = C.c_uint64
        L.orc_num_nodes.argtypes = [C.c_void_p]
        L.orc_free.argtypes = [C.c_void_p]
        L.orc_wm_nodes.restype = C.c_int64
        L.orc_wm_query.restype = C.c_int64
        L.orc_wm_query.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64]
        L.orc_wm_nodes.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
        _libs["o"] = L
    return _libs["o"]


class OracleDir:
    """An octree directory loaded by this library's own copy of the oracle (orc_load_dir), so its handle only meets the code
    that made it."""

    def __init__(self, d):
        self.h = oracle().orc_load_dir(str(d).encode())
        if not self.h:
            raise IOError("oracle could not load " + str(d))
        self.num_nodes = int(oracle().orc_num_nodes(self.h))

    def __del__(self):
        if getattr(self, "h", None):
            oracle().orc_free(self.h)
            self.h = None


def backend():
    if "t" not in _libs:
        _libs["t"] = C.CDLL(_TBW)
    return _libs["t"]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f64(a, shape=None):
    a = np.ascontiguousarray(a, np.float64)
    return a if shape is None else a.reshape(shape)


def rect(mn, mx, z, lib=None):
    """(nw.x, nw.y, se.x, se.y) of from_zoomed_coordinates, or None; lib None = the product's constructor."""
    out = np.zeros(4)
    fn = backend().tbw_rect if lib is None else lib.orc_wm_rect
    ok = fn(_p(_f64(mn)), _p(_f64(mx)), C.c_uint32(z), _p(out))
    return out if ok else None


def coords(xyz, lib=None):
    """(normalised map positions, lat / lng) of ECEF points, from the product's shared code or the oracle."""
    xyz = _f64(xyz, (-1, 3))
    w, ll = np.zeros((len(xyz), 2)), np.zeros((len(xyz), 2))
    (backend().tbw_coords if lib is None else lib.orc_wm_coords)(_p(xyz), C.c_uint64(len(xyz)), _p(w), _p(ll))
    return w, ll


def to_ecef(llh, lib=None):
    llh = _f64(llh, (-1, 3))
    out = np.zeros_like(llh)
    (backend().tbw_to_ecef if lib is None else lib.orc_wm_to_ecef)(_p(llh), C.c_uint64(len(llh)), _p(out))
    return out


def to_lat_lng(w, lib=None):
    w = _f64(w, (-1, 2))
    out = np.zeros_like(w)
    (backend().tbw_to_lat_lng if lib is None else lib.orc_wm_to_lat_lng)(_p(w), C.c_uint64(len(w)), _p(out))
    return out


def contains(nw_se, xyz, lib=None):
    xyz = _f64(xyz, (-1, 3))
    out = np.zeros(len(xyz), np.uint8)
    (backend().tbw_contains_n if lib is None else lib.orc_wm_contains_n)(_p(_f64(nw_se)), _p(xyz), C.c_uint64(len(xyz)), _p(out))
    return out.astype(bool)


def geometry(nw_se, lib=None):
    corners, axes = np.zeros(24), np.zeros(3 * 64)
    fn = backend().tbw_geometry if lib is None else lib.orc_wm_geometry
    n = fn(_p(_f64(nw_se)), _p(corners), _p(axes), 64)
    return corners.reshape(8, 3), axes[: 3 * n].reshape(n, 3)


def from_lat_lng(ll):
    ll = _f64(ll, (-1, 2))
    out = np.zeros_like(ll)
    oracle().orc_wm_from_lat_lng(_p(ll), C.c_uint64(len(ll)), _p(out))
    return out


def band_count(w, nw_se, delta=2.0 ** -40):
    """How many of the normalised positions w lie within delta of one of the rect's four edges (the contract's band)."""
    d = np.abs(np.stack([w[:, 0] - nw_se[0], w[:, 0] - nw_se[2], w[:, 1] - nw_se[1], w[:, 1] - nw_se[3]], 1))
    return (d <= delta).any(1)


def slab_points(n=N):
    x, y, z, _ = O.synth_points(1, SEED, 0, n)  # PCV_SYNTH_SLAB_ECEF
    return np.stack([x, y, z], 1)


def slab_rect(zoom=21, half=128.0):
    """queries.rs:59-72: the rect of +-half pixels at `zoom` around the map position of the slab centre."""
    w, _ = coords(np.array([SLAB_CENTRE]))
    c = w[0] * float(256 << zoom)
    return rect(c - half, c + half, zoom)


# ---- the reference's unit-test facts ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lib", ["product", "oracle"])
def test_projection_corners(lib):
    L = None if lib == "product" else oracle()
    for f in FACTS["projection_corners"]:
        # from_lat_lng on latitude / longitude directly: the map corners lie on no ECEF point's round trip
        w = from_lat_lng([[f["lat_rad"], f["lng_rad"]]])[0] if L else None
        if L is None:  # the product's shared function, reached through a point at that latitude / longitude on the ellipsoid
            e = to_ecef([[f["lat_rad"], f["lng_rad"], 0.0]])
            w = coords(e)[0][0]
        assert np.allclose(w * float(256 << f["zoom"]), f["xy"], rtol=0, atol=f["epsilon"]), (lib, w)


def test_projection_roundtrip():
    f = FACTS["projection_roundtrip"]
    lat, lng = f["lat_deg"] * (math.pi / 180.0), f["lng_deg"] * (math.pi / 180.0)
    w = from_lat_lng([[lat, lng]])
    for L in (None, oracle()):
        back = to_lat_lng(w, L)[0]
        assert back[0] == pytest.approx(lat, rel=4e-16, abs=0) and back[1] == pytest.approx(lng, rel=4e-16, abs=0)
    # the same place as an ECEF point at its altitude: the point test's latitude / longitude recover it
    e = to_ecef([[lat, lng, f["alt_m"]]])
    for L in (None, oracle()):
        ll = coords(e, L)[1][0]
        assert abs(ll[0] - lat) < 1e-14 and abs(ll[1] - lng) < 1e-14


def test_projection_ground_truth():
    f = FACTS["projection_ground_truth"]
    e = to_ecef([[f["lat_deg"] * (math.pi / 180.0), f["lng_deg"] * (math.pi / 180.0), f["alt_m"]]])
    for L in (None, oracle()):
        xy = coords(e, L)[0][0] * float(256 << f["zoom"])
        assert np.abs(xy - f["xy"]).max() <= f["epsilon_px"], xy


def test_sagitta():
    f = FACTS["sagitta"]
    for L in (None, oracle()):
        nw_se = rect(f["min"], f["max"], f["zoom"], L)
        ll = to_lat_lng(nw_se.reshape(2, 2), L)
        lat_diff, lng_diff = abs(ll[1, 0] - ll[0, 0]), abs(ll[1, 1] - ll[0, 1])
        assert f["lat_radius_m"] * (1.0 - math.cos(lat_diff / 2.0)) < f["max_m"]
        assert f["lng_radius_m"] * (1.0 - math.cos(lng_diff / 2.0)) < f["max_m"]


def test_wraparound():
    for f in FACTS["wraparound"]:
        for L in (None, oracle()):
            assert (rect(f["min"], f["max"], f["zoom"], L) is not None) == f["some"], f


def test_intersection_relations():
    """rect_a.intersector().intersect(&rect_b.intersector()) (oracle), over polyhedra whose corners and cached axes are the
    product's bit for bit."""
    f = FACTS["intersection"]
    rs = [rect(r["min"], r["max"], r["zoom"], oracle()) for r in f["rects"]]
    names = {0: "In", 1: "Cross", 2: "Out"}
    for a, b, want in f["relations"]:
        assert names[oracle().orc_wm_intersect(_p(rs[a]), _p(rs[b]))] == want
    for r in f["rects"]:
        nw_se = rect(r["min"], r["max"], r["zoom"])
        assert np.array_equal(nw_se, rect(r["min"], r["max"], r["zoom"], oracle()))
        pc, pa = geometry(nw_se)
        oc, oa = geometry(nw_se, oracle())
        assert np.array_equal(pc, oc) and np.array_equal(pa, oa)


# ---- conversions, constructor, geometry -----------------------------------------------------------------------------------
def test_ecef_round_trip_within_a_micrometre():
    rng = np.random.default_rng(5)
    n = 200_000
    lat = np.concatenate([rng.uniform(-math.pi / 2, math.pi / 2, n), [math.pi / 2, -math.pi / 2, 0.0, 1e-9, -1e-9]])
    lng = np.concatenate([rng.uniform(-math.pi, math.pi, n), [0.3, -2.0, math.pi, -math.pi, 0.0]])
    h = np.concatenate([rng.uniform(-500.0, 10000.0, n), [-500.0, 10000.0, 0.0, 5000.0, -500.0]])
    e = to_ecef(np.stack([lat, lng, h], 1))
    w, ll = coords(e)
    back = to_ecef(np.stack([ll[:, 0], ll[:, 1], h], 1))
    assert np.abs(back - e).max() <= 1e-6
    w2, ll2 = coords(e, oracle())
    assert np.array_equal(w, w2) and np.array_equal(ll, ll2)
    assert np.array_equal(to_ecef(np.stack([lat, lng, h], 1), oracle()), e)


@pytest.mark.parametrize("mn,mx,z", [
    ((0.0, 0.0), (1.0, 1.0), 24),                       # z > 23
    ((-1.0, 0.0), (0.5, 0.5), 0),                       # negative
    ((0.0, -0.5), (0.5, 0.5), 3),
    ((0.0, 0.0), (256.0, 0.5), 0),                      # >= 256 * 2^z
    ((10.0, 10.0), (10.5, float(256 << 5)), 5),
    ((0.0, 100.0), (0.5, 99.0), 0),                     # diff.y < 0
    ((10.0, 10.0), (11.5, 10.5), 0),                    # more than one pixel at zoom 0
    ((10.0, 10.0), (10.5, 11.5), 0),
    ((100.0 * 1024, 0.0), (102.0 * 1024, 0.0), 10),
    ((float("nan"), 0.0), (0.5, 0.5), 0),               # NaN / infinite
    ((0.0, 0.0), (0.5, float("nan")), 0),
    ((0.0, 0.0), (float("inf"), 0.5), 0),
])
def test_constructor_rejects(mn, mx, z):
    assert rect(mn, mx, z) is None
    assert rect(mn, mx, z, oracle()) is None


def test_constructor_and_validation_equal_the_oracle():
    """Random corners around every case boundary: same accept / reject, same corners; what the constructor makes is valid, and
    a kind-4 location is valid exactly when some zoom's constructor could have made it."""
    rng = np.random.default_rng(11)
    tb = backend()
    for _ in range(20000):
        z = int(rng.integers(0, 26))
        zoom = float(256 << min(z, 23))
        mn = rng.choice([rng.uniform(-0.1, 1.1) * zoom, rng.uniform(0, zoom), 0.0, zoom - 2.0 ** -20], size=2)
        d = rng.choice([rng.uniform(-1.5, 1.5) * (1 << min(z, 23)), float(1 << min(z, 23)), 0.0, rng.uniform(-300, 300) * (1 << min(z, 23))], size=2)
        mx = mn + d
        a, b = rect(mn, mx, z), rect(mn, mx, z, oracle())
        assert (a is None) == (b is None), (mn, mx, z)
        if a is not None:
            assert np.array_equal(a, b)
            assert tb.tbw_valid(_p(a)) == 1
    for nw_se in ([0.5, 0.5, 0.5 + 1 / 256, 0.5 + 1 / 256], [0.999, 0.2, 0.001, 0.2], [0.5, 0.5, 0.5 + 1.01 / 256, 0.5], [0.5, 0.5, 0.5, 0.4999],
                  [1.0, 0.5, 0.5, 0.5], [0.5, 0.5, 0.5, -0.0], [0.5, float("nan"), 0.5, 0.5], [0.99, 0.5, 0.99 + 1 / 256 - 1, 0.5]):
        want = rect(np.array(nw_se[:2]) * 256, np.array(nw_se[2:]) * 256, 0, oracle()) is not None
        assert tb.tbw_valid(_p(_f64(nw_se))) == int(want), nw_se


def test_geometry_equals_the_oracle():
    """make_query_geom of a kind-4 location: the oracle's corners and cached axes bit for bit, within the 45 the geometry can
    hold; wrapped rects keep their corners unsorted."""
    rng = np.random.default_rng(3)
    most = 0
    for k in range(300):
        z = int(rng.integers(0, 24))
        zoom = float(256 << z)
        mn = rng.uniform(0, zoom, 2)
        mx = mn + rng.uniform(0, 1, 2) * (1 << z) * rng.choice([1.0, 1e-3, 1e-6])
        if k % 10 == 0:
            mx[0] = mx[0] - zoom if mx[0] >= zoom else mx[0]
        mx = np.minimum(mx, np.nextafter(zoom, 0))
        nw_se = rect(mn, mx, z, oracle())
        if nw_se is None:
            continue
        pc, pa = geometry(nw_se)
        oc, oa = geometry(nw_se, oracle())
        assert np.array_equal(pc, oc) and np.array_equal(pa, oa), (mn, mx, z)
        most = max(most, len(pa))
    assert 9 < most <= 45


# ---- the point test -------------------------------------------------------------------------------------------------------
def test_point_test_equals_the_oracle_bit_for_bit():
    """1e6 points (the slab and the whole globe, poles, the antimeridian and latitudes beyond 85.05 degrees) against rects
    around them, and rects whose edges are a point's own coordinate: in on north_west, out on south_east."""
    rng = np.random.default_rng(17)
    slab = slab_points(500_000)
    lat = rng.uniform(-math.pi / 2, math.pi / 2, 500_000)
    lat[:1000] = rng.uniform(1.48, math.pi / 2, 1000) * rng.choice([-1.0, 1.0], 1000)
    lng = rng.uniform(-math.pi, math.pi, 500_000)
    lng[1000:2000] = rng.choice([math.pi, -math.pi, np.nextafter(math.pi, 0)], 1000)
    glob = to_ecef(np.stack([lat, lng, rng.uniform(-1000.0, 20000.0, 500_000)], 1))
    pts = np.concatenate([slab, glob])
    w, _ = coords(pts)
    w2, _ = coords(pts, oracle())
    assert np.array_equal(w, w2)
    rects = [slab_rect(z) for z in (17, 19, 21, 23)] + [np.array([0.9, 0.0, 0.1, 0.003]), np.array([0.999, 0.0, 0.001, 0.0039]),
                                                        np.array([0.5, 0.0, 0.5039, 0.0039])]
    for nw_se in rects:
        a, b = contains(nw_se, pts), contains(nw_se, pts, oracle())
        assert np.array_equal(a, b)
    assert not contains(rects[4], pts).any()  # wrapped
    # edges at points' own coordinates
    for i in rng.integers(0, len(slab), 200):
        wi = w[i]
        on_nw = np.array([wi[0], wi[1], wi[0] + 1e-7, wi[1] + 1e-7])
        on_se = np.array([wi[0] - 1e-7, wi[1] - 1e-7, wi[0], wi[1]])
        on_se_x = np.array([wi[0] - 1e-7, wi[1] - 1e-7, wi[0], wi[1] + 1e-7])
        for r, want in ((on_nw, True), (on_se, False), (on_se_x, False)):
            got = contains(r, pts[i : i + 1])[0]
            assert got == want and got == contains(r, pts[i : i + 1], oracle())[0]


def test_point_culling_equality_on_the_slab():
    """check_web_mercator_rect_point_culling_equality (point_cloud_test/tests/main.rs): on the slab, contains equals SAT-In over
    the polyhedron's face normals for every point, and some point is in."""
    pts = slab_points()
    nw_se = slab_rect()
    got = contains(nw_se, pts)
    sat = np.zeros(len(pts), np.uint8)
    oracle().orc_wm_contains_sat_n(_p(nw_se), _p(_f64(pts)), C.c_uint64(len(pts)), _p(sat))
    assert got.any()
    assert np.array_equal(got, sat.astype(bool)), int((got != sat.astype(bool)).sum())


def test_axes_past_the_record_live_in_its_table():
    """A polyhedron with 12 edges and 6 normals in general position caches all 45 axes (6 + 3 + 12 x 3): the 19 past the 26 a
    location record holds come from its table, in order, and sat_box over all of them equals a numpy restatement of sat()."""
    rng = np.random.default_rng(29)
    unit = lambda v: v / np.linalg.norm(v, axis=-1, keepdims=True)  # noqa: E731
    for _ in range(20):
        corners = rng.normal(0.0, 10.0, (8, 3))
        edges, normals = unit(rng.normal(size=(12, 3))), unit(rng.normal(size=(6, 3)))
        boxes_mn = rng.normal(0.0, 15.0, (400, 3))
        boxes_mx = boxes_mn + rng.uniform(0.1, 20.0, (400, 3))
        axes = np.zeros((45, 3))
        rel = np.zeros(400, np.int32)
        n = backend().tbw_poly_sat_box(_p(_f64(corners)), _p(_f64(edges)), _p(_f64(normals)), _p(axes), _p(_f64(boxes_mn)), _p(_f64(boxes_mx)),
                                       C.c_uint64(400), _p(rel))
        assert n == 45
        want_axes = np.concatenate([normals, np.eye(3), unit(np.cross(edges[:, None, :], np.eye(3)[None, :, :]).reshape(-1, 3))])
        assert np.allclose(axes, want_axes, rtol=0, atol=1e-15)
        ca = corners @ axes.T
        for k in range(400):
            bc = np.array([[(boxes_mx if i & 1 else boxes_mn)[k, 0], (boxes_mx if i & 2 else boxes_mn)[k, 1], (boxes_mx if i & 4 else boxes_mn)[k, 2]]
                           for i in range(8)]) @ axes.T
            amin, amax, bmin, bmax = ca.min(0), ca.max(0), bc.min(0), bc.max(0)
            want = 2 if ((bmin > amax) | (bmax < amin)).any() else (1 if ((amin > bmin) | (bmax > amax)).any() else 0)
            assert rel[k] == want
