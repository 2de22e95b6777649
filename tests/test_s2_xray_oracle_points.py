"""The oracle's point-list X-ray (oracle/oracle_xray_points.hpp, built here from oracle/oracle_xray_points_capi.cpp) pinned to
its octree X-ray: fed the decoded points of an oracle octree in the octree's order, with the octree's box, it gives the same
quadtree tile for tile and bit for bit, in the global frame and under query_from_global, for every strategy, and the same
single tiles as orc_xray_tile / orc_xray_tile_attr.  Filter intervals are pinned to the same quadtree over the points that pass
them.  No GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_api as O

_ORACLE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle")
_SO = os.path.join(_ORACLE, "_build", "liboracle_points.so")
_lib_points = None


def _lib():
    """liboracle_points.so, compiled with the flags of oracle/Makefile when a source is newer than it."""
    global _lib_points
    if _lib_points is None:
        srcs = [os.path.join(_ORACLE, f) for f in os.listdir(_ORACLE) if f.endswith((".cpp", ".hpp"))]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = _SO + ".%d.tmp" % os.getpid()
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-pthread", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
                                   "-shared", "-o", tmp, os.path.join(_ORACLE, "oracle_xray_points_capi.cpp")])
            os.replace(tmp, _SO)
        L = C.CDLL(_SO)
        L.orc_xray_quadtree_build_points.restype = C.c_void_p
        L.orc_xray_quadtree_build_points.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32,
                                                     C.POINTER(O.XrayQuadtreeParams)]
        L.orc_points_quadtree_info.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
        L.orc_points_quadtree_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_points_quadtree_tile.argtypes = [C.c_void_p, C.c_uint8, C.c_uint64, C.c_void_p]
        L.orc_points_quadtree_free.argtypes = [C.c_void_p]
        dp = C.POINTER(C.c_double)
        L.orc_xray_tile_points.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, dp, dp, C.c_uint32, C.c_uint32, C.c_void_p,
                                           C.c_int, C.c_float, C.c_float, C.c_int, C.c_void_p]
        _lib_points = L
    return _lib_points


def tile_points(xyz, rgb, intensity, tmin, tmax, w, h, mode=0, p0=0.0, p1=0.0, colormap=0, query_from_global=None, filters=()):
    """xray_tile (mode 0) / xray_tile_attr (modes 1-3) of one tile over a point list: (any, RGBA)."""
    xyz = np.ascontiguousarray(xyz, np.float64)
    rgb = None if rgb is None else np.ascontiguousarray(rgb, np.uint8)
    intensity = None if intensity is None else np.ascontiguousarray(intensity, np.float32)
    f = np.ascontiguousarray(np.asarray(filters, np.float64).reshape(-1))
    q = O._d(query_from_global) if query_from_global is not None else None
    rgba = np.zeros((h, w, 4), np.uint8)
    any_ = _lib().orc_xray_tile_points(O._ptr(xyz), O._ptr(rgb), O._ptr(intensity), len(xyz), O._ptr(f) if len(f) else None, len(f) // 2, O._d(tmin),
                                       O._d(tmax), w, h, q, mode, p0, p1, colormap, O._ptr(rgba))
    return bool(any_), rgba


def points_quadtree(xyz, rgb, intensity, bbox6, tile_size_px, pixel_size_m, strategy=0, p0=0.0, p1=0.0, colormap=0, query_from_global=None,
                    background=(255, 255, 255, 255), root=(0, 0), filters=()):
    """build_xray_quadtree over a point list: {(level, index): RGBA}, or None when the root is outside the quadtree."""
    L = _lib()
    pr = O.XrayQuadtreeParams()
    pr.strategy, pr.p0, pr.p1, pr.colormap, pr.bin_size = int(strategy), float(p0), float(p1), int(colormap), 0.0
    pr.has_query_from_global = 0 if query_from_global is None else 1
    if query_from_global is not None:
        pr.query_from_global = (C.c_double * 7)(*[float(v) for v in query_from_global])
    pr.background = (C.c_uint8 * 4)(*[int(v) for v in background])
    pr.tile_size_px, pr.pixel_size_m = int(tile_size_px), float(pixel_size_m)
    pr.root_level, pr.root_index = int(root[0]), int(root[1])
    xyz = np.ascontiguousarray(xyz, np.float64)
    rgb = None if rgb is None else np.ascontiguousarray(rgb, np.uint8)
    intensity = None if intensity is None else np.ascontiguousarray(intensity, np.float32)
    f = np.ascontiguousarray(np.asarray(filters, np.float64).reshape(-1))
    b6 = np.ascontiguousarray(bbox6, np.float64)
    q = L.orc_xray_quadtree_build_points(O._ptr(xyz), O._ptr(rgb), O._ptr(intensity), len(xyz), O._ptr(b6), O._ptr(f) if len(f) else None, len(f) // 2,
                                         C.byref(pr))
    if not q:
        return None
    try:
        rect = (C.c_double * 3)()
        deepest, nt = C.c_int(), C.c_uint64()
        L.orc_points_quadtree_info(q, rect, C.byref(deepest), C.byref(nt))
        levels = np.zeros(nt.value, np.uint8)
        idx = np.zeros(nt.value, np.uint64)
        L.orc_points_quadtree_ids(q, O._ptr(levels), O._ptr(idx))
        tiles = {}
        for lv, i in zip(levels, idx):
            img = np.zeros((tile_size_px, tile_size_px, 4), np.uint8)
            assert L.orc_points_quadtree_tile(q, int(lv), int(i), O._ptr(img)) == 0
            tiles[(int(lv), int(i))] = img
        return dict(rect=tuple(rect), deepest_level=deepest.value), tiles
    finally:
        L.orc_points_quadtree_free(q)


def _qfg(angle=0.6, t=(-3.0, 12.0, 0.5)):
    # a rotation about (0.3, -0.2, 1) and a translation: the quadtree's frame is tilted against the octree's axes
    ax = np.array([0.3, -0.2, 1.0])
    ax /= np.linalg.norm(ax)
    s = np.sin(angle / 2)
    return [t[0], t[1], t[2], ax[0] * s, ax[1] * s, ax[2] * s, np.cos(angle / 2)]


@pytest.fixture(scope="module")
def octree():
    rng = np.random.default_rng(7)
    n = 12000
    # two clusters and a sparse background, so that some leaves stay empty
    xyz = np.concatenate([rng.normal((10, 20, 3), (4, 3, 1), (n // 2, 3)), rng.normal((30, 8, 5), (2, 5, 2), (n // 3, 3)),
                          rng.uniform((0, 0, 0), (40, 30, 10), (n - n // 2 - n // 3, 3))])
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    inten = rng.uniform(0, 100, n).astype(np.float32)
    bmin, bmax = xyz.min(0), xyz.max(0)
    x, y, z = (np.ascontiguousarray(xyz[:, k]) for k in range(3))
    h = O.lib().orc_build(n, O._ptr(x), O._ptr(y), O._ptr(z), 1, O._ptr(rgb), O._ptr(inten), 0.001, O._d(bmin), O._d(bmax), 300, 2)
    oct_ = O.OracleOctree(h)
    loc = O.Location()
    loc.kind = 0
    pts = oct_.query(loc, with_intensity=True)
    _, bb, _ = oct_.meta()
    return oct_, pts, np.array(bb, np.float64)


@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
@pytest.mark.parametrize("frame", [None, "qfg"])
def test_point_list_equals_octree_quadtree(octree, strategy, frame):
    oct_, pts, bb = octree
    q = _qfg() if frame else None
    kw = dict(strategy=strategy, p0={0: 0.0, 1: 0.0, 2: 1.0, 3: 0.5}[strategy], p1={2: 90.0}.get(strategy, 0.0), colormap=1 if strategy == 3 else 0,
              query_from_global=q)
    want = oct_.xray_quadtree(16, 0.25, **kw)
    got = points_quadtree(pts["xyz"], pts["rgb"], pts["intensity"], bb, 16, 0.25, **kw)
    assert want is not None and got is not None
    winfo, wt = want
    ginfo, gt = got
    assert ginfo["deepest_level"] == winfo["deepest_level"] >= 3
    assert ginfo["rect"] == (winfo["rect_min_x"], winfo["rect_min_y"], winfo["rect_edge"])
    assert set(gt) == set(wt)
    assert sum(1 for k in wt if k[0] == winfo["deepest_level"]) < 4 ** winfo["deepest_level"]  # some leaves are empty
    for k in wt:
        assert np.array_equal(gt[k], wt[k]), k


def test_point_list_sub_root_and_background(octree):
    oct_, pts, bb = octree
    for root in [(1, 2), (2, 9)]:
        want = oct_.xray_quadtree(16, 0.25, query_from_global=_qfg(), background=(255, 255, 255, 0), root=root)
        got = points_quadtree(pts["xyz"], pts["rgb"], pts["intensity"], bb, 16, 0.25, query_from_global=_qfg(), background=(255, 255, 255, 0), root=root)
        assert set(got[1]) == set(want[1]) and all(np.array_equal(got[1][k], want[1][k]) for k in want[1])


@pytest.mark.parametrize("frame", [None, "qfg"])
def test_point_list_filters_equal_prefiltered_points(octree, frame):
    _, pts, bb = octree
    q = _qfg() if frame else None
    inten = pts["intensity"].astype(np.float64)
    for filters in [[(10.0, 70.0)], [(10.0, 70.0), (50.0, 95.0)]]:
        keep = np.ones(len(inten), bool)
        for lo, hi in filters:
            keep &= (lo <= inten) & (inten <= hi)
        got = points_quadtree(pts["xyz"], pts["rgb"], pts["intensity"], bb, 16, 0.25, query_from_global=q, filters=filters)[1]
        want = points_quadtree(pts["xyz"][keep], pts["rgb"][keep], pts["intensity"][keep], bb, 16, 0.25, query_from_global=q)[1]
        assert set(got) == set(want) and all(np.array_equal(got[k], want[k]) for k in want)
    # an interval no point passes: no tile at all
    assert points_quadtree(pts["xyz"], pts["rgb"], pts["intensity"], bb, 16, 0.25, query_from_global=q, filters=[(200.0, 300.0)])[1] == {}


@pytest.mark.parametrize("frame", [None, "qfg"])
def test_point_list_tiles_equal_octree_tiles(octree, frame):
    oct_, pts, bb = octree
    q = _qfg() if frame else None
    tmin, tmax = bb[:3] + [6.0, 9.0, 0.0], bb[:3] + [22.0, 25.0, 8.0]
    want = oct_.xray_tile(tmin, tmax, 48, 40, query_from_global=q)
    got = tile_points(pts["xyz"], pts["rgb"], pts["intensity"], tmin, tmax, 48, 40, query_from_global=q)
    assert got[0] == want[0] and np.array_equal(got[1], want[1])
    for mode, p0, p1, cm in [(1, 0.0, 0.0, 0), (2, 1.0, 90.0, 0), (3, 0.5, 0.0, 1)]:
        want = oct_.xray_tile_attr(tmin, tmax, 48, 40, mode, p0, p1, cm, query_from_global=q)
        got = tile_points(pts["xyz"], pts["rgb"], pts["intensity"], tmin, tmax, 48, 40, mode, p0, p1, cm, query_from_global=q)
        assert got[0] == want[0] and np.array_equal(got[1], want[1]), mode
