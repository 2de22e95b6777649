"""ctypes wrapper around oracle/_build/liboracle.so — TEST INFRASTRUCTURE ONLY.

The oracle is the CPU restatement of the reference algorithm (see oracle/oracle_core.hpp).  Only
tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(_ROOT, "oracle", "_build", "liboracle.so")


def build_oracle(force=False):
    srcs = [os.path.join(_ROOT, "oracle", f) for f in os.listdir(os.path.join(_ROOT, "oracle")) if f.endswith((".cpp", ".hpp"))]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
        subprocess.check_call(["make", "-C", os.path.join(_ROOT, "oracle"), "-s"])
    return _SO


class Location(C.Structure):
    """Same layout as pcv_location in include/pcv.h and orc_location in oracle_capi.cpp."""

    _fields_ = [
        ("kind", C.c_int32),
        ("pad", C.c_int32),
        ("aabb_min", C.c_double * 3),
        ("aabb_max", C.c_double * 3),
        ("clip_from_query", C.c_double * 16),
        ("query_from_clip", C.c_double * 16),
        ("query_from_obb", C.c_double * 7),
        ("obb_from_query", C.c_double * 7),
        ("half_extent", C.c_double * 3),
    ]


class PlyInfo(C.Structure):
    _fields_ = [("num_points", C.c_uint64), ("header_bytes", C.c_uint64), ("record_bytes", C.c_uint32), ("has_color", C.c_int32),
                ("has_intensity", C.c_int32), ("num_fields", C.c_int32), ("offset", C.c_double * 3)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build_oracle()
        L = C.CDLL(_SO)
        dp, u8p, fp, u64p = C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_float), C.POINTER(C.c_uint64)
        L.orc_build.restype = C.c_void_p
        L.orc_build.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_double, dp, dp, C.c_int64, C.c_int]
        L.orc_build_faithful.restype = C.c_double
        L.orc_build_faithful.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_double, dp, dp, C.c_int64, C.c_int,
                                         C.c_char_p, u64p]
        L.orc_synth_points.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_synth_bbox.argtypes = [C.c_int, dp, dp, dp]
        L.orc_build_seconds.restype = C.c_double
        L.orc_build_seconds.argtypes = [C.c_void_p]
        L.orc_free.argtypes = [C.c_void_p]
        L.orc_num_nodes.restype = C.c_uint64
        L.orc_num_nodes.argtypes = [C.c_void_p]
        L.orc_node_info.argtypes = [C.c_void_p, C.c_uint64, u64p, u64p, C.POINTER(C.c_int64), C.POINTER(C.c_int32), dp]
        L.orc_node_data.restype = C.c_int64
        L.orc_node_data.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_bbox.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, dp]
        L.orc_encode.restype = C.c_uint64
        L.orc_encode.argtypes = [C.c_double, C.c_double, C.c_double, C.c_int]
        L.orc_decode.restype = C.c_double
        L.orc_decode.argtypes = [C.c_uint64, C.c_double, C.c_double, C.c_int]
        L.orc_position_encoding.argtypes = [C.c_double, C.c_double]
        L.orc_find_bounding_cube.argtypes = [C.c_uint64, C.c_uint64, dp, C.c_double, dp]
        L.orc_cube_bounding.argtypes = [dp, dp, dp]
        L.orc_child_index.argtypes = [dp, dp]
        L.orc_node_id_from_string.argtypes = [C.c_char_p, u64p, u64p]
        L.orc_node_id_to_string.argtypes = [C.c_uint64, C.c_uint64, C.c_char_p, C.c_int]
        L.orc_node_id_parent.argtypes = [C.c_uint64, C.c_uint64, u64p, u64p, C.POINTER(C.c_int)]
        L.orc_node_id_child.argtypes = [C.c_uint64, C.c_uint64, C.c_int, u64p, u64p]
        L.orc_intersector_intersect.argtypes = [dp, dp, C.c_int, dp, C.c_int, dp, dp, C.c_int, dp, C.c_int]
        LP = C.POINTER(Location)
        L.orc_location_intersect_aabb_generic.argtypes = [LP, dp, dp]
        L.orc_cached_axes.argtypes = [LP, dp, C.c_int]
        L.orc_cached_intersect_aabb.argtypes = [LP, dp, dp]
        L.orc_location_contains.argtypes = [LP, dp]
        L.orc_location_contains_n.argtypes = [LP, C.c_void_p, C.c_uint64, C.c_void_p]
        L.orc_location_contains_sat.argtypes = [LP, dp]
        L.orc_location_corners.argtypes = [LP, dp]
        L.orc_try_inverse.argtypes = [dp, dp]
        L.orc_nodes_in_location.restype = C.c_int64
        L.orc_nodes_in_location.argtypes = [C.c_void_p, LP, C.c_void_p, C.c_int64]
        L.orc_visible_nodes.restype = C.c_int64
        L.orc_visible_nodes.argtypes = [C.c_void_p, dp, C.c_void_p, C.c_int64]
        L.orc_query.restype = C.c_int64
        L.orc_query.argtypes = [C.c_void_p, LP, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
        L.orc_reshuffle.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
        L.orc_query_batch_timed.restype = C.c_double
        L.orc_query_batch_timed.argtypes = [C.c_void_p, LP, C.c_uint32, C.c_int, C.c_uint64, u64p, u64p, u64p]
        L.orc_xray_tile_attr.argtypes = [C.c_void_p, dp, dp, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_int, C.c_void_p]
        L.orc_xray_tile.argtypes = [C.c_void_p, dp, dp, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_xray_tile_attr_binned.argtypes = [C.c_void_p, dp, dp, C.c_uint32, C.c_uint32, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_double, C.c_void_p]
        L.orc_resize_lanczos3.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
        L.orc_build_parent_tile.argtypes = [C.POINTER(C.c_void_p), C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.orc_assign_background.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        L.orc_xray_quadtree_build.restype = C.c_void_p
        L.orc_xray_quadtree_build.argtypes = [C.c_void_p, C.POINTER(XrayQuadtreeParams)]
        L.orc_xray_quadtree_info.argtypes = [C.c_void_p, dp, C.POINTER(C.c_int), u64p]
        L.orc_xray_quadtree_ids.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_xray_quadtree_tile.argtypes = [C.c_void_p, C.c_uint8, C.c_uint64, C.c_void_p]
        L.orc_xray_quadtree_free.argtypes = [C.c_void_p]
        L.orc_write_dir.argtypes = [C.c_void_p, C.c_char_p]
        L.orc_load_dir.restype = C.c_void_p
        L.orc_load_dir.argtypes = [C.c_char_p]
        L.orc_octree_meta.argtypes = [C.c_void_p, dp, dp, C.POINTER(C.c_int)]
        L.orc_nodes_data_blob.restype = C.c_int64
        L.orc_nodes_data_blob.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64]
        L.orc_ply_error.restype = C.c_char_p
        L.orc_ply_open.argtypes = [C.c_char_p, C.POINTER(PlyInfo)]
        L.orc_ply_field.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.orc_ply_read.argtypes = [C.c_char_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_ply_find_bounding_box.argtypes = [C.c_char_p, dp]
        _lib = L
    return _lib


def _d(a):
    return (C.c_double * len(a))(*[float(v) for v in a])


class XrayQuadtreeParams(C.Structure):  # orc_xray_quadtree_params (same layout as the product's pcv_xray_quadtree_params)
    _fields_ = [("strategy", C.c_int32), ("p0", C.c_float), ("p1", C.c_float), ("colormap", C.c_int32), ("bin_size", C.c_double),
                ("has_query_from_global", C.c_int32), ("query_from_global", C.c_double * 7), ("background", C.c_uint8 * 4),
                ("tile_size_px", C.c_uint32), ("pixel_size_m", C.c_double), ("root_level", C.c_uint8), ("root_index", C.c_uint64)]


def resize_lanczos3(img, nw, nh):
    """image 0.23 imageops::resize(.., Lanczos3) restated (oracle_xray_pyramid.hpp).  img: (h, w, 4) uint8."""
    img = np.ascontiguousarray(img, np.uint8)
    out = np.zeros((nh, nw, 4), np.uint8)
    lib().orc_resize_lanczos3(_ptr(img), img.shape[1], img.shape[0], nw, nh, _ptr(out))
    return out


def build_parent_tile(children, background, tile_px, want_mosaic=False):
    """build_parent + resize (xray/src/generation.rs:410-451, 722-759).  children: 4 x (N, N, 4) uint8 or None."""
    child_px = next(c.shape[0] for c in children if c is not None)
    keep = [np.ascontiguousarray(c, np.uint8) if c is not None else None for c in children]
    ptrs = (C.c_void_p * 4)(*[c.ctypes.data if c is not None else None for c in keep])
    bg = np.asarray(background, np.uint8)
    out = np.zeros((tile_px, tile_px, 4), np.uint8)
    mosaic = np.zeros((2 * child_px, 2 * child_px, 4), np.uint8) if want_mosaic else None
    lib().orc_build_parent_tile(ptrs, child_px, _ptr(bg), tile_px, _ptr(out), _ptr(mosaic))
    return (out, mosaic) if want_mosaic else out


def assign_background(rgba, background):
    out = np.ascontiguousarray(rgba, np.uint8).copy()
    bg = np.asarray(background, np.uint8)
    lib().orc_assign_background(_ptr(out), out.size // 4, _ptr(bg))
    return out


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


ENC_BPC = {1: 1, 2: 2, 3: 4, 4: 8}


def id_str(hi, lo):
    buf = C.create_string_buffer(64)
    lib().orc_node_id_to_string(int(hi), int(lo), buf, 64)
    return buf.value.decode()


def id_from_str(s):
    hi, lo = C.c_uint64(), C.c_uint64()
    lib().orc_node_id_from_string(s.encode(), C.byref(hi), C.byref(lo))
    return hi.value, lo.value


class OracleOctree:
    def __init__(self, handle):
        self.h = handle
        L = lib()
        n = L.orc_num_nodes(self.h)
        self.nodes = {}  # "r012" -> dict(num_points, enc, cube, hi, lo)
        self.order = []
        hi, lo, npts, enc = C.c_uint64(), C.c_uint64(), C.c_int64(), C.c_int32()
        cube = (C.c_double * 4)()
        for i in range(n):
            L.orc_node_info(self.h, i, C.byref(hi), C.byref(lo), C.byref(npts), C.byref(enc), cube)
            name = id_str(hi.value, lo.value)
            self.order.append(name)
            self.nodes[name] = dict(num_points=npts.value, enc=enc.value, cube=tuple(cube), hi=hi.value, lo=lo.value)

    def __del__(self):
        try:
            lib().orc_free(self.h)
        except Exception:
            pass

    @property
    def build_seconds(self):
        return lib().orc_build_seconds(self.h)

    def node_data(self, name, with_intensity=False):
        m = self.nodes[name]
        n = m["num_points"]
        bpc = ENC_BPC[m["enc"]]
        xyz = np.zeros(n * 3 * bpc, np.uint8)
        rgb = np.zeros(n * 3, np.uint8)
        inten = np.zeros(n, np.float32) if with_intensity else None
        src = np.zeros(n, np.uint64)
        got = lib().orc_node_data(self.h, m["hi"], m["lo"], _ptr(xyz), _ptr(rgb), _ptr(inten), _ptr(src))
        assert got == n, (name, got, n)
        return xyz, rgb, inten, src

    def nodes_in_location(self, loc):
        cap = len(self.nodes) + 1
        out = np.zeros(2 * cap, np.uint64)
        n = lib().orc_nodes_in_location(self.h, C.byref(loc), _ptr(out), cap)
        return [id_str(out[2 * i], out[2 * i + 1]) for i in range(n)]

    def visible_nodes(self, m16):
        cap = len(self.nodes) + 1
        out = np.zeros(2 * cap, np.uint64)
        n = lib().orc_visible_nodes(self.h, _d(m16), _ptr(out), cap)
        if n < 0:
            raise ValueError("Invalid projection matrix.")
        return [id_str(out[2 * i], out[2 * i + 1]) for i in range(n)]

    def query(self, loc, filters=(), with_intensity=False):
        f = np.asarray(filters, np.float64).reshape(-1)
        nf = len(f) // 2
        tested = C.c_int64()
        n = lib().orc_query(self.h, C.byref(loc), _ptr(f) if nf else None, nf, None, None, None, None, 0, C.byref(tested))
        xyz = np.zeros((n, 3), np.float64)
        rgb = np.zeros((n, 3), np.uint8)
        inten = np.zeros(n, np.float32) if with_intensity else None
        src = np.zeros(n, np.uint64)
        lib().orc_query(self.h, C.byref(loc), _ptr(f) if nf else None, nf, _ptr(xyz), _ptr(rgb), _ptr(inten), _ptr(src), n, C.byref(tested))
        return dict(xyz=xyz, rgb=rgb, intensity=inten, src=src, tested=tested.value)

    def xray_tile_attr(self, bmin, bmax, w, h, mode, p0=0.0, p1=0.0, colormap=0, query_from_global=None):
        rgba = np.zeros((h, w, 4), np.uint8)
        q = _d(query_from_global) if query_from_global is not None else None
        any_ = lib().orc_xray_tile_attr(self.h, _d(bmin), _d(bmax), w, h, q, mode, p0, p1, colormap, _ptr(rgba))
        return bool(any_), rgba

    def xray_tile_attr_binned(self, bmin, bmax, w, h, mode, bin_size, p0=0.0, p1=0.0, query_from_global=None):
        rgba = np.zeros((h, w, 4), np.uint8)
        q = _d(query_from_global) if query_from_global is not None else None
        any_ = lib().orc_xray_tile_attr_binned(self.h, _d(bmin), _d(bmax), w, h, q, mode, p0, p1, float(bin_size), _ptr(rgba))
        return bool(any_), rgba

    def xray_quadtree(self, tile_size_px, pixel_size_m, strategy=0, p0=0.0, p1=0.0, colormap=0, bin_size=0.0, query_from_global=None,
                      background=(255, 255, 255, 255), root=(0, 0)):
        """build_xray_quadtree restated: (info dict, {(level, index): RGBA}) or None when the root id is outside the quadtree."""
        pr = XrayQuadtreeParams()
        pr.strategy, pr.p0, pr.p1, pr.colormap, pr.bin_size = int(strategy), float(p0), float(p1), int(colormap), float(bin_size)
        pr.has_query_from_global = 0 if query_from_global is None else 1
        if query_from_global is not None:
            pr.query_from_global = (C.c_double * 7)(*[float(v) for v in query_from_global])
        pr.background = (C.c_uint8 * 4)(*[int(v) for v in background])
        pr.tile_size_px, pr.pixel_size_m = int(tile_size_px), float(pixel_size_m)
        pr.root_level, pr.root_index = int(root[0]), int(root[1])
        q = lib().orc_xray_quadtree_build(self.h, C.byref(pr))
        if not q:
            return None
        try:
            rect = (C.c_double * 3)()
            deepest, nt = C.c_int(), C.c_uint64()
            lib().orc_xray_quadtree_info(q, rect, C.byref(deepest), C.byref(nt))
            levels = np.zeros(nt.value, np.uint8)
            idx = np.zeros(nt.value, np.uint64)
            lib().orc_xray_quadtree_ids(q, _ptr(levels), _ptr(idx))
            tiles = {}
            for l, i in zip(levels, idx):
                img = np.zeros((tile_size_px, tile_size_px, 4), np.uint8)
                assert lib().orc_xray_quadtree_tile(q, int(l), int(i), _ptr(img)) == 0
                tiles[(int(l), int(i))] = img
            return dict(rect_min_x=rect[0], rect_min_y=rect[1], rect_edge=rect[2], deepest_level=deepest.value, num_nodes=int(nt.value)), tiles
        finally:
            lib().orc_xray_quadtree_free(q)

    def xray_tile(self, bmin, bmax, w, h, query_from_global=None):
        rgba = np.zeros((h, w, 4), np.uint8)
        zbits = np.zeros((h, w, 32), np.uint32)
        zover = np.zeros((h, w), np.uint8)
        q = _d(query_from_global) if query_from_global is not None else None
        any_ = lib().orc_xray_tile(self.h, _d(bmin), _d(bmax), w, h, q, _ptr(rgba), _ptr(zbits), _ptr(zover))
        return bool(any_), rgba, zbits, zover

    def write_dir(self, d):
        assert lib().orc_write_dir(self.h, d.encode()) == 0

    def query_batch_timed(self, locs, num_threads, batch_size=500000):
        """ParallelIterator port over `locs` with `num_threads` workers: dict(seconds, tested, returned, bytes = B_query of SURVEY 8d)."""
        arr = (Location * len(locs))()
        for i, l in enumerate(locs):
            for f, _ in Location._fields_:
                setattr(arr[i], f, getattr(l, f))
        t, r, b = C.c_uint64(), C.c_uint64(), C.c_uint64()
        s = lib().orc_query_batch_timed(self.h, arr, len(locs), int(num_threads), int(batch_size), C.byref(t), C.byref(r), C.byref(b))
        return dict(seconds=s, tested=t.value, returned=r.value, bytes=b.value)

    def nodes_data_blob(self, names):
        """The web viewer's /nodes_data reply for the named nodes (backend.rs:92-165); KeyError(name) if one has no files."""
        ids = np.array([v for nm in names for v in id_from_str(nm)], np.uint64)
        size = lib().orc_nodes_data_blob(self.h, _ptr(ids), len(names), None, 0)
        if size < 0:
            raise KeyError(names[-1 - size])
        out = np.zeros(max(size, 1), np.uint8)
        assert lib().orc_nodes_data_blob(self.h, _ptr(ids), len(names), _ptr(out), size) == size
        return out[:size].tobytes()

    def meta(self):
        res, bb, wi = C.c_double(), (C.c_double * 6)(), C.c_int()
        lib().orc_octree_meta(self.h, C.byref(res), bb, C.byref(wi))
        return res.value, tuple(bb), bool(wi.value)


def build(x, y, z, rgb, resolution, bbox_min, bbox_max, intensity=None, max_points_per_node=100000, num_threads=0, stride=1):
    n = len(rgb) // 3 if rgb.ndim == 1 else rgb.shape[0]
    rgb = np.ascontiguousarray(rgb, np.uint8)
    h = lib().orc_build(n, _ptr(x), _ptr(y), _ptr(z), stride, _ptr(rgb), _ptr(intensity), float(resolution), _d(bbox_min), _d(bbox_max), int(max_points_per_node), int(num_threads))
    return OracleOctree(h)


def build_faithful(x, y, z, rgb, resolution, bbox_min, bbox_max, directory, intensity=None, max_points_per_node=100000, num_threads=0, stride=1):
    """build_octree with the reference's file round trips: node files + meta.pb are left in `directory`.  Returns (seconds, nodes)."""
    n = len(rgb) // 3 if rgb.ndim == 1 else rgb.shape[0]
    rgb = np.ascontiguousarray(rgb, np.uint8)
    nn = C.c_uint64()
    t = lib().orc_build_faithful(n, _ptr(x), _ptr(y), _ptr(z), stride, _ptr(rgb), _ptr(intensity), float(resolution), _d(bbox_min), _d(bbox_max),
                                 int(max_points_per_node), int(num_threads), os.fsencode(directory), C.byref(nn))
    if t < 0:
        raise IOError("oracle faithful build failed in " + directory)
    return t, nn.value


SYNTH_SLAB_ECEF, SYNTH_GAUSS_CLUSTERS = 1, 2


def synth_points(kind, seed, first, n, num_threads=0):
    """The benchmark's input generators (include/pcv_synth.h) on host threads: x, y, z (f64) and rgb (n*3 u8)."""
    n = int(n)
    x, y, z = np.empty(n), np.empty(n), np.empty(n)
    rgb = np.empty(3 * n, np.uint8)
    lib().orc_synth_points(kind, seed, first, n, _ptr(x), _ptr(y), _ptr(z), _ptr(rgb), num_threads)
    return x, y, z, rgb


def synth_bbox(kind):
    mn, mx, res = (C.c_double * 3)(), (C.c_double * 3)(), C.c_double()
    lib().orc_synth_bbox(kind, mn, mx, C.byref(res))
    return np.array(mn), np.array(mx), res.value


def reshuffle(new_order, old_data, bytes_per_vertex):
    """sdl_viewer's reshuffle (node_drawer.rs:34-43)."""
    order = np.ascontiguousarray(new_order, np.uint64)
    old = np.ascontiguousarray(old_data).view(np.uint8).reshape(-1)
    out = np.zeros(len(old), np.uint8)
    rc = lib().orc_reshuffle(_ptr(order), len(order), _ptr(old), len(old), int(bytes_per_vertex), _ptr(out))
    assert rc == 0, rc
    return out


def load_dir(d):
    h = lib().orc_load_dir(d.encode())
    if not h:
        raise IOError("oracle could not load " + d)
    return OracleOctree(h)


def location_contains(loc, xyz):
    """Location::contains of every row of xyz (n, 3) as a bool array."""
    xyz = np.ascontiguousarray(xyz, np.float64).reshape(-1, 3)
    out = np.zeros(len(xyz), np.uint8)
    lib().orc_location_contains_n(C.byref(loc), _ptr(xyz), len(xyz), _ptr(out))
    return out.astype(bool)


def bbox(x, y, z, stride=1):
    out = (C.c_double * 6)()
    n = len(x) if stride == 1 else len(x) // 1
    lib().orc_bbox(n, _ptr(x), _ptr(y), _ptr(z), stride, out)
    return tuple(out)


# ---- PLY input (oracle/oracle_ply.hpp) ----
class PlyError(Exception):
    pass


def ply_open(path):
    info = PlyInfo()
    if lib().orc_ply_open(os.fsencode(path), C.byref(info)) != 0:
        raise PlyError(lib().orc_ply_error().decode())
    return dict(num_points=info.num_points, header_bytes=info.header_bytes, record_bytes=info.record_bytes, has_color=bool(info.has_color),
                has_intensity=bool(info.has_intensity), num_fields=info.num_fields, offset=tuple(info.offset))


def ply_fields(path):
    out = []
    for i in range(ply_open(path)["num_fields"]):
        role, typ, off, nb = C.c_int32(), C.c_int32(), C.c_uint32(), C.c_uint32()
        assert lib().orc_ply_field(os.fsencode(path), i, C.byref(role), C.byref(typ), C.byref(off), C.byref(nb)) == 0
        out.append((role.value, typ.value, off.value, nb.value))
    return out


def ply_read(path, first=0, count=None):
    """Points [first, first + count) as the PointsBatch stream delivers them: x, y, z (offset added), rgb (n, 3) or None, intensity or None."""
    info = ply_open(path)
    if count is None:
        count = info["num_points"] - first
    x, y, z = np.empty(count), np.empty(count), np.empty(count)
    rgb = np.zeros((count, 3), np.uint8) if info["has_color"] else None
    inten = np.zeros(count, np.float32) if info["has_intensity"] else None
    rc = lib().orc_ply_read(os.fsencode(path), first, count, _ptr(x), _ptr(y), _ptr(z), _ptr(rgb) if rgb is not None else None,
                            _ptr(inten) if inten is not None else None)
    if rc != 0:
        raise PlyError(lib().orc_ply_error().decode())
    return x, y, z, rgb, inten


def ply_batches(path, batch_size):
    """PlyIterator::next (ply.rs:522-556): ceil(n / batch_size) batches, the last one short."""
    n = ply_open(path)["num_points"]
    return [ply_read(path, first, min(batch_size, n - first)) for first in range(0, n, batch_size)]


def ply_find_bounding_box(path):
    out = (C.c_double * 6)()
    if lib().orc_ply_find_bounding_box(os.fsencode(path), out) != 0:
        raise PlyError(lib().orc_ply_error().decode())
    return tuple(out[:3]), tuple(out[3:])
