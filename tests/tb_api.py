"""ctypes wrapper of the TEST-ONLY CPU backend (tests/cpu_backend): runs csrc/build_host.hpp with sequential
stand-ins for the CUDA kernels so the host orchestration can be checked against the oracle without a GPU."""
import ctypes as C
import os

import numpy as np

from point_cloud_viewer_b200._native import NodeMeta
from point_cloud_viewer_b200 import node_name, ENC_BYTES

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpu_backend", "_build", "libtb.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(_SO)
        L.tb_build.restype = C.c_void_p
        L.tb_build.argtypes = [C.c_uint64] + [C.c_void_p] * 3 + [C.c_uint64, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_char_p, C.c_int]
        L.tb_num_nodes.restype = C.c_uint64
        L.tb_num_nodes.argtypes = [C.c_void_p]
        L.tb_nodes.argtypes = [C.c_void_p, C.c_void_p]
        L.tb_xyz_bytes.restype = C.c_uint64
        L.tb_xyz_bytes.argtypes = [C.c_void_p]
        L.tb_passes.restype = C.c_uint32
        L.tb_passes.argtypes = [C.c_void_p]
        L.tb_download.argtypes = [C.c_void_p] * 5
        L.tb_free.argtypes = [C.c_void_p]
        L.tb_level_table.argtypes = [C.c_double, C.c_double, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]
        L.tb_div_unguarded.restype = C.c_double
        L.tb_div_unguarded.argtypes = [C.c_double] * 3
        _lib = L
    return _lib


def level_table(root_edge, resolution, root_min=None):
    """make_level_table (csrc/build_host.hpp) as the build calls it: dict(fast, last_level, enc[41]).  PCV_CHECKED_FAST and
    PCV_NO_POW2 in the environment apply as they do in the library."""
    fast, last = C.c_int(), C.c_int()
    enc = np.zeros(41, np.int8)
    rm = (C.c_double * 3)(*[float(v) for v in root_min]) if root_min is not None else None
    lib().tb_level_table(float(root_edge), float(resolution), rm, C.byref(fast), C.byref(last), enc.ctypes.data)
    return dict(fast=fast.value, last_level=last.value, enc=[int(e) for e in enc])


def div_unguarded(a, b, y):
    """The reciprocal (Markstein) division of chain.h without its range guard."""
    return lib().tb_div_unguarded(float(a), float(b), float(y))


class TbTree:
    def __init__(self, x, y, z, rgb, resolution, bmin, bmax, max_points, G, intensity=None, stride=1):
        L = lib()
        n = len(rgb) // 3
        err = C.create_string_buffer(512)
        h = L.tb_build(n, x.ctypes.data, y.ctypes.data, z.ctypes.data, stride, rgb.ctypes.data, intensity.ctypes.data if intensity is not None else None,
                       float(resolution), (C.c_double * 3)(*[float(v) for v in bmin]), (C.c_double * 3)(*[float(v) for v in bmax]), max_points, G, err, 512)
        if not h:
            raise RuntimeError(err.value.decode())
        nn = L.tb_num_nodes(h)
        arr = (NodeMeta * max(nn, 1))()
        L.tb_nodes(h, arr)
        self.passes = L.tb_passes(h)
        self.has_intensity = intensity is not None
        xb = L.tb_xyz_bytes(h)
        self.xyz, self.rgb, self.src = np.zeros(max(xb, 1), np.uint8), np.zeros(max(3 * n, 1), np.uint8), np.zeros(max(n, 1), np.uint32)
        self.inten = np.zeros(max(n, 1), np.float32) if intensity is not None else None
        L.tb_download(h, self.xyz.ctypes.data, self.rgb.ctypes.data, self.inten.ctypes.data if self.inten is not None else None, self.src.ctypes.data)
        L.tb_free(h)
        self.nodes = {}
        for i in range(nn):
            m = arr[i]
            self.nodes[node_name(m.id_high, m.id_low)] = dict(num_points=m.num_points, enc=m.position_encoding, cube=(m.cube_min[0], m.cube_min[1], m.cube_min[2], m.cube_edge),
                                                              point_offset=m.point_offset, xyz_byte_offset=m.xyz_byte_offset)

    def node_data(self, name):
        m = self.nodes[name]
        n, po, bo, bpc = m["num_points"], m["point_offset"], m["xyz_byte_offset"], ENC_BYTES[m["enc"]]
        return (self.xyz[bo:bo + n * 3 * bpc], self.rgb[3 * po:3 * (po + n)], self.inten[po:po + n] if self.inten is not None else None, self.src[po:po + n].astype(np.uint64))


# ---- sharded build with the test-only stand-ins (used by the gloo world_size-2 test) --------------------------------
def _shard_lib():
    L = lib()
    if not hasattr(L, "_shard_ready"):
        L.tb_prefix_cells.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_double, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.tb_build_sharded.restype = C.c_void_p
        L.tb_build_sharded.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_void_p, C.c_char_p, C.c_int]
        L.tb_assemble_top.restype = C.c_void_p
        L.tb_assemble_top.argtypes = [C.c_double, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_char_p, C.c_int]
        L.tb_nsub.argtypes = [C.c_void_p, C.c_void_p]
        L._shard_ready = True
    return L


class _TbHandleTree:
    """Tree object with the subset of pcv.Octree's interface that distributed.build_sharded uses."""

    def __init__(self, h, n, has_intensity):
        L = _shard_lib()
        nn = L.tb_num_nodes(h)
        arr = (NodeMeta * max(nn, 1))()
        L.tb_nodes(h, arr)
        ns = np.zeros(max(nn, 1), np.uint64)
        L.tb_nsub(h, ns.ctypes.data)
        xb = L.tb_xyz_bytes(h)
        self.has_intensity = has_intensity
        self.xyz, self.rgb, self.src = np.zeros(max(xb, 1), np.uint8), np.zeros(max(3 * n, 1), np.uint8), np.zeros(max(n, 1), np.uint32)
        self.inten = np.zeros(max(n, 1), np.float32) if has_intensity else None
        L.tb_download(h, self.xyz.ctypes.data, self.rgb.ctypes.data, self.inten.ctypes.data if has_intensity else None, self.src.ctypes.data)
        L.tb_free(h)
        self.nodes, self._nsub = {}, {}
        for i in range(nn):
            m = arr[i]
            name = node_name(m.id_high, m.id_low)
            self.nodes[name] = dict(num_points=m.num_points, enc=m.position_encoding, level=m.level, cube=(m.cube_min[0], m.cube_min[1], m.cube_min[2], m.cube_edge),
                                    point_offset=m.point_offset, xyz_byte_offset=m.xyz_byte_offset)
            self._nsub[name] = int(ns[i])

    def node_data(self, name):
        m = self.nodes[name]
        n, po, bo, bpc = m["num_points"], m["point_offset"], m["xyz_byte_offset"], ENC_BYTES[m["enc"]]
        return (self.xyz[bo:bo + n * 3 * bpc], self.rgb[3 * po:3 * (po + n)], self.inten[po:po + n] if self.inten is not None else None, self.src[po:po + n].astype(np.uint64))

    def node_nsub(self, name):
        return self._nsub[name]

    def free(self):
        pass


class TbOps:
    """CPU stand-in for distributed.CudaOps (numpy arrays in, torch CPU tensors on the wire)."""

    def __init__(self, x, y, z, rgb, intensity, resolution, bmin, bmax, max_points, G=2):
        self.x, self.y, self.z, self.rgb, self.intensity = x, y, z, rgb, intensity
        self.res, self.bmin, self.bmax, self.max_points, self.G = resolution, np.asarray(bmin, np.float64), np.asarray(bmax, np.float64), max_points, G
        self.n = len(x)

    def local_bbox(self):
        if self.n == 0:
            return np.full(3, np.inf), np.full(3, -np.inf)
        P = np.stack([self.x, self.y, self.z], 1)
        return P.min(0), P.max(0)

    def _cells(self, k):
        cells = np.zeros(max(self.n, 1), np.uint32)
        _shard_lib().tb_prefix_cells(self.n, self.x.ctypes.data, self.y.ctypes.data, self.z.ctypes.data, 1, float(self.res), self.bmin.ctypes.data, self.bmax.ctypes.data, k, cells.ctypes.data)
        return cells[: self.n]

    def prefix_histogram(self, k):
        return np.bincount(self._cells(k), minlength=8 ** k).astype(np.uint64)

    def pack(self, k, cell_to_rank, nranks, index_base):
        import torch

        dest = np.asarray(cell_to_rank)[self._cells(k)]
        order = np.argsort(dest, kind="stable")
        xyz = torch.from_numpy(np.stack([self.x, self.y, self.z], 1)[order].copy())
        rgb = torch.from_numpy(self.rgb.reshape(-1, 3)[order].copy())
        inten = torch.from_numpy(self.intensity[order].copy()) if self.intensity is not None else None
        idx = torch.from_numpy((index_base + order).astype(np.int64))
        return xyz, rgb, inten, idx, np.bincount(dest, minlength=nranks).astype(np.int64)

    def build_sharded(self, xyz, rgb, inten, k, prefix_counts):
        L = _shard_lib()
        n = xyz.shape[0]
        a = np.ascontiguousarray(xyz.numpy(), np.float64).reshape(-1)
        c = np.ascontiguousarray(rgb.numpy(), np.uint8).reshape(-1)
        i = np.ascontiguousarray(inten.numpy(), np.float32) if inten is not None else None
        pc = np.ascontiguousarray(prefix_counts, np.uint64)
        err = C.create_string_buffer(512)
        if n == 0:
            a, c = np.zeros(3), np.zeros(3, np.uint8)
        h = L.tb_build_sharded(n, a.ctypes.data, c.ctypes.data, i.ctypes.data if i is not None else None, float(self.res), self.bmin.ctypes.data, self.bmax.ctypes.data,
                               self.max_points, self.G, k, pc.ctypes.data, err, 512)
        if not h:
            raise RuntimeError(err.value.decode())
        return _TbHandleTree(h, n, inten is not None)

    def assemble_top(self, k, prefix_counts, unit_nsub, xyz_codes, rgb, inten):
        L = _shard_lib()
        pc, un = np.ascontiguousarray(prefix_counts, np.uint64), np.ascontiguousarray(unit_nsub, np.uint64)
        xyz_codes, rgb = np.ascontiguousarray(xyz_codes, np.uint8), np.ascontiguousarray(rgb, np.uint8)
        n = len(rgb) // 3
        err = C.create_string_buffer(512)
        h = L.tb_assemble_top(float(self.res), self.bmin.ctypes.data, self.bmax.ctypes.data, k, pc.ctypes.data, un.ctypes.data, xyz_codes.ctypes.data, rgb.ctypes.data,
                              inten.ctypes.data if inten is not None else None, n, err, 512)
        if not h:
            raise RuntimeError(err.value.decode())
        return _TbHandleTree(h, n, inten is not None)
