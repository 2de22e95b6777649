"""Calls that fail, or are cancelled, after they have allocated device memory give every byte back.

The library allocates from the device's default memory pool; CU_MEMPOOL_ATTR_USED_MEM_CURRENT of that pool counts what this
process holds in it, so other users of the GPU do not move it.  Each case runs one successful call of the same shape first (so
that lazily grown state is in place), then compares the counter around the failing call, with the context's cached blocks
released before each reading.  Only numpy host arrays are used between the readings.  Every failure here is detected on the
host: an argument check, a callback's return value or a file-system error."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_IO, ERR_NOT_FOUND, ERR_CANCELLED = -1, -3, -4, -5
CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7


def _pool_used(device=0):
    cu = C.CDLL("libcuda.so.1")
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuInit(0) == 0
    assert cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, C.byref(used)) == 0
    return used.value


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    """The 100k-point ECEF slab, built once with max_points_per_node=3000 and written as an octree directory."""
    import point_cloud_viewer_b200 as pcv

    n = 100_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    c = pcv.Context(0, max_points_per_node=3000)
    d = str(tmp_path_factory.mktemp("octree"))
    tree = c.build_octree(x, y, z, rgb, res, bmin, bmax)
    tree.write_dir(d)
    tree.free()
    yield dict(pcv=pcv, ctx=c, dir=d, x=x, y=y, z=z, rgb=rgb, bmin=bmin, bmax=bmax, res=res)
    c.close()


def _reading(ctx):
    ctx.release_cached_memory()
    return _pool_used()


def _fails(scene, code, call):
    """`call` raises PcvError `code`, and the pool holds as much afterwards as before."""
    ctx = scene["ctx"]
    before = _reading(ctx)
    with pytest.raises(scene["pcv"]._native.PcvError) as e:
        call()
    assert e.value.code == code, str(e.value)
    assert _reading(ctx) == before


def test_build_octree_invalid_resolution(scene):
    s, ctx = scene, scene["ctx"]
    ctx.build_octree(s["x"], s["y"], s["z"], s["rgb"], s["res"], s["bmin"], s["bmax"]).free()
    _fails(s, ERR_INVALID, lambda: ctx.build_octree(s["x"], s["y"], s["z"], s["rgb"], 0.0, s["bmin"], s["bmax"]))


def test_build_octree_from_file_invalid_resolution(scene, tmp_path):
    s, ctx = scene, scene["ctx"]
    n = len(s["x"])
    rec = np.zeros(n, dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    rec["x"], rec["y"], rec["z"] = s["x"], s["y"], s["z"]
    rgb = s["rgb"].reshape(n, 3)
    rec["red"], rec["green"], rec["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    path = tmp_path / "slab.ply"
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty double x\nproperty double y\nproperty double z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n" % n)
    with open(path, "wb") as f:
        f.write(header.encode())
        f.write(rec.tobytes())
    ctx.build_octree_from_file(path, s["res"]).free()
    # the file is on the device when the build rejects the resolution
    _fails(s, ERR_INVALID, lambda: ctx.build_octree_from_file(path, 0.0))


def test_s2_build_point_at_origin(scene):
    s, ctx = scene, scene["ctx"]
    ctx.build_s2_cloud(s["x"], s["y"], s["z"], s["rgb"], split_level=20).free()
    x, y, z = s["x"].copy(), s["y"].copy(), s["z"].copy()
    x[777] = y[777] = z[777] = 0.0  # not a valid ECEF point: found after the keys are computed
    _fails(s, ERR_INVALID, lambda: ctx.build_s2_cloud(x, y, z, s["rgb"], split_level=20))


def test_s2_load_dir_missing_cell(scene, tmp_path):
    s, ctx = scene, scene["ctx"]
    cloud = ctx.build_s2_cloud(s["x"], s["y"], s["z"], s["rgb"], split_level=20)
    d = tmp_path / "s2"
    cloud.write_dir(d)
    cloud.free()
    ctx.load_s2_dir(d).free()
    cells = sorted(p for p in os.listdir(d) if p.endswith(".xyz"))
    assert len(cells) > 2
    os.remove(d / cells[len(cells) // 2])  # the arrays are allocated and the cells before it uploaded
    _fails(s, ERR_NOT_FOUND, lambda: ctx.load_s2_dir(d))


def test_query_points_cancelled(scene):
    s, ctx, pcv = scene, scene["ctx"], scene["pcv"]
    tree = ctx.load_dir(s["dir"])
    try:
        tree.query_points(pcv.geometry.all_points(), batch_size=1000)
        _fails(s, ERR_CANCELLED, lambda: tree.query_points(pcv.geometry.all_points(), callback=lambda b: True, batch_size=1000))
    finally:
        tree.free()


def _xray_shape(s):
    T = 32
    px = float(max(s["bmax"][0] - s["bmin"][0], s["bmax"][1] - s["bmin"][1])) / (8 * T) * 1.01
    return T, px


def test_xray_quadtree_bounded_cancelled(scene):
    s, ctx = scene, scene["ctx"]
    T, px = _xray_shape(s)
    tree = ctx.load_dir(s["dir"])
    try:
        tree.xray_quadtree(T, px, keep_tiles=False)
        _fails(s, ERR_CANCELLED, lambda: tree.xray_quadtree(T, px, keep_tiles=False, on_tile=lambda l, i, img: True))
    finally:
        tree.free()


def test_xray_quadtree_from_dir_cancelled(scene):
    s, ctx = scene, scene["ctx"]
    T, px = _xray_shape(s)
    ctx.xray_quadtree_from_dir(s["dir"], T, px, keep_tiles=False)
    _fails(s, ERR_CANCELLED, lambda: ctx.xray_quadtree_from_dir(s["dir"], T, px, keep_tiles=False, on_tile=lambda l, i, img: True))


def test_dir_query_missing_node_file(scene, tmp_path):
    import shutil

    s, ctx, pcv = scene, scene["ctx"], scene["pcv"]
    d = tmp_path / "octree"
    shutil.copytree(s["dir"], d)
    h = ctx.open_dir(str(d))
    h.query_points(pcv.geometry.all_points(), batch_size=1 << 20)
    h.close()
    before = _reading(ctx)
    h = ctx.open_dir(str(d))
    try:
        files = sorted((os.path.getsize(d / f), f) for f in os.listdir(d) if f.endswith(".xyz"))
        assert len(files) > 2
        os.remove(d / files[-1][1])  # the largest node: every query over all points reads it
        with pytest.raises(pcv._native.PcvError) as e:
            h.query_points(pcv.geometry.all_points(), batch_size=1 << 20)
        assert e.value.code == ERR_NOT_FOUND, str(e.value)
    finally:
        h.close()
    assert _reading(ctx) == before


def test_build_octree_to_dir_unwritable(scene, tmp_path):
    s, ctx = scene, scene["ctx"]
    n = len(s["x"])
    ctx.build_octree_to_dir(tmp_path / "ok", s["x"], s["y"], s["z"], s["rgb"], s["res"], s["bmin"], s["bmax"], max_points_in_core=n // 2)
    blocker = tmp_path / "file"
    blocker.write_bytes(b"")
    # mkdir fails quietly under a regular file; the first node-file write of the first group fails
    _fails(s, ERR_IO, lambda: ctx.build_octree_to_dir(blocker / "out", s["x"], s["y"], s["z"], s["rgb"], s["res"], s["bmin"], s["bmax"],
                                                       max_points_in_core=n // 2))
