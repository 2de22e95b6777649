"""Out-of-core build_octree (pcv_build_octree_to_dir / pcv_build_octree_from_file_to_dir): the directory it writes must be
byte for byte the one the in-core build + write_dir writes for the same input - the same file names, the same .xyz / .rgb /
.intensity bytes, the same meta.pb - whatever the group budget, input layout or encoding."""
import ctypes as C
import filecmp
import os
import shutil

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MAXPTS = 2000


def assert_same_dir(got, want):
    fg, fw = sorted(os.listdir(got)), sorted(os.listdir(want))
    assert fg == fw, (sorted(set(fg) ^ set(fw))[:10], len(fg), len(fw))
    for f in fw:
        assert filecmp.cmp(os.path.join(got, f), os.path.join(want, f), shallow=False), f


@pytest.fixture(scope="module")
def octx():
    import point_cloud_viewer_b200 as pcv

    c = pcv.Context(0, max_points_per_node=MAXPTS)
    yield c
    c.close()


def _cloud(kind, n, seed=5):
    import point_cloud_viewer_b200 as pcv

    x, y, z, rgb = pcv.synth_points_host(kind, seed, 0, n)
    bmin, bmax, res = pcv.synth_bbox(kind)
    return x, y, z, rgb, bmin, bmax, res


def _in_core_dir(ctx, d, x, y, z, rgb, res, bmin, bmax, inten=None, stride=1, n=None):
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten, stride=stride, n=n)
    tree.write_dir(d)
    tree.free()


def _largest_cell(ctx, x, y, z, rgb, res, bmin, bmax, k):
    import torch

    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, y, z)]
    counts = ctx.prefix_histogram_device(dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), len(x), res, bmin, bmax, k)
    return int(np.max(counts))


@pytest.mark.parametrize("with_int", [False, True])
@pytest.mark.parametrize("aos", [False, True])
def test_config2_budgets_match_in_core(octx, tmp_path, with_int, aos):
    import point_cloud_viewer_b200 as pcv

    n = 2_000_000
    x, y, z, rgb, bmin, bmax, res = _cloud(pcv.SYNTH_GAUSS_CLUSTERS, n)
    inten = np.random.default_rng(3).random(n).astype(np.float32) if with_int else None
    if aos:
        flat = np.ascontiguousarray(np.stack([x, y, z], 1)).reshape(-1)
        px, py, pz, stride = flat[0:], flat[1:], flat[2:], 3
    else:
        px, py, pz, stride = x, y, z, 1
    want = tmp_path / "in_core"
    _in_core_dir(octx, want, px, py, pz, rgb, res, bmin, bmax, inten=inten, stride=stride, n=n)
    biggest = _largest_cell(octx, x, y, z, rgb, res, bmin, bmax, 3)
    for budget, many in ((n, False), (n // 3, True), (biggest + 1, True)):
        got = tmp_path / ("ooc_%d" % budget)
        info = octx.build_octree_to_dir(got, px, py, pz, rgb, res, bmin, bmax, intensity=inten, stride=stride, n=n, max_points_in_core=budget)
        assert info["prefix_levels"] == 3 and info["num_points"] == n
        assert (info["groups"] > 1) == many, info
        assert info["largest_group"] <= budget
        assert info["h2d_bytes"] == (1 + info["groups"]) * n * (27 + (4 if with_int else 0))
        assert sum(info["ms_" + p] for p in ("histogram", "select", "build", "write", "top")) <= info["ms_total"] + 1.0
        assert_same_dir(got, want)
        shutil.rmtree(got)


def test_config1_slab_and_float64_encoding(octx, tmp_path):
    import point_cloud_viewer_b200 as pcv

    n = 1_000_000
    x, y, z, rgb, bmin, bmax, res = _cloud(pcv.SYNTH_SLAB_ECEF, n, seed=9)
    _in_core_dir(octx, tmp_path / "a", x, y, z, rgb, res, bmin, bmax)
    info = octx.build_octree_to_dir(tmp_path / "b", x, y, z, rgb, res, bmin, bmax, max_points_in_core=n // 4)
    assert info["groups"] > 1
    assert_same_dir(tmp_path / "b", tmp_path / "a")
    # resolution 1e-6 over the 1024 m cube of config 2: the upper levels are Float64 encoded (wide records)
    x, y, z, rgb, bmin, bmax, _ = _cloud(pcv.SYNTH_GAUSS_CLUSTERS, n, seed=2)
    _in_core_dir(octx, tmp_path / "c", x, y, z, rgb, 1e-6, bmin, bmax)
    info = octx.build_octree_to_dir(tmp_path / "d", x, y, z, rgb, 1e-6, bmin, bmax, max_points_in_core=n // 3)
    assert info["groups"] > 1
    assert_same_dir(tmp_path / "d", tmp_path / "c")


def test_leaf_above_group_level(octx, tmp_path):
    """A few outliers alone in one octant of the root: that level-1 node is a leaf, so the groups are level-1 cells."""
    import point_cloud_viewer_b200 as pcv
    from point_cloud_viewer_b200 import _native as N

    n = 500_000
    x, y, z, rgb, bmin, bmax, res = _cloud(pcv.SYNTH_GAUSS_CLUSTERS, n, seed=4)
    E = float(max(np.asarray(bmax) - np.asarray(bmin)))
    bmax2 = np.asarray(bmin, np.float64) + 2 * E  # the cloud fills octant 0 of the doubled cube
    x[-5:], y[-5:], z[-5:] = bmin[0] + 1.9 * E, bmin[1] + 1.8 * E, bmin[2] + 1.7 * E  # octant 7: five points
    _in_core_dir(octx, tmp_path / "a", x, y, z, rgb, res, bmin, bmax2)
    info = octx.build_octree_to_dir(tmp_path / "b", x, y, z, rgb, res, bmin, bmax2, max_points_in_core=n - 5)
    assert info["prefix_levels"] == 1 and info["groups"] == 2
    assert_same_dir(tmp_path / "b", tmp_path / "a")
    with pytest.raises(N.PcvError) as e:
        octx.build_octree_to_dir(tmp_path / "c", x, y, z, rgb, res, bmin, bmax2, max_points_in_core=n // 3)
    assert e.value.code == -6
    msg = str(e.value)
    assert "r0 holds %d points" % (n - 5) in msg and str(n // 3) in msg and "leaf" in msg, msg


def test_ply_file_matches_in_core(octx, tmp_path):
    from ply_util import write_ply

    n = 1_000_000
    path = tmp_path / "cloud.ply"
    props = [("double", "x"), ("double", "y"), ("double", "z"), ("uchar", "red"), ("uchar", "green"), ("uchar", "blue"), ("float", "intensity")]
    write_ply(path, n, props, np.random.default_rng(7), offset=(4.1e6, 6.6e5, 4.7e6))
    res = 0.001
    tree = octx.build_octree_from_file(path, res, attributes=("color", "intensity"))
    tree.write_dir(tmp_path / "a")
    tree.free()
    info = octx.build_octree_from_file_to_dir(tmp_path / "b", path, res, attributes=("color", "intensity"), max_points_in_core=n // 4)
    assert info["groups"] > 1 and info["prefix_levels"] == 3
    body = n * (3 * 8 + 3 + 4)
    assert info["h2d_bytes"] == (2 + info["groups"]) * body
    assert_same_dir(tmp_path / "b", tmp_path / "a")


def test_edge_inputs(octx, tmp_path):
    import point_cloud_viewer_b200 as pcv
    from point_cloud_viewer_b200 import _native as N

    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_GAUSS_CLUSTERS)
    e = np.zeros(0)
    _in_core_dir(octx, tmp_path / "a", e, e, e, np.zeros(0, np.uint8), res, bmin, bmax, n=0)
    info = octx.build_octree_to_dir(tmp_path / "b", e, e, e, np.zeros(0, np.uint8), res, bmin, bmax, n=0)
    assert info["groups"] == 0 and info["num_nodes"] == 0
    assert_same_dir(tmp_path / "b", tmp_path / "a")
    assert os.listdir(tmp_path / "b") == ["meta.pb"]
    x, y, z, rgb, bmin, bmax, res = _cloud(pcv.SYNTH_GAUSS_CLUSTERS, 10_000)
    blocker = tmp_path / "file"
    blocker.write_bytes(b"")
    with pytest.raises(N.PcvError) as ex:  # a directory below a regular file cannot be created or written
        octx.build_octree_to_dir(blocker / "out", x, y, z, rgb, res, bmin, bmax)
    assert ex.value.code == -3
    L = N.lib()
    d3 = (C.c_double * 3)(*bmin)
    pts = N.Points(x.ctypes.data, y.ctypes.data, z.ctypes.data, 1, rgb.ctypes.data, None, len(x))
    assert L.pcv_build_octree_to_dir(None, C.byref(pts), res, d3, d3, 0, b"/tmp", None) == -1
    assert L.pcv_build_octree_to_dir(octx.h, None, res, d3, d3, 0, b"/tmp", None) == -1
    assert L.pcv_build_octree_to_dir(octx.h, C.byref(pts), res, d3, d3, 0, None, None) == -1
    assert L.pcv_build_octree_from_file_to_dir(octx.h, None, res, 0, 0, b"/tmp", None) == -1
    assert L.pcv_build_octree_from_file_to_dir(octx.h, b"/nonexistent.ply", res, 0, 0, None, None) == -1
    assert L.pcv_in_core_capacity(octx.h, 0, None) == -1
    cap = octx.in_core_capacity()
    assert 0 < cap <= 2 ** 32 - 2 and octx.in_core_capacity(True) <= cap


def test_at_scale_4e8_matches_in_core(tmp_path):
    """4e8 config-2 points in groups of at most 1e8 against the in-core build of the same points."""
    import torch

    import point_cloud_viewer_b200 as pcv

    n, budget = 400_000_000, 100_000_000
    avail_ram = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail_ram < 40e9:
        pytest.skip("needs 40 GB of free host memory, have %.1f GB" % (avail_ram / 1e9))
    free_disk = shutil.disk_usage(tmp_path).free
    if free_disk < 25e9:
        pytest.skip("needs 25 GB of free disk under %s, have %.1f GB" % (tmp_path, free_disk / 1e9))
    kind = pcv.SYNTH_GAUSS_CLUSTERS
    bmin, bmax, res = pcv.synth_bbox(kind)
    ctx = pcv.Context(0)
    x, y, z = (np.empty(n, np.float64) for _ in range(3))
    rgb = np.empty(3 * n, np.uint8)
    step = 50_000_000
    dx, dy, dz = (torch.empty(step, dtype=torch.float64, device="cuda") for _ in range(3))
    drgb = torch.empty(3 * step, dtype=torch.uint8, device="cuda")
    for first in range(0, n, step):
        m = min(step, n - first)
        ctx.synth_points_device(kind, 1, first, m, dx.data_ptr(), dy.data_ptr(), dz.data_ptr(), drgb.data_ptr())
        x[first:first + m], y[first:first + m], z[first:first + m] = dx[:m].cpu().numpy(), dy[:m].cpu().numpy(), dz[:m].cpu().numpy()
        rgb[3 * first:3 * (first + m)] = drgb[:3 * m].cpu().numpy()
    del dx, dy, dz, drgb
    torch.cuda.empty_cache()
    info = ctx.build_octree_to_dir(tmp_path / "b", x, y, z, rgb, res, bmin, bmax, max_points_in_core=budget)
    assert info["groups"] >= 4 and info["largest_group"] <= budget and info["num_points"] == n
    _in_core_dir(ctx, tmp_path / "a", x, y, z, rgb, res, bmin, bmax)
    assert_same_dir(tmp_path / "b", tmp_path / "a")
    ctx.close()


def test_drop_ins_write_out_of_core_above_capacity(octx, tmp_path, monkeypatch):
    """build_octree / build_octree_from_file: a cloud above in_core_capacity goes to the directory out of core (None is returned
    even with a ctx); below it the in-core path returns the resident octree as before."""
    import point_cloud_viewer_b200 as pcv
    from ply_util import write_ply

    n = 300_000
    x, y, z, rgb, bmin, bmax, res = _cloud(pcv.SYNTH_GAUSS_CLUSTERS, n, seed=8)
    batches = [{"position": np.stack([x, y, z], 1)[i:i + 100_000], "color": rgb.reshape(-1, 3)[i:i + 100_000]} for i in range(0, n, 100_000)]
    tree = pcv.build_octree(tmp_path / "a", res, (bmin, bmax), batches, ctx=octx)
    assert tree is not None
    tree.free()
    path = tmp_path / "c.ply"
    write_ply(path, n, [("float", "x"), ("float", "y"), ("float", "z"), ("uchar", "red"), ("uchar", "green"), ("uchar", "blue")], np.random.default_rng(1))
    tree = pcv.build_octree_from_file(tmp_path / "c", 0.01, path, ctx=octx)
    assert tree is not None
    tree.free()
    monkeypatch.setattr(pcv.Context, "in_core_capacity", lambda self, with_intensity=False: n // 2)
    assert pcv.build_octree(tmp_path / "b", res, (bmin, bmax), batches, ctx=octx) is None
    assert_same_dir(tmp_path / "b", tmp_path / "a")
    assert pcv.build_octree_from_file(tmp_path / "d", 0.01, path, ctx=octx) is None
    assert_same_dir(tmp_path / "d", tmp_path / "c")
