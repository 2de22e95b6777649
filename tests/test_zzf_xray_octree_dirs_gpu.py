"""X-ray quadtrees straight from several octree directories (pcv_xray_quadtree_from_dirs, Context.xray_quadtree_from_dirs).  Three
directories with different boxes, cubes and max_points_per_node - two overlapping parts of the config-1 ECEF slab written with
write_dir, config-2 clusters beside it written by build_octree_to_dir - all with intensities, and a fourth part of the slab
without.  Every tile, the node set, the rect, the levels and the node and leaf counts equal xray_quadtree_clouds over load_dir of
each directory (XRay byte for byte) in the global and local frames, under a sub-root, on a transparent background, with filter
intervals and at budgets from the smallest one accepted up to the default; the directories in another order give the same XRay
tiles; a one-element list equals xray_quadtree_from_dir in tiles, delivery order and every counter; attribute strategies lie in
the xray_attr_ref envelope of the union of the points; write_dir, cancellation, every error row, and one case against the
oracle's point-list quadtree."""
import ctypes as C

import numpy as np
import pytest

import xray_attr_ref as R
from test_s2_xray_oracle_points import points_quadtree

pytestmark = pytest.mark.gpu

T = 32
TRANSPARENT = (255, 255, 255, 0)


def _decoded(pcv, tree):
    """Every point of the octree as AllPoints streams it: decoded f64 positions, colours, intensities (zeros without)."""
    bs = tree.query_points(pcv.geometry.all_points(), batch_size=1 << 20)
    xyz = np.concatenate([b["xyz"] for b in bs])
    it = [np.asarray(b["intensity"]) for b in bs]
    inten = np.concatenate(it).astype(np.float32) if all(v.ndim for v in it) else np.zeros(len(xyz), np.float32)
    return xyz, np.concatenate([b["rgb"] for b in bs]), inten


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    n = 150_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    xyz = np.stack([x, y, z], 1)
    rgb = np.asarray(rgb).reshape(-1, 3)
    inten = ((np.arange(n) * 7919) % 1000).astype(np.float32)
    _, _, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    m = 40_000
    cx, cy, cz, crgb = pcv.synth_points_host(pcv.SYNTH_GAUSS_CLUSTERS, 7, 0, m)
    c = np.stack([cx, cy, cz], 1)
    c = (c - c.min(0)) / np.ptp(c, 0).max()
    ext = xyz.max(0) - xyz.min(0)
    cxyz = xyz.max(0) + np.array([0.05, -0.3, -0.5]) * ext + c * 0.4 * ext
    cinten = ((np.arange(m) * 31) % 1000).astype(np.float32)
    base = tmp_path_factory.mktemp("octree_dirs")
    col = lambda p, k: np.ascontiguousarray(p[:, k])  # noqa: E731
    dirs = [str(base / name) for name in ("a", "b", "c", "bare")]
    # a, b: overlapping parts of the slab, written from resident octrees at 4000 and 1500 points per node
    for d, (lo, hi), mppn in ((dirs[0], (0, 90_000), 4000), (dirs[1], (60_000, n), 1500)):
        bc = pcv.Context(0, max_points_per_node=mppn)
        p = xyz[lo:hi]
        t = bc.build_octree(col(p, 0), col(p, 1), col(p, 2), rgb[lo:hi].reshape(-1).copy(), res, p.min(0), p.max(0), intensity=inten[lo:hi].copy())
        t.write_dir(d)
        t.free()
        bc.close()
    # c: the clusters, straight to disk at 2500 points per node
    bc = pcv.Context(0, max_points_per_node=2500)
    bc.build_octree_to_dir(dirs[2], col(cxyz, 0), col(cxyz, 1), col(cxyz, 2), np.asarray(crgb).reshape(-1).copy(), res, cxyz.min(0), cxyz.max(0),
                           intensity=cinten, max_points_in_core=15_000)
    bc.close()
    # bare: a part of the slab without intensities
    bc = pcv.Context(0, max_points_per_node=4000)
    p = xyz[20_000:70_000]
    t = bc.build_octree(col(p, 0), col(p, 1), col(p, 2), rgb[20_000:70_000].reshape(-1).copy(), res, p.min(0), p.max(0))
    t.write_dir(dirs[3])
    t.free()
    bc.close()
    ctx = pcv.Context(0)
    loaded = [ctx.load_dir(d) for d in dirs]
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    qfg = list(G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7())
    s = dict(pcv=pcv, ctx=ctx, dirs=dirs, loaded=loaded, dec=[_decoded(pcv, t) for t in loaded], qfg=qfg)
    yield s
    for t in loaded:
        t.free()
    ctx.close()


def _box(trees):
    return np.concatenate([np.min([t.bbox_min for t in trees], 0), np.max([t.bbox_max for t in trees], 0)])


def _px(box, levels=4):
    return float(max(box[3] - box[0], box[4] - box[1])) / (T * 2 ** levels)


def _same_tiles(tiles, want):
    assert set(tiles) == set(want), (len(tiles), len(want))
    for k in want:
        assert np.array_equal(tiles[k], want[k]), k


def _same_quadtree(info, tiles, winfo, wtiles):
    for k in ("deepest_level", "rect_min_x", "rect_min_y", "rect_edge", "num_nodes", "num_leaves"):
        assert info[k] == winfo[k], k
    _same_tiles(tiles, wtiles)


def _no_ms(info):
    return {k: v for k, v in info.items() if not k.startswith("ms_")}


def _kw(s, case):
    return dict(global_=dict(), local=dict(query_from_global=s["qfg"]), subroot=dict(query_from_global=s["qfg"], root=(1, 2)),
                transparent=dict(background=TRANSPARENT))[case]


@pytest.mark.parametrize("case", ["global_", "local", "subroot", "transparent"])
def test_equals_loaded_clouds(scene, case):
    s = scene
    kw = _kw(s, case)
    dirs, loaded = s["dirs"][:3], s["loaded"][:3]
    box = _box(loaded)
    for t in loaded:  # the united box is none of the directories' own
        assert not np.array_equal(np.concatenate([t.bbox_min, t.bbox_max]), box)
    px = _px(box)
    winfo, want = s["ctx"].xray_quadtree_clouds(loaded, T, px, **kw)
    for budget in (0, 3 << 20):
        info, tiles = s["ctx"].xray_quadtree_from_dirs(dirs, T, px, max_device_bytes=budget, **kw)
        assert info["peak_device_bytes"] <= info["max_device_bytes"]
        _same_quadtree(info, tiles, winfo, want)
        assert info["windows_loaded"] >= 1 and info["occupied_leaves"] >= info["num_leaves"] > 0
    # all four directories: the one without intensities takes part in XRay
    winfo, want = s["ctx"].xray_quadtree_clouds(s["loaded"], T, px, **kw)
    info, tiles = s["ctx"].xray_quadtree_from_dirs(s["dirs"], T, px, max_device_bytes=3 << 20, **kw)
    _same_quadtree(info, tiles, winfo, want)


def test_oracle(scene):
    s = scene
    box = _box(s["loaded"][:3])
    px = _px(box)
    kw = dict(query_from_global=s["qfg"])
    info, tiles = s["ctx"].xray_quadtree_from_dirs(s["dirs"][:3], T, px, max_device_bytes=2 << 20, **kw)
    xyz, rgb, inten = (np.concatenate([d[k] for d in s["dec"][:3]]) for k in range(3))
    winfo, want = points_quadtree(xyz, rgb, inten, box, T, px, **kw)
    assert info["deepest_level"] == winfo["deepest_level"] and (info["rect_min_x"], info["rect_min_y"], info["rect_edge"]) == winfo["rect"]
    _same_tiles(tiles, want)
    assert info["num_nodes"] == len(want)


def test_budget_scan(scene):
    """From budgets too small for one leaf's windows up to the default: every accepted run gives the loaded clouds' tiles within
    its bound; the smallest accepted ones load many windows and reuse nodes of the previous block's."""
    s = scene
    pcv = s["pcv"]
    dirs, loaded = s["dirs"][:3], s["loaded"][:3]
    kw = dict(query_from_global=s["qfg"])
    px = _px(_box(loaded), 5)
    _, want = s["ctx"].xray_quadtree_clouds(loaded, T, px, **kw)
    infos, refused = [], []
    for b in [int(v) for v in np.geomspace(64 << 10, 256 << 20, 24)] + [0]:
        try:
            info, tiles = s["ctx"].xray_quadtree_from_dirs(dirs, T, px, max_device_bytes=b, **kw)
        except pcv.PcvError as e:
            assert e.code == -6, e
            refused.append((b, str(e)))
            continue
        assert info["peak_device_bytes"] <= info["max_device_bytes"] and (b == 0 or b == info["max_device_bytes"])
        _same_tiles(tiles, want)
        infos.append(info)
    assert refused and infos and max(b for b, _ in refused) < min(i["max_device_bytes"] for i in infos)
    assert any("window of leaf" in m for _, m in refused), refused
    assert infos[0]["windows_loaded"] > 1, infos[0]
    assert any(i["nodes_reused"] > 0 for i in infos), [(i["max_device_bytes"], i["windows_loaded"], i["nodes_reused"]) for i in infos]
    assert infos[-1]["windows_loaded"] <= infos[0]["windows_loaded"]


def test_filter_intervals(scene):
    s = scene
    dirs, loaded = s["dirs"][:3], s["loaded"][:3]
    box = _box(loaded)
    px = _px(box)
    kw = dict(query_from_global=s["qfg"])
    for filters in ([(200.0, 700.0)], [(200.0, 700.0), (500.0, 900.0)], [(5000.0, 6000.0)]):
        winfo, want = s["ctx"].xray_quadtree_clouds(loaded, T, px, filter_intervals=filters, **kw)
        info, tiles = s["ctx"].xray_quadtree_from_dirs(dirs, T, px, filter_intervals=filters, max_device_bytes=2 << 20, **kw)
        assert info["peak_device_bytes"] <= info["max_device_bytes"]
        _same_quadtree(info, tiles, winfo, want)
    assert tiles == {} and info["num_nodes"] == 0


def test_permuted_order(scene):
    s = scene
    box = _box(s["loaded"])
    px = _px(box)
    kw = dict(query_from_global=s["qfg"])
    _, tiles = s["ctx"].xray_quadtree_from_dirs(s["dirs"], T, px, max_device_bytes=2 << 20, **kw)
    for order in ([3, 2, 1, 0], [1, 3, 0, 2]):
        _, other = s["ctx"].xray_quadtree_from_dirs([s["dirs"][k] for k in order], T, px, max_device_bytes=2 << 20, **kw)
        _same_tiles(other, tiles)


def test_one_directory_equals_from_dir(scene):
    """A list of one is xray_quadtree_from_dir: tiles, delivery order and every counter, at three budgets."""
    s = scene
    d = s["dirs"][1]
    px = _px(_box(s["loaded"][1:2]), 5)
    pcv = s["pcv"]
    ran = 0
    for budget in (2 << 20, 8 << 20, 256 << 20):
        for kw in (dict(query_from_global=s["qfg"]), dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0, filter_intervals=[(100.0, 900.0)])):
            runs = []
            for fn, arg in ((s["ctx"].xray_quadtree_from_dir, d), (s["ctx"].xray_quadtree_from_dirs, [d]), (s["ctx"].xray_quadtree_from_dirs, d)):
                order = []
                try:
                    info, tiles = fn(arg, T, px, max_device_bytes=budget, on_tile=lambda l, i, img: order.append((l, i)) and False, **kw)
                except pcv.PcvError as e:  # refused alike, with the same message
                    runs.append((e.code, str(e), order))
                    continue
                runs.append((_no_ms(info), tiles, order))
            (i0, t0, o0) = runs[0]
            for i1, t1, o1 in runs[1:]:
                assert i1 == i0, (budget, kw)
                assert o1 == o0
                if isinstance(t0, dict):
                    _same_tiles(t1, t0)
                else:
                    assert t1 == t0
            ran += isinstance(t0, dict)
    assert ran >= 4


def _leaf_box(info, level, index, box):
    mx, my, e = info["rect_min_x"], info["rect_min_y"], info["rect_edge"]
    for lv in range(level - 1, -1, -1):
        k = (index >> (2 * lv)) & 3
        e /= 2.0
        if k & 1:
            my += e
        if k & 2:
            mx += e
    return np.array([mx, my, box[2]]), np.array([mx + e, my + e, box[5]])


@pytest.mark.parametrize("kw", [dict(strategy=R.COLORED), dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0), dict(strategy=R.HEIGHT_STDDEV, p0=1.5, colormap=1)])
def test_attribute_strategies(scene, kw):
    s = scene
    dirs, loaded = s["dirs"][:3], s["loaded"][:3]
    box = _box(loaded)
    px = _px(box)
    info, tiles = s["ctx"].xray_quadtree_from_dirs(dirs, T, px, background=TRANSPARENT, max_device_bytes=3 << 20, **kw)
    assert info["peak_device_bytes"] <= info["max_device_bytes"]
    winfo, want = s["ctx"].xray_quadtree_clouds(loaded, T, px, background=TRANSPARENT, **kw)
    assert set(tiles) == set(want) and (info["num_nodes"], info["num_leaves"]) == (winfo["num_nodes"], winfo["num_leaves"])
    deepest = info["deepest_level"]
    xyz, rgb, inten = (np.concatenate([d[k] for d in s["dec"][:3]]) for k in range(3))
    leaves = sorted(k for k in tiles if k[0] == deepest)
    assert leaves and info["blocks_processed"] >= 2
    for level, index in leaves[:: max(1, len(leaves) // 40)]:
        tmin, tmax = _leaf_box(info, level, index, box)
        m = np.all((tmin <= xyz) & (xyz < tmax), axis=1)  # Aabb::contains (aabb.rs:46-48)
        lo, hi, cov = R.tile_ranges(xyz[m], rgb[m], inten[m], tmin, tmax, T, T, kw["strategy"], kw.get("p0", 0.0), kw.get("p1", 0.0), kw.get("colormap", 0))
        R.check_tile(tiles[(level, index)], lo, hi, cov, (kw, level, index))


def test_write_dir(scene, tmp_path):
    from PIL import Image

    from proto_meta import XrayMeta

    s = scene
    dirs, loaded = s["dirs"][:3], s["loaded"][:3]
    px = _px(_box(loaded))
    kw = dict(query_from_global=s["qfg"], filter_intervals=[(10.0, 950.0)])
    a, b = tmp_path / "from_dirs", tmp_path / "loaded"
    info = s["ctx"].xray_quadtree_from_dirs_write_dir(dirs, a, T, px, max_device_bytes=2 << 20, **kw)
    winfo = s["ctx"].xray_quadtree_clouds_write_dir(loaded, b, T, px, **kw)
    assert info["num_nodes"] == winfo["num_nodes"] > 0 and info["windows_loaded"] >= 1
    pngs = sorted(f.name for f in b.iterdir() if f.suffix == ".png")
    assert pngs == sorted(f.name for f in a.iterdir() if f.suffix == ".png") and s["pcv"].xray_node_name(0, 0) + ".png" in pngs
    for f in pngs:
        assert np.array_equal(np.asarray(Image.open(a / f).convert("RGBA")), np.asarray(Image.open(b / f).convert("RGBA"))), f
    ma, mb = (XrayMeta.FromString((p / "meta.pb").read_bytes()) for p in (a, b))
    assert (ma.version, ma.tile_size, ma.deepest_level) == (mb.version, mb.tile_size, mb.deepest_level)
    assert (ma.bounding_rect.min.x, ma.bounding_rect.min.y, ma.bounding_rect.edge_length) == (mb.bounding_rect.min.x, mb.bounding_rect.min.y,
                                                                                             mb.bounding_rect.edge_length)
    assert sorted((k.level, k.index) for k in ma.nodes) == sorted((k.level, k.index) for k in mb.nodes)


def test_cancel(scene):
    s = scene
    seen = []
    with pytest.raises(s["pcv"].PcvError) as e:
        s["ctx"].xray_quadtree_from_dirs(s["dirs"], T, _px(_box(s["loaded"])), on_tile=lambda l, i, img: seen.append((l, i)) or len(seen) >= 5)
    assert e.value.code == -5 and len(seen) == 5


def test_errors(scene, tmp_path):
    s = scene
    pcv, ctx = s["pcv"], s["ctx"]
    N = pcv._native
    px = _px(_box(s["loaded"]))
    seen = []
    on_tile = lambda l, i, img: seen.append((l, i))  # noqa: E731

    def err(dirs, **kw):
        with pytest.raises(pcv.PcvError) as e:
            ctx.xray_quadtree_from_dirs(dirs, T, px, on_tile=on_tile, **kw)
        return e.value.code, str(e.value)

    a, b, c, bare = s["dirs"]
    assert err([])[0] == -1
    assert err([a, str(tmp_path / "nowhere")])[0] == -3  # no meta.pb
    assert err([a, b], strategy=R.COLORED, bin_size=10.0)[0] == -6
    assert err(a, strategy=R.COLORED, bin_size=10.0, filter_intervals=[(0.0, 1.0)])[0] == -6
    assert err([a, bare], filter_intervals=[(0.0, 1000.0)])[0] == -1
    assert err([bare, c], strategy=R.INTENSITY, p0=0.0, p1=1000.0)[0] == -1
    assert err([a, b, c], max_device_bytes=64 << 10)[0] == -6  # below one leaf's windows (test_budget_scan names the leaf)
    assert seen == []
    # a null entry in the C list
    pr = pcv._xray_params(T, px, 0, 0.0, 0.0, 0, 0.0, None, (255, 255, 255, 255), (0, 0))
    arr = (C.c_char_p * 2)(a.encode(), None)
    info, bi, di = N.XrayQuadtreeInfo(), N.XrayBoundedInfo(), N.XrayDirInfo()
    fn = N.XRAY_TILE_FN(lambda user, level, index, rgba, t: 0)
    assert N.lib().pcv_xray_quadtree_from_dirs(ctx.h, arr, 2, C.byref(pr), None, 0, 0, fn, None, C.byref(info), C.byref(bi), C.byref(di)) == -1
    assert N.lib().pcv_xray_quadtree_from_dirs(ctx.h, arr, 0, C.byref(pr), None, 0, 0, fn, None, C.byref(info), C.byref(bi), C.byref(di)) == -1
