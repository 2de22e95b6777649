"""X-ray quadtrees straight from S2 directories (pcv_s2_xray_quadtree_from_dirs, Context.xray_quadtree_from_s2_dirs): the 1e6-point
ECEF slab of test_zz8, written with build_s2_dir.  XRay tiles equal load_s2_dir(d).xray_quadtree and the oracle's point-list
quadtree byte for byte - global frame, the slab's local frame, a sub-root, a transparent background - at budgets that force
several windows, at a coarse split level whose cells span several blocks and exceed the scan chunk, with filter intervals, and
over three overlapping directories in either order; attribute strategies make the resident path's leaves, lie in the
xray_attr_ref envelope and have build_parent parents; write_dir, cancellation, the I/O counters and every error of the contract.
Tiles are compared as sets: the order in which finished ancestors are delivered between blocks follows the block level, which
the budget and the windows decide."""
import os
import shutil

import numpy as np
import pytest

import xray_attr_ref as R
from test_s2_xray_oracle_points import points_quadtree

pytestmark = pytest.mark.gpu

T = 64
TRANSPARENT = (255, 255, 255, 0)


@pytest.fixture(scope="module")
def slab(ctx, tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    n = 1_000_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    inten = np.random.default_rng(3).uniform(0.0, 100.0, n).astype(np.float32)
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    qfg = list(G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7())  # the slab's local frame
    base = tmp_path_factory.mktemp("s2dirs")
    d = base / "l20"
    ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=20)
    loaded = ctx.load_s2_dir(d)
    xyz = np.stack([x, y, z], 1)
    box = np.concatenate([loaded.bbox_min, loaded.bbox_max])
    ext = loaded.bbox_max - loaded.bbox_min
    px = float(max(ext[0], ext[1])) / (T * 32)
    s = dict(pcv=pcv, ctx=ctx, d=d, base=base, loaded=loaded, xyz=xyz, x=x, y=y, z=z, rgb=np.asarray(rgb).reshape(-1, 3), rgb_flat=rgb, inten=inten,
             box=box, qfg=qfg, px=px, n=n)
    yield s
    loaded.free()


def _kw(s, case):
    return dict(global_=dict(), local=dict(query_from_global=s["qfg"]), subroot=dict(query_from_global=s["qfg"], root=(2, 6)),
                transparent=dict(query_from_global=s["qfg"], background=TRANSPARENT))[case]


def _same_tiles(tiles, want):
    assert set(tiles) == set(want), (len(tiles), len(want))
    for k in want:
        assert np.array_equal(tiles[k], want[k]), k


def _same(info, tiles, want):
    winfo, wt = want
    assert info["deepest_level"] == winfo["deepest_level"] and (info["rect_min_x"], info["rect_min_y"], info["rect_edge"]) == winfo["rect"]
    _same_tiles(tiles, wt)
    assert info["num_nodes"] == len(wt)


def _bounded(info):
    assert info["peak_device_bytes"] <= info["max_device_bytes"], info


@pytest.mark.parametrize("case", ["global_", "local", "subroot", "transparent"])
def test_xray_equals_loaded_and_oracle(slab, case):
    s = slab
    kw = _kw(s, case)
    info, tiles = s["ctx"].xray_quadtree_from_s2_dirs(s["d"], T, s["px"], **kw)
    _bounded(info)
    _, want = s["loaded"].xray_quadtree(T, s["px"], **kw)
    _same_tiles(tiles, want)
    _same(info, tiles, points_quadtree(s["xyz"], s["rgb"], s["inten"], s["box"], T, s["px"], **kw))
    assert info["windows_loaded"] >= 1 and info["occupied_leaves"] >= info["num_leaves"] > 0


def _budget_scan(s, d, want, kw, budgets, t=T, px=None):
    """Runs at every budget; returns the infos of the runs that fit, each checked for equal tiles and its bound."""
    pcv = s["pcv"]
    out = []
    for b in budgets:
        try:
            info, tiles = s["ctx"].xray_quadtree_from_s2_dirs(d, t, px or s["px"], max_device_bytes=b, **kw)
        except pcv.PcvError as e:
            assert e.code == -6, e
            continue
        assert info["peak_device_bytes"] <= info["max_device_bytes"] and (b == 0 or b == info["max_device_bytes"])
        _same_tiles(tiles, want)
        out.append(info)
    return out


def test_budgets_force_windows(slab):
    s = slab
    kw = dict(query_from_global=s["qfg"])
    _, want = s["loaded"].xray_quadtree(T, s["px"], **kw)
    infos = _budget_scan(s, s["d"], want, kw, [int(v) for v in np.geomspace(1 << 20, 48 << 20, 10)])
    many = [i for i in infos if i["windows_loaded"] >= 4]
    assert many, [(i["max_device_bytes"], i["windows_loaded"]) for i in infos]
    assert any(i["nodes_reused"] > 0 for i in many) and all(i["windows_loaded"] > 1 for i in many)


def test_coarse_cells(slab):
    """Split level 14: single cells span several blocks and exceed the scan chunk."""
    s = slab
    pcv = s["pcv"]
    d = s["base"] / "l14"
    if not d.exists():
        s["ctx"].build_s2_dir(d, s["x"], s["y"], s["z"], s["rgb_flat"], s["inten"], split_level=14)
    coarse = s["ctx"].load_s2_dir(d)
    try:
        kw = dict(query_from_global=s["qfg"])
        info0, want = coarse.xray_quadtree(T, s["px"], **kw)
        _same_tiles(want, s["loaded"].xray_quadtree(T, s["px"], **kw)[1])  # the same points: the same tiles
        infos = _budget_scan(s, d, want, kw, [0] + [int(v) for v in np.geomspace(2 << 20, 64 << 20, 8)])
        assert any(i["windows_loaded"] > 1 for i in infos)
        # the scan chunk holds min(64 MiB, budget / 8) of 24 B positions: some run cut the largest cell across chunks
        assert any(int(coarse.cell_counts.max()) > min(64 << 20, i["max_device_bytes"] // 8) // 24 for i in infos)
        # a budget that holds the scan pass but not one leaf's window
        with pytest.raises(pcv.PcvError) as e:
            s["ctx"].xray_quadtree_from_s2_dirs(d, T, s["px"], max_device_bytes=1 << 20, **kw)
        assert e.value.code == -6 and "window of leaf" in str(e.value), e.value
    finally:
        coarse.free()


def test_filter_intervals(slab, tmp_path):
    s = slab
    kw = dict(query_from_global=s["qfg"])
    for filters in ([(20.0, 60.0)], [(20.0, 60.0), (50.0, 90.0)]):
        info, tiles = s["ctx"].xray_quadtree_from_s2_dirs(s["d"], T, s["px"], filter_intervals=filters, max_device_bytes=48 << 20, **kw)
        _bounded(info)
        _same(info, tiles, points_quadtree(s["xyz"], s["rgb"], s["inten"], s["box"], T, s["px"], filters=filters, **kw))
    # the points of one corner of the slab only: the other leaves and their empty ancestors are absent
    xq = R.transformed(s["xyz"], s["qfg"])
    inten = np.where(xq[:, 0] < np.median(xq[:, 0]), 200.0, s["inten"]).astype(np.float32)
    d = tmp_path / "corner"
    s["ctx"].build_s2_dir(d, s["x"], s["y"], s["z"], s["rgb_flat"], inten, split_level=20)
    base, _ = s["ctx"].xray_quadtree_from_s2_dirs(d, T, s["px"], **kw)
    info, tiles = s["ctx"].xray_quadtree_from_s2_dirs(d, T, s["px"], filter_intervals=[(150.0, 250.0)], **kw)
    _same(info, tiles, points_quadtree(s["xyz"], s["rgb"], inten, s["box"], T, s["px"], filters=[(150.0, 250.0)], **kw))
    assert 0 < info["num_leaves"] < base["num_leaves"]
    info, tiles = s["ctx"].xray_quadtree_from_s2_dirs(d, T, s["px"], filter_intervals=[(500.0, 600.0)], **kw)
    assert tiles == {} and info["num_nodes"] == 0


def test_several_directories(slab, tmp_path):
    s = slab
    n = s["n"]
    parts = [(0, int(0.45 * n)), (int(0.3 * n), int(0.75 * n)), (int(0.6 * n), n)]  # overlapping: shared points count twice
    dirs, clouds = [], []
    for k, (a, b) in enumerate(parts):
        d = tmp_path / ("part%d" % k)
        s["ctx"].build_s2_dir(d, s["x"][a:b].copy(), s["y"][a:b].copy(), s["z"][a:b].copy(), s["rgb"][a:b].reshape(-1).copy(), s["inten"][a:b].copy(),
                              split_level=20)
        dirs.append(d)
        clouds.append(s["ctx"].load_s2_dir(d))
    try:
        kw = dict(query_from_global=s["qfg"])
        _, want = s["ctx"].xray_quadtree_clouds(clouds, T, s["px"], **kw)
        info, tiles = s["ctx"].xray_quadtree_from_s2_dirs(dirs, T, s["px"], max_device_bytes=48 << 20, **kw)
        _bounded(info)
        _same_tiles(tiles, want)
        idx = np.concatenate([np.arange(a, b) for a, b in parts])
        _same(info, tiles, points_quadtree(s["xyz"][idx], s["rgb"][idx], s["inten"][idx], s["box"], T, s["px"], **kw))
        _, rev = s["ctx"].xray_quadtree_from_s2_dirs(dirs[::-1], T, s["px"], **kw)
        _same_tiles(rev, tiles)
    finally:
        for c in clouds:
            c.free()


def _leaf_box(info, level, index, bmin, bmax):
    mx, my, e = info["rect_min_x"], info["rect_min_y"], info["rect_edge"]
    for lv in range(level - 1, -1, -1):
        k = (index >> (2 * lv)) & 3
        half = e / 2.0
        if k & 1:
            my += half
        if k & 2:
            mx += half
        e = half
    return np.array([mx, my, bmin[2]]), np.array([mx + e, my + e, bmax[2]])


@pytest.mark.parametrize("kw", [dict(strategy=R.COLORED), dict(strategy=R.INTENSITY, p0=0.0, p1=100.0), dict(strategy=R.HEIGHT_STDDEV, p0=0.5, colormap=1)])
def test_attribute_strategies(slab, kw):
    s = slab
    pcv = s["pcv"]
    info, tiles = s["ctx"].xray_quadtree_from_s2_dirs(s["d"], T, s["px"], background=TRANSPARENT, max_device_bytes=48 << 20, **kw)
    _bounded(info)
    _, res = s["loaded"].xray_quadtree(T, s["px"], background=TRANSPARENT, **kw)
    assert set(tiles) == set(res)
    deepest = info["deepest_level"]
    leaves = sorted(k for k in tiles if k[0] == deepest)
    assert leaves and info["blocks_processed"] >= 2
    xyz = s["xyz"]
    bmin, bmax = s["loaded"].bbox_min, s["loaded"].bbox_max
    for level, index in leaves[:: max(1, len(leaves) // 40)]:
        tmin, tmax = _leaf_box(info, level, index, bmin, bmax)
        m = np.all((tmin <= xyz) & (xyz < tmax), axis=1)  # Aabb::contains (aabb.rs:46-48)
        lo, hi, cov = R.tile_ranges(xyz[m], s["rgb"][m], s["inten"][m], tmin, tmax, T, T, kw["strategy"], kw.get("p0", 0.0), kw.get("p1", 0.0),
                                    kw.get("colormap", 0))
        R.check_tile(tiles[(level, index)], lo, hi, cov, (kw, level, index))
    for (level, index), img in tiles.items():
        if level == deepest:
            continue
        ch = [tiles.get((level + 1, 4 * index + k)) for k in range(4)]
        assert any(c is not None for c in ch)
        assert np.array_equal(img, pcv.xray_build_parent(s["ctx"], ch, TRANSPARENT, T)), (level, index)


def test_io_counters(slab):
    s = slab
    n = s["n"]
    info, _ = s["ctx"].xray_quadtree_from_s2_dirs(s["d"], T, s["px"], query_from_global=s["qfg"], max_device_bytes=48 << 20)
    # XRay without filters reads .xyz only: the scan 24 B per point, then every point again in some window
    assert info["bytes_read"] % 24 == 0 and info["bytes_read"] >= 2 * 24 * n
    assert info["bytes_read"] == info["bytes_uploaded"]
    assert info["windows_loaded"] >= 1 and info["largest_window_points"] > 0 and info["ms_occupancy"] > 0
    cells = len([f for f in os.listdir(s["d"]) if f.endswith(".xyz")])
    assert info["node_files_read"] >= 2 * cells
    # with filters the windows read intensities too
    info2, _ = s["ctx"].xray_quadtree_from_s2_dirs(s["d"], T, s["px"], query_from_global=s["qfg"], max_device_bytes=48 << 20, filter_intervals=[(0.0, 100.0)])
    assert (info2["bytes_read"] - 24 * n) % 28 == 0 and info2["bytes_read"] > info["bytes_read"]


def test_write_dir(slab, tmp_path):
    from PIL import Image

    s = slab
    pcv = s["pcv"]
    kw = dict(query_from_global=s["qfg"], filter_intervals=[(10.0, 95.0)])
    a, b = tmp_path / "from_dirs", tmp_path / "loaded"
    info = s["ctx"].xray_quadtree_from_s2_dirs_write_dir([s["d"]], a, T, s["px"], max_device_bytes=48 << 20, **kw)
    winfo = s["ctx"].xray_quadtree_clouds_write_dir([s["loaded"]], b, T, s["px"], **kw)
    assert info["num_nodes"] == winfo["num_nodes"] > 0 and info["windows_loaded"] >= 1
    pngs = sorted(f for f in os.listdir(b) if f.endswith(".png"))
    assert pngs == sorted(f for f in os.listdir(a) if f.endswith(".png"))
    for f in pngs:
        assert np.array_equal(np.asarray(Image.open(a / f).convert("RGBA")), np.asarray(Image.open(b / f).convert("RGBA"))), f
    # the meta lists the nodes in delivery order, which follows the block level each budget allows: equal as a set, and byte
    # for byte when both runs used the same block level
    from proto_meta import XrayMeta

    ma, mb = (XrayMeta.FromString((p / "meta.pb").read_bytes()) for p in (a, b))
    assert (ma.version, ma.tile_size, ma.deepest_level) == (mb.version, mb.tile_size, mb.deepest_level)
    assert (ma.bounding_rect.min.x, ma.bounding_rect.min.y, ma.bounding_rect.edge_length) == (mb.bounding_rect.min.x, mb.bounding_rect.min.y,
                                                                                             mb.bounding_rect.edge_length)
    assert sorted((k.level, k.index) for k in ma.nodes) == sorted((k.level, k.index) for k in mb.nodes)
    if info["block_level"] == winfo["block_level"]:
        assert (a / "meta.pb").read_bytes() == (b / "meta.pb").read_bytes()
    same = s["ctx"].xray_quadtree_from_s2_dirs_write_dir([s["d"]], tmp_path / "default", T, s["px"], **kw)
    if same["block_level"] == winfo["block_level"]:
        assert (tmp_path / "default" / "meta.pb").read_bytes() == (b / "meta.pb").read_bytes()
    assert pcv.xray_node_name(0, 0) + ".png" in pngs


def test_cancel(slab):
    s = slab
    seen = []
    with pytest.raises(s["pcv"].PcvError) as e:
        s["ctx"].xray_quadtree_from_s2_dirs(s["d"], T, s["px"], on_tile=lambda l, i, img: seen.append((l, i)) or len(seen) >= 5)
    assert e.value.code == -5 and len(seen) == 5


def test_errors(slab, tmp_path):
    s = slab
    pcv, ctx = s["pcv"], s["ctx"]
    seen = []
    on_tile = lambda l, i, img: seen.append((l, i))  # noqa: E731

    def code(dirs, **kw):
        with pytest.raises(pcv.PcvError) as e:
            ctx.xray_quadtree_from_s2_dirs(dirs, T, s["px"], on_tile=on_tile, **kw)
        return e.value.code

    assert code([]) == -1
    assert code(tmp_path / "nowhere") == -3
    bad = tmp_path / "bad"
    bad.mkdir()
    (bad / "meta.pb").write_bytes(b"\x3a\x32\x01")
    assert code(bad) == -1
    # missing or short cell files fail before any tile, in any of several directories
    cells = sorted(f[:-4] for f in os.listdir(s["d"]) if f.endswith(".xyz"))
    for k, (ext, how) in enumerate([(".xyz", "rm"), (".xyz", "short"), (".rgb", "short"), (".intensity", "rm")]):
        d = tmp_path / ("broken%d" % k)
        shutil.copytree(s["d"], d)
        f = d / (cells[len(cells) // 2] + ext)
        if how == "rm":
            f.unlink()
        else:
            f.write_bytes(f.read_bytes()[:-1])
        assert code([s["d"], d]) == -4, (ext, how)
        assert seen == []
    assert code(s["d"], strategy=R.COLORED, bin_size=10.0) == -6
    bare = tmp_path / "bare"
    ctx.build_s2_dir(bare, s["x"][:200_000].copy(), s["y"][:200_000].copy(), s["z"][:200_000].copy(), None, None, split_level=20)
    assert code(bare, filter_intervals=[(0.0, 1.0)]) == -1
    assert code([s["d"], bare], strategy=R.COLORED) == -1
    assert code(s["d"], max_device_bytes=64 << 10) == -6  # not even the scan pass
    assert seen == []
    # the bare directory on its own: the oracle's tiles without colour or intensity
    info, tiles = ctx.xray_quadtree_from_s2_dirs(bare, T, s["px"], query_from_global=s["qfg"])
    xyz = s["xyz"][:200_000]
    box = np.concatenate([xyz.min(0), xyz.max(0)])
    _same(info, tiles, points_quadtree(xyz, None, None, box, T, s["px"], query_from_global=s["qfg"]))
