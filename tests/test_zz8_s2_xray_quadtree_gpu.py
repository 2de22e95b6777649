"""X-ray quadtrees of an S2 cloud (pcv_s2_xray_quadtree, S2Cloud.xray_quadtree): the 1e6-point ECEF slab of test_zz5, split at
level 20, at pixel sizes where one cell spans many leaves.  XRay tiles equal the oracle's point-list quadtree
(orc_xray_quadtree_build_points) byte for byte - global frame, the slab's local frame as query_from_global, a sub-root, white and
transparent backgrounds, filter intervals, small budgets; attribute strategies lie in the xray_attr_ref envelope of the
brute-force point set of every leaf, and their parents are pcv_xray_build_parent of the delivered leaves."""
import numpy as np
import pytest

import xray_attr_ref as R
from test_s2_xray_oracle_points import points_quadtree

pytestmark = pytest.mark.gpu

T = 64
TRANSPARENT = (255, 255, 255, 0)


@pytest.fixture(scope="module")
def slab(ctx):
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    n = 1_000_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    inten = np.random.default_rng(3).uniform(0.0, 100.0, n).astype(np.float32)
    cloud = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=20)
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    qfg = list(G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7())  # the slab's local frame
    xyz = np.stack([x, y, z], 1)
    box = np.concatenate([cloud.bbox_min, cloud.bbox_max])
    assert np.array_equal(cloud.bbox_min, xyz.min(0)) and np.array_equal(cloud.bbox_max, xyz.max(0))
    d = cloud.bbox_max - cloud.bbox_min
    px = float(max(d[0], d[1])) / (T * 32)  # five levels: a 10 m cell spans several 64 px leaves
    yield dict(pcv=pcv, ctx=ctx, cloud=cloud, xyz=xyz, rgb=np.asarray(rgb).reshape(-1, 3), inten=inten, box=box, qfg=qfg, px=px)
    cloud.free()


def _oracle(s, **kw):
    return points_quadtree(s["xyz"], s["rgb"], s["inten"], s["box"], T, s["px"], **kw)


def _same(info, tiles, want):
    winfo, wt = want
    assert info["deepest_level"] == winfo["deepest_level"] and (info["rect_min_x"], info["rect_min_y"], info["rect_edge"]) == winfo["rect"]
    assert set(tiles) == set(wt), (len(tiles), len(wt))
    for k in wt:
        assert np.array_equal(tiles[k], wt[k]), k
    assert info["num_nodes"] == len(wt)


@pytest.mark.parametrize("case", ["global", "local", "subroot", "transparent"])
def test_xray_equals_oracle(slab, case):
    s = slab
    kw = dict(global_=dict(), local=dict(query_from_global=s["qfg"]), subroot=dict(query_from_global=s["qfg"], root=(2, 6)),
              transparent=dict(query_from_global=s["qfg"], background=TRANSPARENT))["global_" if case == "global" else case]
    info, tiles = s["cloud"].xray_quadtree(T, s["px"], **kw)
    _same(info, tiles, _oracle(s, **kw))
    assert info["deepest_level"] >= 5 and info["peak_device_bytes"] <= info["max_device_bytes"]
    assert info["leaf_points"] >= (s["cloud"].num_points if case != "subroot" else 1) and info["key_batches"] >= 1


def test_filter_intervals(slab):
    s = slab
    base, base_tiles = s["cloud"].xray_quadtree(T, s["px"], query_from_global=s["qfg"])
    for filters in ([(20.0, 60.0)], [(20.0, 60.0), (50.0, 90.0)]):
        info, tiles = s["cloud"].xray_quadtree(T, s["px"], query_from_global=s["qfg"], filter_intervals=filters)
        _same(info, tiles, _oracle(s, query_from_global=s["qfg"], filters=filters))
    # the points of one corner of the slab only: the other leaves and their empty ancestors are absent
    xq = R.transformed(s["xyz"], s["qfg"])
    inten = np.where(xq[:, 0] < np.median(xq[:, 0]), 200.0, s["inten"]).astype(np.float32)
    cloud2 = s["ctx"].build_s2_cloud(s["xyz"][:, 0].copy(), s["xyz"][:, 1].copy(), s["xyz"][:, 2].copy(), s["rgb"].reshape(-1).copy(), inten, split_level=20)
    try:
        info, tiles = cloud2.xray_quadtree(T, s["px"], query_from_global=s["qfg"], filter_intervals=[(150.0, 250.0)])
        want = points_quadtree(s["xyz"], s["rgb"], inten, s["box"], T, s["px"], query_from_global=s["qfg"], filters=[(150.0, 250.0)])
        _same(info, tiles, want)
        assert 0 < info["num_leaves"] < base["num_leaves"] and len(tiles) < len(base_tiles)
    finally:
        cloud2.free()
    info, tiles = s["cloud"].xray_quadtree(T, s["px"], query_from_global=s["qfg"], filter_intervals=[(500.0, 600.0)])
    assert tiles == {} and info["num_nodes"] == 0


def test_budgets(slab):
    s = slab
    pcv = s["pcv"]
    info0, tiles0 = s["cloud"].xray_quadtree(T, s["px"], query_from_global=s["qfg"])
    assert info0["peak_device_bytes"] <= info0["max_device_bytes"]
    with pytest.raises(pcv.PcvError) as e:
        s["cloud"].xray_quadtree(T, s["px"], query_from_global=s["qfg"], max_device_bytes=64 << 10)
    assert e.value.code == -6
    # 16 px leaves of eight times the pixel size hold several thousand points each: near the smallest budgets that work, a
    # block of four leaves needs several key batches
    t, px = 16, s["px"] * 8
    info1, tiles1 = s["cloud"].xray_quadtree(t, px, query_from_global=s["qfg"])
    _same(info1, tiles1, points_quadtree(s["xyz"], s["rgb"], s["inten"], s["box"], t, px, query_from_global=s["qfg"]))
    found = False
    for budget in [int(v) for v in np.geomspace(16 << 10, 4 << 20, 80)]:
        try:
            info, tiles = s["cloud"].xray_quadtree(t, px, query_from_global=s["qfg"], max_device_bytes=budget)
        except pcv.PcvError as err:
            assert err.code == -6, err
            continue
        assert info["peak_device_bytes"] <= budget == info["max_device_bytes"]
        assert set(tiles) == set(tiles1) and all(np.array_equal(tiles[k], tiles1[k]) for k in tiles1)
        if info["blocks_processed"] >= 8 and info["key_batches"] >= 2 * info["blocks_processed"]:
            found = True
            break
    assert found


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


@pytest.mark.parametrize("kw", [dict(strategy=R.COLORED), dict(strategy=R.INTENSITY, p0=0.0, p1=100.0), dict(strategy=R.HEIGHT_STDDEV, p0=0.5, colormap=0),
                                dict(strategy=R.HEIGHT_STDDEV, p0=0.5, colormap=1)])
def test_attribute_strategies(slab, kw):
    s = slab
    pcv = s["pcv"]
    info, tiles = s["cloud"].xray_quadtree(T, s["px"], background=TRANSPARENT, max_device_bytes=3 << 20, **kw)
    deepest = info["deepest_level"]
    leaves = sorted(k for k in tiles if k[0] == deepest)
    assert leaves and info["blocks_processed"] >= 2
    xyz = s["xyz"]
    bmin, bmax = s["cloud"].bbox_min, s["cloud"].bbox_max
    for level, index in leaves[:: max(1, len(leaves) // 60)]:
        tmin, tmax = _leaf_box(info, level, index, bmin, bmax)
        m = np.all((tmin <= xyz) & (xyz < tmax), axis=1)  # Aabb::contains (aabb.rs:46-48)
        lo, hi, cov = R.tile_ranges(xyz[m], s["rgb"][m], s["inten"][m], tmin, tmax, T, T, kw["strategy"], kw.get("p0", 0.0), kw.get("p1", 0.0),
                                    kw.get("colormap", 0))
        R.check_tile(tiles[(level, index)], lo, hi, cov, (kw, level, index))
    # every parent is build_parent of the delivered children
    for (level, index), img in tiles.items():
        if level == deepest:
            continue
        ch = [tiles.get((level + 1, 4 * index + k)) for k in range(4)]
        assert any(c is not None for c in ch)
        want = pcv.xray_build_parent(s["ctx"], ch, TRANSPARENT, T)
        assert np.array_equal(img, want), (level, index)


def test_errors_cancel_and_no_colour(slab):
    s = slab
    pcv, ctx = s["pcv"], s["ctx"]
    cloud = s["cloud"]
    with pytest.raises(pcv.PcvError) as e:
        cloud.xray_quadtree(T, s["px"], strategy=R.COLORED, bin_size=10.0)
    assert e.value.code == -6
    with pytest.raises(pcv.PcvError) as e:
        cloud.xray_quadtree(0, s["px"])
    assert e.value.code == -1
    seen = []
    with pytest.raises(pcv.PcvError) as e:
        cloud.xray_quadtree(T, s["px"], on_tile=lambda l, i, img: seen.append((l, i)) or len(seen) >= 5)
    assert e.value.code == -5 and len(seen) == 5
    x, y, z = (np.ascontiguousarray(s["xyz"][:200_000, k]) for k in range(3))
    bare = ctx.build_s2_cloud(x, y, z, None, None, split_level=20)
    try:
        with pytest.raises(pcv.PcvError) as e:
            bare.xray_quadtree(T, s["px"], strategy=R.COLORED)
        assert e.value.code == -1
        with pytest.raises(pcv.PcvError) as e:
            bare.xray_quadtree(T, s["px"], filter_intervals=[(0.0, 1.0)])
        assert e.value.code == -1
        info, tiles = bare.xray_quadtree(T, s["px"], query_from_global=s["qfg"])
        box = np.concatenate([bare.bbox_min, bare.bbox_max])
        _same(info, tiles, points_quadtree(s["xyz"][:200_000], None, None, box, T, s["px"], query_from_global=s["qfg"]))
    finally:
        bare.free()


def test_reloaded_and_write_dir(slab, tmp_path):
    from PIL import Image

    from proto_meta import XrayMeta

    s = slab
    pcv, ctx = s["pcv"], s["ctx"]
    info, tiles = s["cloud"].xray_quadtree(T, s["px"], query_from_global=s["qfg"], filter_intervals=[(10.0, 95.0)])
    d = tmp_path / "s2"
    s["cloud"].write_dir(d)
    loaded = ctx.load_s2_dir(d)
    try:
        info2, tiles2 = loaded.xray_quadtree(T, s["px"], query_from_global=s["qfg"], filter_intervals=[(10.0, 95.0)])
        assert set(tiles2) == set(tiles) and all(np.array_equal(tiles2[k], tiles[k]) for k in tiles)
    finally:
        loaded.free()
    out = tmp_path / "xray"
    winfo = s["cloud"].xray_quadtree_write_dir(out, T, s["px"], query_from_global=s["qfg"], filter_intervals=[(10.0, 95.0)])
    assert winfo["num_nodes"] == len(tiles)
    for (lv, i), img in tiles.items():
        got = np.asarray(Image.open(out / (pcv.xray_node_name(lv, i) + ".png")).convert("RGBA"))
        assert np.array_equal(got, img), (lv, i)
    m = XrayMeta.FromString((out / "meta.pb").read_bytes())
    assert m.deepest_level == info["deepest_level"] and m.tile_size == T and len(m.nodes) == len(tiles)
