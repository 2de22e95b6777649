"""X-ray quadtrees over several clouds at once (Context.xray_quadtree_clouds: pcv_xray_quadtree_clouds,
pcv_s2_xray_quadtree_clouds) and filter intervals on every octree source.  Three resident octrees with different boxes - two
overlapping parts of the config-1 ECEF slab and config-2 clusters moved next to it - give XRay tiles byte-identical to the
point-list oracle over their concatenated decoded points, in any order; two S2 clouds of the halves of one slab equal the
S2 cloud of all of it; filtered octree and directory quadtrees equal the filtered oracle; one cloud through the new entry equals
the existing entry in every tile and counter."""
import numpy as np
import pytest

import xray_attr_ref as R
from test_s2_xray_oracle_points import points_quadtree

pytestmark = pytest.mark.gpu

T = 32
TRANSPARENT = (255, 255, 255, 0)
ALL = (-1e30, 1e30)


def _decoded(pcv, tree):
    """Every point of the octree as AllPoints streams it: decoded f64 positions, colours, intensities."""
    bs = tree.query_points(pcv.geometry.all_points(), batch_size=1 << 20)
    return (np.concatenate([b["xyz"] for b in bs]), np.concatenate([b["rgb"] for b in bs]),
            np.concatenate([b["intensity"] for b in bs]).astype(np.float32))


@pytest.fixture(scope="module")
def scene():
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    ctx = pcv.Context(0, max_points_per_node=4000)
    n = 150_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    xyz = np.stack([x, y, z], 1)
    rgb = np.asarray(rgb).reshape(-1, 3)
    inten = ((np.arange(n) * 7919) % 1000).astype(np.float32)
    _, _, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    # config 2's clusters, scaled into a box beside the slab's (disjoint from it)
    m = 40_000
    cx, cy, cz, crgb = pcv.synth_points_host(pcv.SYNTH_GAUSS_CLUSTERS, 7, 0, m)
    c = np.stack([cx, cy, cz], 1)
    c = (c - c.min(0)) / np.ptp(c, 0).max()
    ext = xyz.max(0) - xyz.min(0)
    cxyz = xyz.max(0) + np.array([0.05, -0.3, -0.5]) * ext + c * 0.4 * ext
    parts = [(xyz[:90_000], rgb[:90_000], inten[:90_000]), (xyz[60_000:], rgb[60_000:], inten[60_000:]),
             (cxyz, np.asarray(crgb).reshape(-1, 3), ((np.arange(m) * 31) % 1000).astype(np.float32))]
    trees = []
    for p, r, i in parts:
        trees.append(ctx.build_octree(*(np.ascontiguousarray(p[:, k]) for k in range(3)), np.ascontiguousarray(r).reshape(-1), res, p.min(0), p.max(0),
                                      intensity=np.ascontiguousarray(i)))
    full = ctx.build_octree(x, y, z, rgb.reshape(-1), res, xyz.min(0), xyz.max(0), intensity=inten)
    dec = [_decoded(pcv, t) for t in trees]
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    qfg = list(G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7())
    yield dict(pcv=pcv, ctx=ctx, trees=trees, full=full, dec=dec, full_dec=_decoded(pcv, full), qfg=qfg, xyz=xyz, rgb=rgb, inten=inten, res=res)
    for t in trees + [full]:
        t.free()
    ctx.close()


def _box(trees):
    return np.concatenate([np.min([t.bbox_min for t in trees], 0), np.max([t.bbox_max for t in trees], 0)])


def _px(box, levels=4):
    return float(max(box[3] - box[0], box[4] - box[1])) / (T * 2 ** levels)


def _oracle(dec, box, px, **kw):
    xyz, rgb, inten = (np.concatenate([d[k] for d in dec]) for k in range(3))
    return points_quadtree(xyz, rgb, inten, box, T, px, **kw)


def _same(info, tiles, want):
    winfo, wt = want
    assert info["deepest_level"] == winfo["deepest_level"] and (info["rect_min_x"], info["rect_min_y"], info["rect_edge"]) == winfo["rect"]
    assert set(tiles) == set(wt), (len(tiles), len(wt))
    for k in wt:
        assert np.array_equal(tiles[k], wt[k]), k
    assert info["num_nodes"] == len(wt)


def _no_ms(info):
    return {k: v for k, v in info.items() if not k.startswith("ms_")}


@pytest.mark.parametrize("case", ["global", "local", "subroot", "transparent", "small"])
def test_three_octrees_equal_oracle(scene, case):
    s = scene
    trees = s["trees"]
    box = _box(trees)
    for t in trees:  # the united box is none of the clouds' own
        assert not np.array_equal(np.concatenate([t.bbox_min, t.bbox_max]), box)
    px = _px(box)
    kw = dict(global_=dict(), local=dict(query_from_global=s["qfg"]), subroot=dict(query_from_global=s["qfg"], root=(1, 2)),
              transparent=dict(background=TRANSPARENT), small=dict(query_from_global=s["qfg"]))["global_" if case == "global" else case]
    budget = 2 << 20 if case == "small" else 0
    info, tiles = s["ctx"].xray_quadtree_clouds(trees, T, px, max_device_bytes=budget, **kw)
    _same(info, tiles, _oracle(s["dec"], box, px, **kw))
    if case == "small":
        assert info["blocks_processed"] >= 2 and info["key_batches"] > info["blocks_processed"]
        assert info["peak_device_bytes"] <= info["max_device_bytes"]
    rinfo, rtiles = s["ctx"].xray_quadtree_clouds(trees[::-1], T, px, max_device_bytes=budget, **kw)
    assert set(rtiles) == set(tiles) and all(np.array_equal(rtiles[k], tiles[k]) for k in tiles)
    assert rinfo["leaf_points"] == info["leaf_points"] and rinfo["num_nodes"] == info["num_nodes"]


def test_two_overlapping_octrees(scene):
    s = scene
    trees = s["trees"][:2]
    box = _box(trees)
    px = _px(box, 5)
    info, tiles = s["ctx"].xray_quadtree_clouds(trees, T, px, query_from_global=s["qfg"], max_device_bytes=3 << 20)
    _same(info, tiles, _oracle(s["dec"][:2], box, px, query_from_global=s["qfg"]))


def test_one_cloud_equals_existing_entry(scene):
    """The three ways to X-ray one octree (pcv_xray_quadtree_bounded, a list of one, Octree.xray_quadtree) agree in every tile
    and counter.  They share the driver; that the driver's one-cloud case is the parent commit's is what
    scripts/xray_driver_ab.py checks against a build of the parent."""
    s = scene
    pcv = s["pcv"]
    N = pcv._native
    t = s["full"]
    px = _px(_box([t]))
    # explicit budgets: the default one is read from the free device memory of the moment
    for kw in (dict(), dict(query_from_global=s["qfg"], max_device_bytes=2 << 20), dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0),
               dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0, bin_size=50.0), dict(strategy=R.HEIGHT_STDDEV, p0=1.5, colormap=1)):
        budget = kw.pop("max_device_bytes", 256 << 20)
        pr = pcv._xray_params(T, px, kw.get("strategy", 0), kw.get("p0", 0.0), kw.get("p1", 0.0), kw.get("colormap", 0), kw.get("bin_size", 0.0),
                              kw.get("query_from_global"), (255, 255, 255, 255), (0, 0))
        old, old_tiles = pcv._xray_call(N.lib().pcv_xray_quadtree_bounded, (t.h, pcv.C.byref(pr), budget), False, True)
        new, new_tiles = s["ctx"].xray_quadtree_clouds([t], T, px, max_device_bytes=budget, **kw)
        one, one_tiles = t.xray_quadtree(T, px, max_device_bytes=budget, **kw)
        assert _no_ms(new) == _no_ms(old) == _no_ms(one), kw
        assert set(new_tiles) == set(old_tiles) == set(one_tiles)
        if kw.get("strategy", 0) in (0, R.INTENSITY):  # integer intensities: exact f32 sums in any order (the other strategies' float atomics are not)
            assert all(np.array_equal(new_tiles[k], old_tiles[k]) and np.array_equal(one_tiles[k], old_tiles[k]) for k in old_tiles), kw


@pytest.mark.parametrize("kw", [dict(strategy=R.COLORED), dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0), dict(strategy=R.HEIGHT_STDDEV, p0=1.5, colormap=1)])
def test_attribute_strategies_over_octrees(scene, kw):
    s = scene
    trees = s["trees"]
    box = _box(trees)
    px = _px(box)
    info, tiles = s["ctx"].xray_quadtree_clouds(trees, T, px, background=TRANSPARENT, max_device_bytes=3 << 20, **kw)
    xinfo, xtiles = s["ctx"].xray_quadtree_clouds(trees, T, px, background=TRANSPARENT, max_device_bytes=3 << 20)
    deepest = info["deepest_level"]
    assert set(tiles) == set(xtiles)  # the same leaves exist whatever the strategy
    xyz, rgb, inten = (np.concatenate([d[k] for d in s["dec"]]) for k in range(3))
    leaves = sorted(k for k in tiles if k[0] == deepest)
    for level, index in leaves[:: max(1, len(leaves) // 40)]:
        tmin, tmax = _leaf_box(info, level, index, box)
        m = np.all((tmin <= xyz) & (xyz < tmax), axis=1)  # Aabb::contains (aabb.rs:46-48)
        lo, hi, cov = R.tile_ranges(xyz[m], rgb[m], inten[m], tmin, tmax, T, T, kw["strategy"], kw.get("p0", 0.0), kw.get("p1", 0.0), kw.get("colormap", 0))
        R.check_tile(tiles[(level, index)], lo, hi, cov, (kw, level, index))
        assert np.array_equal(tiles[(level, index)][..., 3] != 0, xtiles[(level, index)][..., 3] != 0)  # identical coverage


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


def test_filters_on_one_octree(scene, tmp_path):
    s = scene
    pcv, ctx, t = s["pcv"], s["ctx"], s["full"]
    box = _box([t])
    px = _px(box)
    base, base_tiles = t.xray_quadtree(T, px, query_from_global=s["qfg"])
    for filters in ([(200.0, 700.0)], [(200.0, 700.0), (500.0, 900.0)]):
        info, tiles = t.xray_quadtree(T, px, query_from_global=s["qfg"], filter_intervals=filters, max_device_bytes=2 << 20)
        _same(info, tiles, _oracle([s["full_dec"]], box, px, query_from_global=s["qfg"], filters=filters))
    info, tiles = t.xray_quadtree(T, px, query_from_global=s["qfg"], filter_intervals=[ALL])
    assert set(tiles) == set(base_tiles) and all(np.array_equal(tiles[k], base_tiles[k]) for k in tiles)
    assert 0 <= info.pop("peak_device_bytes") - base["peak_device_bytes"] <= 16  # the interval's own 16 bytes
    assert _no_ms(info) == {k: v for k, v in _no_ms(base).items() if k != "peak_device_bytes"}
    info, tiles = t.xray_quadtree(T, px, query_from_global=s["qfg"], filter_intervals=[(2000.0, 3000.0)])
    assert tiles == {} and info["num_nodes"] == 0
    # half of the slab only passes: the leaves of the other half and their empty ancestors disappear
    xq = R.transformed(s["xyz"], s["qfg"])
    inten = np.where(xq[:, 0] < np.median(xq[:, 0]), 5000.0, s["inten"]).astype(np.float32)
    half = ctx.build_octree(*(np.ascontiguousarray(s["xyz"][:, k]) for k in range(3)), s["rgb"].reshape(-1).copy(), s["res"], s["xyz"].min(0), s["xyz"].max(0),
                            intensity=inten)
    try:
        info, tiles = half.xray_quadtree(T, px, query_from_global=s["qfg"], filter_intervals=[(0.0, 1500.0)])
        _same(info, tiles, _oracle([_decoded(pcv, half)], box, px, query_from_global=s["qfg"], filters=[(0.0, 1500.0)]))
        assert 0 < info["num_leaves"] < base["num_leaves"]
    finally:
        half.free()
    # the directory streams the same filtered leaves
    d = tmp_path / "octree"
    t.write_dir(d)
    for filters in ([(200.0, 700.0)], [(2000.0, 3000.0)]):
        info, tiles = t.xray_quadtree(T, px, query_from_global=s["qfg"], filter_intervals=filters, max_device_bytes=8 << 20)
        dinfo, dtiles = ctx.xray_quadtree_from_dir(d, T, px, query_from_global=s["qfg"], filter_intervals=filters, max_device_bytes=8 << 20)
        assert set(dtiles) == set(tiles) and all(np.array_equal(dtiles[k], tiles[k]) for k in tiles)
        assert dinfo["num_nodes"] == info["num_nodes"] and dinfo["num_leaves"] == info["num_leaves"]
    for filters in ([(200.0, 700.0)], [(0.0, 1000.0), (100.0, 900.0)]):
        for strategy in (R.INTENSITY, R.HEIGHT_STDDEV):
            info, tiles = t.xray_quadtree(T, px, strategy=strategy, p0=1.0, p1=1000.0, filter_intervals=filters)
            dinfo, dtiles = ctx.xray_quadtree_from_dir(d, T, px, strategy=strategy, p0=1.0, p1=1000.0, filter_intervals=filters)
            assert set(dtiles) == set(tiles)


def test_two_s2_halves_equal_the_whole(scene):
    s = scene
    ctx = s["ctx"]
    n = len(s["xyz"])
    cols = [np.ascontiguousarray(s["xyz"][:, k]) for k in range(3)]
    whole = ctx.build_s2_cloud(*cols, s["rgb"].reshape(-1).copy(), s["inten"], split_level=20)
    halves = [ctx.build_s2_cloud(*(c[a:b].copy() for c in cols), s["rgb"][a:b].reshape(-1).copy(), s["inten"][a:b].copy(), split_level=20)
              for a, b in ((0, n // 2), (n // 2, n))]
    try:
        assert np.array_equal(np.min([h.bbox_min for h in halves], 0), whole.bbox_min)
        assert np.array_equal(np.max([h.bbox_max for h in halves], 0), whole.bbox_max)
        px = _px(np.concatenate([whole.bbox_min, whole.bbox_max]), 5)
        for kw in (dict(), dict(query_from_global=s["qfg"], max_device_bytes=2 << 20), dict(filter_intervals=[(100.0, 800.0)], background=TRANSPARENT)):
            info, tiles = ctx.xray_quadtree_clouds(halves, T, px, **kw)
            winfo, wtiles = whole.xray_quadtree(T, px, **kw)
            assert set(tiles) == set(wtiles) and all(np.array_equal(tiles[k], wtiles[k]) for k in tiles), kw
            assert info["num_nodes"] == winfo["num_nodes"]
        for kw in (dict(strategy=R.COLORED), dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0), dict(strategy=R.HEIGHT_STDDEV, p0=1.5)):
            info, tiles = ctx.xray_quadtree_clouds(halves, T, px, background=TRANSPARENT, **kw)
            box = np.concatenate([whole.bbox_min, whole.bbox_max])
            leaves = sorted(k for k in tiles if k[0] == info["deepest_level"])
            for level, index in leaves[:: max(1, len(leaves) // 30)]:
                tmin, tmax = _leaf_box(info, level, index, box)
                m = np.all((tmin <= s["xyz"]) & (s["xyz"] < tmax), axis=1)
                lo, hi, cov = R.tile_ranges(s["xyz"][m], s["rgb"][m], s["inten"][m], tmin, tmax, T, T, kw["strategy"], kw.get("p0", 0.0), kw.get("p1", 0.0))
                R.check_tile(tiles[(level, index)], lo, hi, cov, (kw, level, index))
            winfo, wtiles = whole.xray_quadtree(T, px, background=TRANSPARENT, **kw)
            assert set(tiles) == set(wtiles)
    finally:
        for c in halves + [whole]:
            c.free()


def test_errors_cancel_and_write_dir(scene, tmp_path):
    from PIL import Image

    from proto_meta import XrayMeta

    s = scene
    pcv, ctx, trees = s["pcv"], s["ctx"], s["trees"]
    N = pcv._native
    px = _px(_box(trees))

    def code(f):
        with pytest.raises(pcv.PcvError) as e:
            f()
        return e.value.code

    pr = pcv._xray_params(T, px, 0, 0.0, 0.0, 0, 0.0, None, (255, 255, 255, 255), (0, 0))
    for fn in (N.lib().pcv_xray_quadtree_clouds, N.lib().pcv_s2_xray_quadtree_clouds):
        assert code(lambda: pcv._xray_call(fn, ((pcv.C.c_void_p * 1)(trees[0].h), 0, pcv.C.byref(pr), None, 0, 0), False, True)) == -1  # n = 0
        assert code(lambda: pcv._xray_call(fn, ((pcv.C.c_void_p * 2)(trees[0].h, None), 2, pcv.C.byref(pr), None, 0, 0), False, True)) == -1  # null
    with pytest.raises(TypeError):
        ctx.xray_quadtree_clouds([trees[0], object()], T, px)
    other = pcv.Context(0)
    x, y, z = (np.ascontiguousarray(s["xyz"][:20_000, k]) for k in range(3))
    bare = ctx.build_octree(x, y, z, s["rgb"][:20_000].reshape(-1).copy(), s["res"], s["xyz"][:20_000].min(0), s["xyz"][:20_000].max(0))
    elsewhere = other.build_octree(x, y, z, s["rgb"][:20_000].reshape(-1).copy(), s["res"], s["xyz"][:20_000].min(0), s["xyz"][:20_000].max(0))
    s2_bare = ctx.build_s2_cloud(x, y, z, None, s["inten"][:20_000].copy(), split_level=20)
    s2_full = ctx.build_s2_cloud(x, y, z, s["rgb"][:20_000].reshape(-1).copy(), s["inten"][:20_000].copy(), split_level=20)
    try:
        assert code(lambda: ctx.xray_quadtree_clouds([trees[0], elsewhere], T, px)) == -1
        assert code(lambda: ctx.xray_quadtree_clouds([trees[0], bare], T, px, filter_intervals=[(0.0, 1.0)])) == -1
        assert code(lambda: ctx.xray_quadtree_clouds([trees[0], bare], T, px, strategy=R.INTENSITY)) == -1
        assert code(lambda: ctx.xray_quadtree_clouds([s2_full, s2_bare], T, px, strategy=R.COLORED)) == -1
        assert code(lambda: ctx.xray_quadtree_clouds(trees[:2], T, px, strategy=R.INTENSITY, bin_size=10.0)) == -6
        assert code(lambda: trees[0].xray_quadtree(T, px, strategy=R.INTENSITY, bin_size=10.0, filter_intervals=[(0.0, 500.0)])) == -6
        info, _ = trees[0].xray_quadtree(T, px, strategy=R.INTENSITY, p1=1000.0, bin_size=10.0)  # binned over one octree still runs
        assert info["num_leaves"] > 0
        ctx.xray_quadtree_clouds([trees[0], bare], T, px)  # XRay needs no intensity
    finally:
        for c in (bare, s2_bare, s2_full):
            c.free()
        elsewhere.free()
        other.close()
    seen = []
    assert code(lambda: ctx.xray_quadtree_clouds(trees, T, px, on_tile=lambda l, i, img: seen.append((l, i)) or len(seen) >= 5)) == -5
    assert len(seen) == 5
    info, tiles = ctx.xray_quadtree_clouds(trees, T, px, filter_intervals=[(100.0, 900.0)])
    out = tmp_path / "xray"
    winfo = ctx.xray_quadtree_clouds_write_dir(trees, out, T, px, filter_intervals=[(100.0, 900.0)], max_device_bytes=3 << 20)
    assert winfo["num_nodes"] == len(tiles)
    for (lv, i), img in tiles.items():
        got = np.asarray(Image.open(out / (pcv.xray_node_name(lv, i) + ".png")).convert("RGBA"))
        assert np.array_equal(got, img), (lv, i)
    m = XrayMeta.FromString((out / "meta.pb").read_bytes())
    assert m.deepest_level == info["deepest_level"] and m.tile_size == T and len(m.nodes) == len(tiles)


def test_filters_over_several_octrees(scene):
    """Filters over three octrees: XRay tiles equal the filtered point-list oracle over the concatenated points, and a filtered
    attribute strategy lies in the envelope of the points that pass."""
    s = scene
    trees = s["trees"]
    box = _box(trees)
    px = _px(box)
    for filters in ([(150.0, 650.0)], [(100.0, 900.0), (400.0, 1000.0)]):
        info, tiles = s["ctx"].xray_quadtree_clouds(trees, T, px, query_from_global=s["qfg"], filter_intervals=filters, max_device_bytes=2 << 20)
        _same(info, tiles, _oracle(s["dec"], box, px, query_from_global=s["qfg"], filters=filters))
        assert info["blocks_processed"] >= 2
    filters = [(150.0, 650.0)]
    xyz, rgb, inten = (np.concatenate([d[k] for d in s["dec"]]) for k in range(3))
    keep = (150.0 <= inten.astype(np.float64)) & (inten.astype(np.float64) <= 650.0)
    _, xtiles = s["ctx"].xray_quadtree_clouds(trees, T, px, background=TRANSPARENT, filter_intervals=filters)
    for kw in (dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0), dict(strategy=R.HEIGHT_STDDEV, p0=1.5, colormap=1)):
        info, tiles = s["ctx"].xray_quadtree_clouds(trees, T, px, background=TRANSPARENT, filter_intervals=filters, max_device_bytes=3 << 20, **kw)
        assert set(tiles) == set(xtiles)
        leaves = sorted(k for k in tiles if k[0] == info["deepest_level"])
        for level, index in leaves[:: max(1, len(leaves) // 30)]:
            tmin, tmax = _leaf_box(info, level, index, box)
            m = keep & np.all((tmin <= xyz) & (xyz < tmax), axis=1)  # Aabb::contains (aabb.rs:46-48)
            lo, hi, cov = R.tile_ranges(xyz[m], rgb[m], inten[m], tmin, tmax, T, T, kw["strategy"], kw.get("p0", 0.0), kw.get("p1", 0.0), kw.get("colormap", 0))
            R.check_tile(tiles[(level, index)], lo, hi, cov, (kw, level, index))


def test_empty_clouds_in_the_list(scene):
    """An empty octree whose box lies inside the others' changes no tile; an empty S2 cloud (whose box is the origin, as
    pcv_s2_info reports it) widens the united box like any other member, and the tiles equal the oracle's over that box."""
    s = scene
    pcv, ctx, trees = s["pcv"], s["ctx"], s["trees"]
    box = _box(trees)
    px = _px(box)
    inner_min, inner_max = box[:3] + 0.25 * (box[3:] - box[:3]), box[:3] + 0.5 * (box[3:] - box[:3])
    e = ctx.build_octree(np.zeros(0), np.zeros(0), np.zeros(0), np.zeros(0, np.uint8), s["res"], inner_min, inner_max, n=0)
    try:
        assert len(e.nodes) == 0 and not e.has_intensity
        want_info, want = ctx.xray_quadtree_clouds(trees, T, px, query_from_global=s["qfg"])
        for order in ([e] + trees, trees[:1] + [e] + trees[1:]):
            for kw in (dict(), dict(max_device_bytes=2 << 20), dict(filter_intervals=[(0.0, 1000.0)])):
                if "filter_intervals" in kw:  # filters need every cloud's intensities
                    with pytest.raises(pcv.PcvError) as err:
                        ctx.xray_quadtree_clouds(order, T, px, query_from_global=s["qfg"], **kw)
                    assert err.value.code == -1
                    continue
                info, tiles = ctx.xray_quadtree_clouds(order, T, px, query_from_global=s["qfg"], **kw)
                assert set(tiles) == set(want) and all(np.array_equal(tiles[k], want[k]) for k in want), kw
            info, tiles = ctx.xray_quadtree_clouds(order, T, px, query_from_global=s["qfg"], strategy=R.HEIGHT_STDDEV, p0=1.5)
            assert info["num_leaves"] == want_info["num_leaves"]
        info, tiles = ctx.xray_quadtree_clouds([e], T, px)  # only empty clouds: no tile
        assert tiles == {} and info["num_nodes"] == 0
    finally:
        e.free()
    n = 40_000
    cols = [np.ascontiguousarray(s["xyz"][:n, k]) for k in range(3)]
    cloud = ctx.build_s2_cloud(*cols, s["rgb"][:n].reshape(-1).copy(), s["inten"][:n].copy(), split_level=20)
    empty = ctx.build_s2_cloud(np.zeros(0), np.zeros(0), np.zeros(0), np.zeros((0, 3), np.uint8), np.zeros(0, np.float32))
    try:
        ubox = np.concatenate([np.minimum(cloud.bbox_min, empty.bbox_min), np.maximum(cloud.bbox_max, empty.bbox_max)])
        upx = _px(ubox, 8)
        for order in ([cloud, empty], [empty, cloud]):
            info, tiles = ctx.xray_quadtree_clouds(order, T, upx)
            _same(info, tiles, points_quadtree(s["xyz"][:n], s["rgb"][:n], s["inten"][:n], ubox, T, upx))
            assert info["num_leaves"] > 0
        info, tiles = ctx.xray_quadtree_clouds([empty, cloud], T, upx, strategy=R.HEIGHT_STDDEV, p0=1.5)
        assert info["num_leaves"] > 0
        with pytest.raises(pcv.PcvError) as err:  # built from an empty colour array: the empty cloud has no colours
            ctx.xray_quadtree_clouds([empty, cloud], T, upx, strategy=R.COLORED)
        assert err.value.code == -1
    finally:
        empty.free()
        cloud.free()
