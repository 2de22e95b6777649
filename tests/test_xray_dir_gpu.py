"""X-ray quadtrees straight from an octree directory (pcv_xray_quadtree_from_dir): every tile, the node set, the rect, the levels
and the delivery order against pcv_xray_quadtree_bounded over pcv_octree_load_dir of the same directory, under budgets from
one window per leaf up to one window for everything; the attribute strategies, an out-of-core-built directory, the write
variant, cancellation, the errors, and one case against the oracle's build_xray_quadtree."""
import os
import shutil

import numpy as np
import pytest

import oracle_api as O

pytestmark = pytest.mark.gpu

WHITE = (255, 255, 255, 255)
TRANSPARENT = (255, 255, 255, 0)


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    n = 150_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    inten = ((np.arange(n) * 7919) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    c = pcv.Context(0, max_points_per_node=4000)
    d = tmp_path_factory.mktemp("octree")
    tree = c.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    tree.write_dir(str(d))
    tree.free()
    loaded = c.load_dir(str(d))
    _, npts, xyz_bytes, _, _, _, _ = _octree_info(pcv, loaded)
    yield dict(pcv=pcv, ctx=c, dir=str(d), loaded=loaded, bmin=np.asarray(bmin), bmax=np.asarray(bmax), x=x, y=y, z=z, rgb=rgb, inten=inten, res=res,
               octree_bytes=xyz_bytes + 3 * npts)
    loaded.free()
    c.close()


def _octree_info(pcv, tree):
    import ctypes as C

    nn, npts, xb, r = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_double()
    mn, mx, hi = (C.c_double * 3)(), (C.c_double * 3)(), C.c_int()
    pcv._native.check(pcv._native.lib().pcv_octree_info(tree.h, C.byref(nn), C.byref(npts), C.byref(xb), C.byref(r), mn, mx, C.byref(hi)))
    return nn.value, npts.value, xb.value, r.value, mn, mx, hi.value


def _ordered(fn, *a, **kw):
    order = []
    info, tiles = fn(*a, on_tile=lambda l, i, img: order.append((l, i)) and False, **kw)
    assert set(order) == set(tiles)
    return info, tiles, order


def _post_order(leaves, depth):
    exist = [set() for _ in range(depth + 1)]
    for l in leaves:
        for up in range(depth + 1):
            exist[up].add(l >> (2 * up))
    out = []

    def walk(up, idx):
        if up > 0:
            for k in range(4):
                if (idx << 2) + k in exist[up - 1]:
                    walk(up - 1, (idx << 2) + k)
        out.append((up, idx))

    for r in sorted(exist[depth]):
        walk(depth, r)
    return out


def _delivery_order(tiles, deepest, block_level):
    """The bounded driver's delivery order for these tiles at this block level: each block's subtree in post-order; the
    ancestors above the block level when the walk moves on to the next block that has tiles, the rest at the end."""
    root_level = min(l for l, _ in tiles)
    g, above = deepest - block_level, block_level - root_level
    leaves = sorted(i for l, i in tiles if l == deepest)
    out, prev = [], None
    for lo in range(len(leaves)):
        b = leaves[lo] >> (2 * g)
        if lo and leaves[lo - 1] >> (2 * g) == b:
            continue
        ls = [v for v in leaves if v >> (2 * g) == b]
        out += [(deepest - up, (b << (2 * (g - up))) + i) for up, i in _post_order([v - (b << (2 * g)) for v in ls], g)]
        if prev is not None:
            k = 0
            while k + 1 < above and prev >> (2 * (k + 1)) != b >> (2 * (k + 1)):
                k += 1
            out += [(block_level - up, prev >> (2 * up)) for up in range(1, k + 1)]
        prev = b
    if prev is not None:
        out += [(block_level - up, prev >> (2 * up)) for up in range(1, above + 1)]
    return out


def _same(a, b, exact=True):
    (ia, ta, oa), (ib, tb, ob) = a, b
    assert set(ta) == set(tb)
    if ia["block_level"] == ib["block_level"]:
        assert oa == ob, "delivery order"
    elif ta:
        assert oa == _delivery_order(ta, ia["deepest_level"], ia["block_level"]), "delivery order"
        assert ob == _delivery_order(tb, ib["deepest_level"], ib["block_level"]), "delivery order"
    for k in ("rect_min_x", "rect_min_y", "rect_edge", "deepest_level", "tile_size_px", "num_nodes", "num_leaves"):
        assert ia[k] == ib[k], k
    assert ia["leaf_points"] <= ib["leaf_points"]  # points decoded: the occupancy pass prunes at the leaf level
    if exact:
        for k in ta:
            assert np.array_equal(ta[k], tb[k]), k
    else:
        for k in ta:
            assert np.array_equal(ta[k][..., 3], tb[k][..., 3]), k
            assert np.abs(ta[k].astype(np.int16) - tb[k].astype(np.int16)).max() <= 1, k


def _smallest_budget(scene, T, px, lo, **kw):
    """The smallest budget of a geometric scan upwards from `lo` that the directory driver accepts."""
    ctx = scene["ctx"]
    b = lo
    while True:
        try:
            return b, _ordered(ctx.xray_quadtree_from_dir, scene["dir"], T, px, max_device_bytes=b, **kw)
        except scene["pcv"]._native.PcvError as e:
            assert e.code == -6, e
            b = int(b * 1.2)
            assert b < 64 << 20


@pytest.mark.parametrize("T,depth", [(32, 4), (16, 5)])
def test_xray_strategy_byte_identical(scene, T, depth):
    ctx, loaded = scene["ctx"], scene["loaded"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (2 ** depth * T) * 1.01
    ob = scene["octree_bytes"]
    for bg in (WHITE, TRANSPARENT):
        want = _ordered(loaded.xray_quadtree, T, px, background=bg)
        assert want[0]["deepest_level"] == depth
        small, got = _smallest_budget(scene, T, px, ob // 8, background=bg)
        info = got[0]
        assert info["peak_device_bytes"] <= small < ob
        assert info["peak_device_bytes"] < ob and info["windows_loaded"] > 1
        assert info["largest_window_bytes"] < ob
        _same(got, want)
        levels = {info["block_level"]}
        for budget in (2 * small, 4 * small, 0):
            got = _ordered(ctx.xray_quadtree_from_dir, scene["dir"], T, px, background=bg, max_device_bytes=budget)
            _same(got, want)
            if budget:
                assert got[0]["peak_device_bytes"] <= budget
            levels.add(got[0]["block_level"])
        assert got[0]["windows_loaded"] == 1 and got[0]["block_level"] == 0  # the default budget: everything in one window
        assert len(levels) >= 2


def test_query_frame_and_sub_root(scene):
    pcv, ctx, loaded = scene["pcv"], scene["ctx"], scene["loaded"]
    G = pcv.geometry
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    qfg = G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7()
    T = 32
    want = _ordered(loaded.xray_quadtree, T, 0.5, query_from_global=qfg)
    small, got = _smallest_budget(scene, T, 0.5, scene["octree_bytes"] // 8, query_from_global=qfg)
    assert got[0]["windows_loaded"] > 1
    _same(got, want)
    _same(_ordered(ctx.xray_quadtree_from_dir, scene["dir"], T, 0.5, query_from_global=qfg), want)
    sub = sorted(k for k in want[1] if k[0] == 2)[0]
    want2 = _ordered(loaded.xray_quadtree, T, 0.5, query_from_global=qfg, root=sub)
    for budget in (small, 0):
        _same(_ordered(ctx.xray_quadtree_from_dir, scene["dir"], T, 0.5, query_from_global=qfg, root=sub, max_device_bytes=budget), want2)


def test_attribute_strategies(scene):
    pcv, ctx, loaded = scene["pcv"], scene["ctx"], scene["loaded"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    T = 32
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (4 * T) * 1.01
    for kw in (dict(strategy=pcv.XRAY_COLORED), dict(strategy=pcv.XRAY_INTENSITY, p0=0.0, p1=1000.0), dict(strategy=pcv.XRAY_COLORED, bin_size=20.0),
               dict(strategy=pcv.XRAY_INTENSITY, p0=0.0, p1=1000.0, bin_size=20.0), dict(strategy=pcv.XRAY_HEIGHT_STDDEV, p0=1.5, colormap=1)):
        want = _ordered(loaded.xray_quadtree, T, px, background=TRANSPARENT, **kw)
        for budget in (0, 24 << 20):
            got = _ordered(ctx.xray_quadtree_from_dir, scene["dir"], T, px, background=TRANSPARENT, max_device_bytes=budget, **kw)
            _same(got, want, exact=False)
            if budget:
                assert got[0]["peak_device_bytes"] <= budget


def test_out_of_core_built_directory(scene, tmp_path):
    pcv, ctx = scene["pcv"], scene["ctx"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    info = ctx.build_octree_to_dir(str(tmp_path), scene["x"], scene["y"], scene["z"], scene["rgb"], scene["res"], bmin, bmax, max_points_in_core=40_000)
    assert info["groups"] > 1
    loaded = ctx.load_dir(str(tmp_path))
    try:
        T = 16
        px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (2 ** 5 * T) * 1.01
        want = _ordered(loaded.xray_quadtree, T, px)
        _, npts, xb, *_ = _octree_info(pcv, loaded)
        small, got = _smallest_budget(dict(scene, dir=str(tmp_path)), T, px, (xb + 3 * npts) // 8)
        assert got[0]["peak_device_bytes"] <= small < xb + 3 * npts and got[0]["windows_loaded"] > 1
        _same(got, want)
        _same(_ordered(ctx.xray_quadtree_from_dir, str(tmp_path), T, px), want)
    finally:
        loaded.free()


def test_write_variant(scene, tmp_path):
    from PIL import Image

    ctx, loaded = scene["ctx"], scene["loaded"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    T = 16
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (8 * T) * 1.01
    from proto_meta import XrayMeta

    a, b, c = tmp_path / "in_core", tmp_path / "from_dir", tmp_path / "from_dir_small"
    loaded.xray_quadtree_write_dir(a, T, px)
    ctx.xray_quadtree_from_dir_write_dir(scene["dir"], b, T, px)  # both in one block: the same delivery order
    assert (a / "meta.pb").read_bytes() == (b / "meta.pb").read_bytes()
    budget = _smallest_budget(scene, T, px, scene["octree_bytes"] // 8)[0]
    info = ctx.xray_quadtree_from_dir_write_dir(scene["dir"], c, T, px, max_device_bytes=budget)
    assert info["peak_device_bytes"] <= budget < scene["octree_bytes"] and info["windows_loaded"] > 1
    # several blocks: the meta file lists the nodes in the order of delivery, which depends on the block level
    ma, mc = XrayMeta(), XrayMeta()
    ma.ParseFromString((a / "meta.pb").read_bytes())
    mc.ParseFromString((c / "meta.pb").read_bytes())
    key = lambda m: sorted((n.level, n.index) for n in m.nodes)  # noqa: E731
    assert key(ma) == key(mc) and len(ma.nodes) == len(mc.nodes)
    for f in ("version", "bounding_rect", "deepest_level", "tile_size"):
        assert getattr(ma, f) == getattr(mc, f), f
    for d in (b, c):
        assert sorted(os.listdir(a)) == sorted(os.listdir(d))
        for name in os.listdir(a):
            if name.endswith(".png"):
                assert np.array_equal(np.asarray(Image.open(a / name).convert("RGBA")), np.asarray(Image.open(d / name).convert("RGBA"))), name


def test_cancellation(scene):
    pcv, ctx = scene["pcv"], scene["ctx"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    T = 16
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (16 * T) * 1.01
    budget = _smallest_budget(scene, T, px, scene["octree_bytes"] // 8)[0]
    full, _ = ctx.xray_quadtree_from_dir(scene["dir"], T, px, max_device_bytes=budget)
    for k in (1, 5, full["num_nodes"] - 1):
        seen = []
        with pytest.raises(pcv._native.PcvError) as e:
            ctx.xray_quadtree_from_dir(scene["dir"], T, px, on_tile=lambda l, i, img: seen.append((l, i)) or len(seen) >= k, max_device_bytes=budget)
        assert e.value.code == -5 and len(seen) == k
    again, _ = ctx.xray_quadtree_from_dir(scene["dir"], T, px, max_device_bytes=budget)
    assert again["num_nodes"] == full["num_nodes"]


def test_errors(scene, tmp_path):
    pcv, ctx = scene["pcv"], scene["ctx"]
    E = pcv._native.PcvError
    T, px = 16, 100.0

    def copy(name):
        d = tmp_path / name
        shutil.copytree(scene["dir"], d)
        return d

    d = copy("missing")
    victim = sorted(f for f in os.listdir(d) if f.endswith(".rgb"))[3]
    os.remove(d / victim)
    with pytest.raises(E) as e:
        ctx.xray_quadtree_from_dir(d, T, px)
    assert e.value.code == -4 and victim in str(e.value)
    d = copy("truncated")
    victim = sorted(f for f in os.listdir(d) if f.endswith(".xyz"))[5]
    data = (d / victim).read_bytes()
    (d / victim).write_bytes(data[:-1])
    with pytest.raises(E) as e:
        ctx.xray_quadtree_from_dir(d, T, px)
    assert e.value.code == -4 and victim in str(e.value)
    d = copy("version")
    meta = bytearray((d / "meta.pb").read_bytes())
    assert meta[:2] == b"\x08\x0d"
    meta[1] = 12
    (d / "meta.pb").write_bytes(bytes(meta))
    with pytest.raises(E) as e:
        ctx.xray_quadtree_from_dir(d, T, px)
    assert e.value.code == -1
    # a budget that holds the tiles and the occupancy pass but not one leaf's window
    with pytest.raises(E) as e:
        ctx.xray_quadtree_from_dir(scene["dir"], T, px, max_device_bytes=700_000)
    assert e.value.code == -6 and "window of leaf r" in str(e.value) and "700000" in str(e.value)
    with pytest.raises(E) as e:  # no octree at all
        ctx.xray_quadtree_from_dir(tmp_path / "nothing", T, px)
    assert e.value.code == -3
    with pytest.raises(E) as e:  # no intensities in the directory
        d = copy("no_intensity")
        for f in os.listdir(d):
            if f.endswith(".intensity"):
                os.remove(d / f)
        ctx.xray_quadtree_from_dir(d, T, px, strategy=pcv.XRAY_INTENSITY, p0=0.0, p1=1.0)
    assert e.value.code == -1 and "without intensity" in str(e.value)
    ctx.xray_quadtree_from_dir(scene["dir"], T, px)  # the context still works


def test_empty_octree(scene, tmp_path):
    """A directory whose octree holds no point: no tile, as the in-core driver over load_dir."""
    pcv, ctx = scene["pcv"], scene["ctx"]
    e = np.zeros(0)
    ctx.build_octree_to_dir(str(tmp_path), e, e, e, np.zeros(0, np.uint8), 0.01, (0.0, 0.0, 0.0), (8.0, 8.0, 8.0))
    loaded = ctx.load_dir(str(tmp_path))
    try:
        want, wt = loaded.xray_quadtree(8, 0.25)
        info, tiles = ctx.xray_quadtree_from_dir(str(tmp_path), 8, 0.25)
        assert tiles == wt == {} and info["num_nodes"] == want["num_nodes"] == 0 and info["windows_loaded"] == 0
    finally:
        loaded.free()


def test_against_the_oracle(tmp_path):
    """A small cloud X-rayed from disk equals the oracle's build_xray_quadtree directly, under a budget of several windows."""
    import point_cloud_viewer_b200 as pcv

    rng = np.random.default_rng(5)
    n = 20_000
    x, y, z = rng.uniform(0.0, 64.0, n), rng.uniform(0.0, 64.0, n), rng.uniform(0.0, 8.0, n)
    keep = ~((x > 40) & (y > 40))
    x, y, z = x[keep], y[keep], z[keep]
    rgb = rng.integers(0, 256, (len(x), 3), dtype=np.uint8)
    bmin, bmax, res = (0.0, 0.0, 0.0), (64.0, 64.0, 8.0), 1.0 / 256
    c = pcv.Context(0, max_points_per_node=500)
    tree = c.build_octree(x, y, z, rgb.reshape(-1), res, bmin, bmax)
    tree.write_dir(str(tmp_path))
    tree.free()
    ref = O.build(x, y, z, rgb, res, bmin, bmax, max_points_per_node=500)
    try:
        for bg in (WHITE, TRANSPARENT):
            oinfo, otiles = ref.xray_quadtree(8, 1.0, background=bg)
            for budget in (600_000, 0):
                info, tiles = c.xray_quadtree_from_dir(str(tmp_path), 8, 1.0, background=bg, max_device_bytes=budget)
                assert set(tiles) == set(otiles) and all(np.array_equal(tiles[k], otiles[k]) for k in otiles)
                assert info["deepest_level"] == oinfo["deepest_level"]
    finally:
        c.close()
