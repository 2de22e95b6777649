"""The X-ray attribute strategies (colour mean, intensity mean, height stddev; binned and not) against the exact per-pixel
reference of tests/xray_attr_ref.py: every byte must lie inside the reference's range, which is a single value wherever
the column sums are exact, and the covered pixels must be exactly those with at least one counted point.

Deliberate deviations, restated from the oracle: a point with a negative intensity does not count in the intensity
strategy (the reference abandons its whole batch at the first one, xray generation.rs:245-247, which makes its output
depend on batch boundaries); the binned colour strategy bins such a point like any other.  The device `logf` may differ
from glibc's by one ulp (its specified bound), which the ranges of general clouds allow; on the exact-sum cloud the bytes
must equal the glibc evaluation."""
import numpy as np
import pytest

import xray_attr_ref as R

pytestmark = pytest.mark.gpu

TRANSPARENT = (255, 255, 255, 0)
INTENSITY_PARAMS = [(0.0, 1000.0), (2.0, 3.0), (1.0, 1.5), (3.0, 60.0)]  # p1 - p0 > 1, == 1, < 1


def _points(tree, tmin, tmax, qfg=None):
    from point_cloud_viewer_b200._native import Location

    bs = tree.query_points(R.location(Location, tmin, tmax, qfg), batch_size=1 << 22)
    if not bs:
        return np.zeros((0, 3)), np.zeros((0, 3), np.uint8), np.zeros(0, np.float32)
    return np.concatenate([b["xyz"] for b in bs]), np.concatenate([b["rgb"] for b in bs]), np.concatenate([b["intensity"] for b in bs])


def _gpu_tile(tree, tmin, tmax, w, h, mode, p0, p1, cm, qfg, b):
    if b:
        return tree.xray_tile_attr_binned(tmin, tmax, w, h, mode, b, p0, p1, query_from_global=qfg)
    return tree.xray_tile_attr(tmin, tmax, w, h, mode, p0, p1, cm, query_from_global=qfg)


def _check(tree, tmin, tmax, w, h, runs, qfg=None, pts=None, strict=False):
    """Every run (mode, p0, p1, colormap, bin_size) of one tile against the reference; returns the single-valued channels.
    strict: the ranges must be single values (exact sums) computed with glibc's logf as is."""
    xyz, rgb, inten = pts if pts is not None else _points(tree, tmin, tmax, qfg)
    single = 0
    for mode, p0, p1, cm, b in runs:
        lo, hi, cov = R.tile_ranges(xyz, rgb, inten, tmin, tmax, w, h, mode, p0, p1, cm, qfg=qfg, bin_size=b, logf_ulps=0 if strict else 1)
        any_, got = _gpu_tile(tree, tmin, tmax, w, h, mode, p0, p1, cm, qfg, b)
        assert any_ == (len(xyz) > 0)
        what = (w, h, mode, p0, p1, cm, b, qfg is not None)
        if strict:
            assert np.array_equal(lo, hi), (what, "not single-valued", int((lo != hi).sum()))
        single += R.check_tile(got, lo, hi, cov, what)
    return single


def _build(pcv, ctx, x, y, z, rgb, inten, res):
    bmin = np.array([x.min(), y.min(), z.min()])
    bmax = np.array([x.max(), y.max(), z.max()])
    return ctx.build_octree(x, y, z, np.ascontiguousarray(rgb).reshape(-1), res, bmin, bmax, intensity=inten)


@pytest.fixture(scope="module")
def ctx():
    import point_cloud_viewer_b200 as pcv

    c = pcv.Context(0, max_points_per_node=1000)
    yield pcv, c
    c.close()


@pytest.fixture(scope="module", params=[0.05, 1e-6], ids=["uint", "float"])
def exact(ctx, request):
    """The exact-sum cloud, built on the GPU; the coarse resolution decodes Uint16 / Uint8 nodes, the fine one Float64 /
    Float32 nodes (and Uint8 deep under the coincident column)."""
    pcv, c = ctx
    x, y, z, rgb, inten, cols = R.exact_cloud()
    tree = _build(pcv, c, x, y, z, rgb, inten, request.param)
    encs = {m["enc"] for m in tree.nodes.values() if m["num_points"]}
    assert ({1, 2} if request.param > 1e-3 else {3, 4}) <= encs, encs
    xyz, _, it = _points(tree, (-1, -1, -1), (200, 200, 100))
    yield tree, R.exact_tiles(xyz, it, cols)
    tree.free()


EXACT_RUNS = ([(R.COLORED, 0.0, 0.0, 0, b) for b in (0.0, 1e9, 1.0)] + [(R.INTENSITY, p0, p1, 0, b) for p0, p1 in INTENSITY_PARAMS for b in (0.0, 1e9, 1.0)])
LOOSE_RUNS = ([(R.COLORED, 0.0, 0.0, 0, b) for b in (7.5, 1e-30)] + [(R.INTENSITY, 0.0, 1000.0, 0, b) for b in (7.5, 1e-30)] +
              [(R.HEIGHT_STDDEV, 0.8, 0.0, 0, 0.0), (R.HEIGHT_STDDEV, 0.05, 0.0, 1, 0.0)])


def test_exact_cloud_every_tile(exact):
    """1x1, 31x33, 96x64 (with and without a query frame) and 4096x4096 tiles; columns of 1 .. 150 000 points, edge
    intensities (-1, -0.0, NaN, +inf, 3e38 + 3e38) and points on all four faces of the 96x64 tile."""
    tree, tiles = exact
    for name, tmin, tmax, w, h, qfg in tiles:
        pts = _points(tree, tmin, tmax, qfg)
        single = _check(tree, tmin, tmax, w, h, EXACT_RUNS, qfg, pts, strict=True)
        _check(tree, tmin, tmax, w, h, LOOSE_RUNS, qfg, pts)
        assert single > 0, name


@pytest.fixture(scope="module")
def slab(ctx):
    pcv, c = ctx
    n = 200_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    inten = (np.random.default_rng(7).random(n) * 1000.0).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    tree = c.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    yield pcv, tree, np.asarray(bmin), np.asarray(bmax)
    tree.free()


GENERAL_RUNS = ([(R.COLORED, 0.0, 0.0, 0, b) for b in (0.0, 1e9, 7.5, 1.0, 1e-30)] +
                [(R.INTENSITY, p0, p1, 0, b) for p0, p1 in ((0.0, 1000.0), (100.0, 800.0), (400.0, 401.0), (0.0, 0.5)) for b in (0.0, 1e9, 7.5)] +
                [(R.HEIGHT_STDDEV, p0, 0.0, cm, 0.0) for p0 in (0.05, 0.8, 2.5) for cm in (0, 1)])


def test_general_slab_with_and_without_a_query_frame(slab):
    pcv, tree, bmin, bmax = slab
    d = bmax - bmin
    G = pcv.geometry
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    qfg = np.asarray(G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7())
    _check(tree, bmin + [0.2, 0.2, 0.0] * d, bmin + [0.7, 0.7, 1.0] * d, 96, 64, GENERAL_RUNS)
    _check(tree, np.array([-40.0, -30.0, -10.0]), np.array([24.0, 34.0, 10.0]), 128, 128, GENERAL_RUNS, qfg)


def test_general_gauss_clusters_with_coincident_blocks(ctx):
    pcv, c = ctx
    n = 1_000_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_GAUSS_CLUSTERS, 1234, 0, n)
    rng = np.random.default_rng(11)
    rgb = rng.integers(0, 256, n * 3).astype(np.uint8)
    inten = (rng.random(n) * 100.0 - 5.0).astype(np.float32)  # some negative
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_GAUSS_CLUSTERS)
    tree = c.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    try:
        bmin, bmax = np.asarray(bmin), np.asarray(bmax)
        runs = ([(R.COLORED, 0.0, 0.0, 0, b) for b in (0.0, 2.5)] + [(R.INTENSITY, 0.0, 100.0, 0, b) for b in (0.0, 2.5)] +
                [(R.HEIGHT_STDDEV, 0.5, 0.0, 0, 0.0)])
        _check(tree, bmin, bmax, 256, 192, runs)
    finally:
        tree.free()


def test_binned_distinct_bin_limit(ctx):
    """More than 2^20 distinct (pixel-independent) bins in one tile: PCV_ERR_UNSUPPORTED with the 'distinct bins' message."""
    pcv, c = ctx
    n = (1 << 20) + 4096
    k = np.arange(n)
    x, y, z = (k % 64) + 0.5, ((k // 64) % 64) + 0.5, np.zeros(n) + (k % 3)
    inten = k.astype(np.float32)
    tree = _build(pcv, c, x, y, z, np.zeros((n, 3), np.uint8), inten, 0.01)
    try:
        with pytest.raises(pcv.PcvError) as e:
            tree.xray_tile_attr_binned((0, 0, -1), (64, 64, 4), 64, 64, pcv.XRAY_INTENSITY, 1.0, 0.0, 1e7)
        assert e.value.code == -6 and "distinct bins" in str(e.value)
        # one bin fewer per pixel fits: bin size 2 halves the distinct bins
        _check(tree, (0, 0, -1), (64, 64, 4), 64, 64, [(R.INTENSITY, 0.0, 1e7, 0, 2.0)])
    finally:
        tree.free()


def test_height_stddev_far_from_mid_height(ctx):
    """Columns of 1 cm spread 1e6 m above and below the mid height of a 4e6 m tall tile."""
    pcv, c = ctx
    x, y, z, rgb, inten, (tmin, tmax, w, h) = R.far_cloud()
    tree = _build(pcv, c, x, y, z, rgb, inten, 1e-4)
    try:
        runs = [(R.HEIGHT_STDDEV, 0.05, 0.0, cm, 0.0) for cm in (0, 1)]
        assert _check(tree, tmin, tmax, w, h, runs) > 0
    finally:
        tree.free()


def _leaf_box(info, level, index, bmin, bmax):
    """quad_rect_of (quadtree lib.rs:62-101) of a leaf, over the z range of the octree's box."""
    mx, my, e = info["rect_min_x"], info["rect_min_y"], info["rect_edge"]
    for l in range(level - 1, -1, -1):
        k = (index >> (2 * l)) & 3
        half = e / 2.0
        if k & 1:
            my += half
        if k & 2:
            mx += half
        e = half
    return (mx, my, bmin[2]), (mx + e, my + e, bmax[2])


QUAD_RUNS = [dict(strategy=R.COLORED), dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0), dict(strategy=R.INTENSITY, p0=0.0, p1=1000.0, bin_size=20.0),
             dict(strategy=R.HEIGHT_STDDEV, p0=1.5, colormap=1)]


def _check_leaves(tree, info, tiles, kw, bmin, bmax):
    T = next(iter(tiles.values())).shape[0]
    leaves = [k for k in tiles if k[0] == info["deepest_level"]]
    assert leaves
    for level, index in leaves:
        tmin, tmax = _leaf_box(info, level, index, bmin, bmax)
        xyz, rgb, inten = _points(tree, tmin, tmax)
        lo, hi, cov = R.tile_ranges(xyz, rgb, inten, tmin, tmax, T, T, kw["strategy"], kw.get("p0", 0.0), kw.get("p1", 0.0), kw.get("colormap", 0),
                                    bin_size=kw.get("bin_size", 0.0))
        R.check_tile(tiles[(level, index)], lo, hi, cov, (kw, level, index))


def test_quadtree_leaves(slab, tmp_path):
    """Every leaf of Octree.xray_quadtree under a budget of several blocks, and of Context.xray_quadtree_from_dir over the
    written directory, for each attribute strategy."""
    pcv, tree, bmin, bmax = slab
    T = 16
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (32 * T) * 1.01
    d = str(tmp_path / "octree")
    tree.write_dir(d)
    ctx = tree.ctx
    for kw in QUAD_RUNS:
        # small blocks: 90 tiles' worth besides the strategy's per-leaf scratch (sums, pivots, counts; the bin table)
        budget = T * T * 4 * 90 + 600_000 + T * T * 28 + 65536 + (((8 << 20) + 8192) if kw.get("bin_size") else 0)
        info, tiles = tree.xray_quadtree(T, px, background=TRANSPARENT, max_device_bytes=budget, **kw)
        assert info["blocks_processed"] >= 2
        _check_leaves(tree, info, tiles, kw, bmin, bmax)
        dinfo, dtiles = ctx.xray_quadtree_from_dir(d, T, px, background=TRANSPARENT, max_device_bytes=budget, **kw)
        assert set(dtiles) == set(tiles)
        _check_leaves(tree, dinfo, dtiles, kw, bmin, bmax)
