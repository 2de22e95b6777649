"""PointLocation::WebMercatorRect on the GPU, for the resident octree, the octree directory and the S2-cell cloud, against the
oracle (oracle/oracle_web_mercator.hpp, liboracle_wm.so: see test_web_mercator.py):
- node lists (pcv_nodes_in_location, resident and directory) and S2 cell lists equal the oracle's exactly, for rects at zoom
  17/19/21/23 over the 1e6-point slab of test_zz5, thin strips at zoom 19 and 20 with more axes than a location record holds, a
  wrapped rect at zoom 0, a rect at the map's top edge over points beyond 85.05 degrees that clamp, and a rect at the antimeridian;
- streamed and batched points of all three sources, with and without filter intervals, equal the oracle's outside the band of
  2^-40 (normalised) around the rect's edges; the band count is printed and stays below 10 per rect;
- points 1e-10 (normalised) on either side of each edge come out exactly as the oracle says; a wrapped rect holds no point;
- a batch mixing rects, frusta and OBBs gives every location the counts of its single-location call;
- check_web_mercator_rect_query_equality (point_cloud_test/tests/main.rs) with the rules of test_zz5 / test_zz7;
- invalid rects: ValueError from geometry.web_mercator_rect, PCV_ERR_INVALID from every source for hand-filled ones."""
import ctypes as C
import math

import numpy as np
import pytest

import oracle_api as O
import test_web_mercator as W

pytestmark = pytest.mark.gpu

SEED, N, LEVEL = 80293751232, 1_000_000, 20
DELTA = 2.0 ** -40
FILTERS = [(100.0, 700.0)]


def _cat(batches):
    if not batches:
        return dict(xyz=np.zeros((0, 3)), rgb=np.zeros((0, 3), np.uint8), src=np.zeros(0, np.uint64))
    return {k: np.concatenate([b[k] for b in batches]) for k in ("xyz", "rgb", "src")}


def _nw_se(loc):
    return np.array([loc.aabb_min[0], loc.aabb_min[1], loc.aabb_max[0], loc.aabb_max[1]])


def _oracle_nodes(ref, loc):
    L = W.oracle()
    cap = ref.num_nodes + 1
    out = np.zeros(2 * cap, np.uint64)
    n = L.orc_wm_nodes(C.c_void_p(ref.h), W._p(_nw_se(loc)), W._p(out), cap)
    return [O.id_str(int(out[2 * i]), int(out[2 * i + 1])) for i in range(n)]


def _oracle_query(ref, loc, filters=()):
    L = W.oracle()
    f = np.ascontiguousarray(np.asarray(filters, np.float64).reshape(-1))
    fp = W._p(f) if len(f) else None
    n = L.orc_wm_query(C.c_void_p(ref.h), W._p(_nw_se(loc)), fp, len(f) // 2, None, None, 0)
    xyz, src = np.zeros((n, 3)), np.zeros(n, np.uint64)
    L.orc_wm_query(C.c_void_p(ref.h), W._p(_nw_se(loc)), fp, len(f) // 2, W._p(xyz), W._p(src), n)
    return dict(xyz=xyz, src=src)


class Cloud:
    """One point set as a resident octree (loaded from its directory, so src is the slot), the same directory opened for
    streaming, the oracle's load of it, and an S2 cloud of the input points."""

    def __init__(self, pcv, ctx, d, x, y, z, rgb, inten, bmin, bmax, res):
        tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
        tree.write_dir(d)
        tree.free()
        self.tree = ctx.load_dir(d)
        self.dir = ctx.open_dir(d)
        self.ref = W.OracleDir(d)
        self.cloud = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=LEVEL)
        self.allp = self.cloud.query_union(None)  # every point in cell order
        counts = np.asarray(self.cloud.cell_counts, np.int64)
        self.starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
        self.ends = self.starts + counts
        xyz = self.allp["xyz"]
        self.mn = np.ascontiguousarray(np.minimum.reduceat(xyz, self.starts, axis=0))
        self.mx = np.ascontiguousarray(np.maximum.reduceat(xyz, self.starts, axis=0))
        self.ids = self.cloud.cells_in_location(pcv.geometry.all_points())

    def free(self):
        self.cloud.free()
        self.dir.close()
        self.tree.free()

    def oracle_cells(self, loc):
        rel = np.zeros(len(self.mn), np.int32)
        W.oracle().orc_wm_intersect_boxes(W._p(_nw_se(loc)), W._p(self.mn), W._p(self.mx), C.c_uint64(len(self.mn)), W._p(rel))
        return np.nonzero(rel != 2)[0]

    def oracle_s2_points(self, loc, filters=()):
        """The oracle's stream of the S2 cloud: the points of the selected cells, in cell order, that the rect contains and that
        pass every interval."""
        idx = np.concatenate([np.arange(self.starts[k], self.ends[k]) for k in self.oracle_cells(loc)] or [np.zeros(0, np.int64)])
        xyz = np.ascontiguousarray(self.allp["xyz"][idx])
        keep = W.contains(_nw_se(loc), xyz, W.oracle())
        v = self.allp["intensity"][idx].astype(np.float64)
        for lo, hi in filters:
            keep &= (lo <= v) & (v <= hi)
        return dict(xyz=xyz[keep], src=self.allp["src"][idx][keep])


def _make_clouds(pcv, ctx, tmp):
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED, 0, N)
    inten = (np.arange(N) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    slab = Cloud(pcv, ctx, str(tmp / "slab"), x, y, z, rgb, inten, bmin, bmax, res)
    # points beyond the map's top edge (84 - 89.9 degrees) and on both sides of the antimeridian, -500 m to 10 km
    rng = np.random.default_rng(23)
    n = 200_000
    lat = np.radians(rng.uniform(84.0, 89.9, n))
    lng = np.radians(np.where(rng.random(n) < 0.5, rng.uniform(179.0, 180.0, n), rng.uniform(-180.0, -179.0, n)))
    e = W.to_ecef(np.stack([lat, lng, rng.uniform(-500.0, 10000.0, n)], 1), W.oracle())
    px, py, pz = (np.ascontiguousarray(e[:, k]) for k in range(3))
    prgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    pint = (np.arange(n) % 1000).astype(np.float32)
    pmin, pmax = e.min(0) - 1.0, e.max(0) + 1.0
    polar = Cloud(pcv, ctx, str(tmp / "polar"), px, py, pz, prgb, pint, pmin, pmax, 0.01)
    return slab, polar


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    ctx = pcv.Context(0, max_points_per_node=3000)
    slab, polar = _make_clouds(pcv, ctx, tmp_path_factory.mktemp("wm"))
    G = pcv.geometry
    c = W.coords(np.array([W.SLAB_CENTRE]), W.oracle())[0][0]
    rects = {}
    for z, half in ((17, 128.0), (19, 200.0), (21, 128.0), (23, 300.0)):
        p = c * float(256 << z)
        rects["slab_z%d" % z] = (slab, G.web_mercator_rect(p - half, p + half, z))
    rects["slab_wrapped_z0"] = (slab, G.web_mercator_rect((255.5, c[1] * 256 - 0.3), (0.5, c[1] * 256 + 0.3), 0))
    # thin strips whose polyhedra cache 27 axes: the axes past the 26 a location record holds come from its table
    for z, hx, dy, h in ((20, 471.0, 0.5, 0.02), (19, 800.0, 0.25, 0.007)):
        p = c * float(256 << z)
        rects["slab_strip_z%d" % z] = (slab, G.web_mercator_rect(p + (-hx, dy), p + (hx, dy + h), z))
    z = 8
    zoom = float(256 << z)
    rects["polar_top_edge_z8"] = (polar, G.web_mercator_rect((zoom - 180.0, 0.0), (zoom - 1e-6, 200.0), z))
    rects["polar_antimeridian_z8"] = (polar, G.web_mercator_rect((zoom - 150.0, 20.0), (zoom - 2.0 ** -20, 220.0), z))
    rects["polar_east_z8"] = (polar, G.web_mercator_rect((0.0, 0.0), (200.0, 250.0), z))
    rects["polar_wrapped_z0"] = (polar, G.web_mercator_rect((255.6, 0.0), (0.4, 0.9), 0))
    yield dict(pcv=pcv, G=G, ctx=ctx, slab=slab, polar=polar, rects=rects, centre=c)
    slab.free()
    polar.free()
    ctx.close()


RECTS = ["slab_z17", "slab_z19", "slab_z21", "slab_z23", "slab_wrapped_z0", "slab_strip_z20", "slab_strip_z19", "polar_top_edge_z8",
         "polar_antimeridian_z8", "polar_east_z8", "polar_wrapped_z0"]


def test_strips_have_axes_past_the_record(scene):
    """The strips reach the table path: more cached axes than the record's 26 (make_query_geom of the CPU test backend)."""
    for name in ("slab_strip_z20", "slab_strip_z19"):
        assert len(W.geometry(_nw_se(scene["rects"][name][1]))[1]) > 26, name


@pytest.mark.parametrize("name", RECTS)
def test_node_and_cell_lists_equal_the_oracle(scene, name):
    cl, loc = scene["rects"][name]
    want = _oracle_nodes(cl.ref, loc)
    assert cl.tree.nodes_in_location(loc) == want
    assert cl.dir.nodes_in_location(loc) == want
    assert np.array_equal(cl.cloud.cells_in_location(loc), cl.ids[cl.oracle_cells(loc)])
    if not name.endswith("wrapped_z0") and name != "polar_east_z8":
        assert len(want) > 1, name


def _outside_band(res, nw_se):
    """The positions and sources of the points outside the band, and how many are in it.  Positions identify octree points:
    a directory's oracle load has no build index."""
    w, _ = W.coords(res["xyz"], W.oracle())
    inb = W.band_count(w, nw_se, DELTA)
    return res["xyz"][~inb], res["src"][~inb], int(inb.sum())


def _check_points(got, want, nw_se, what, by_src=False):
    gx, gs, gb = _outside_band(got, nw_se)
    ox, os_, ob = _outside_band(want, nw_se)
    print("%s: %d points, %d (gpu) / %d (oracle) in the band" % (what, len(want["src"]), gb, ob))
    assert gb < 10 and ob < 10, (what, gb, ob)
    assert np.array_equal(gx, ox), (what, len(gx), len(ox))
    if by_src:
        assert np.array_equal(gs, os_), what


@pytest.mark.parametrize("filt", [False, True], ids=["nofilt", "filt"])
@pytest.mark.parametrize("name", RECTS)
def test_points_equal_the_oracle_outside_the_band(scene, name, filt):
    cl, loc = scene["rects"][name]
    nw_se = _nw_se(loc)
    filters = FILTERS if filt else ()
    want = _oracle_query(cl.ref, loc, filters)
    res = _cat(cl.tree.query_points(loc, filters=filters, batch_size=4099))
    _check_points(res, want, nw_se, name + " octree")
    dres = _cat(cl.dir.query_points(loc, filters=filters, batch_size=1 << 20))
    _check_points(dres, want, nw_se, name + " directory")
    s2want = cl.oracle_s2_points(loc, filters)
    s2 = _cat(cl.cloud.query_points(loc, filters=filters, batch_size=7001))
    _check_points(s2, s2want, nw_se, name + " s2", by_src=True)
    counts, _ = cl.tree.query_batch_device([loc], filters=filters)
    assert int(counts[0]) == len(res["src"])
    counts, _ = cl.dir.query_batch([loc], filters=filters)
    assert int(counts[0]) == len(dres["src"])
    counts, _ = cl.cloud.query_batch_device([loc], filters=filters)
    assert int(counts[0]) == len(s2["src"])
    if name.endswith("wrapped_z0"):
        assert len(res["src"]) == len(dres["src"]) == len(s2["src"]) == 0
    elif not filt and name != "polar_east_z8":
        assert len(want["src"]) > 0, name


def test_points_next_to_every_edge(scene, tmp_path):
    """Points 1e-10 (normalised) inside and outside each edge of a zoom-21 rect, along it: exactly the oracle's answer from
    every source, and every inside point kept."""
    pcv, G, ctx = scene["pcv"], scene["G"], scene["ctx"]
    c = scene["centre"]
    z = 21
    p = c * float(256 << z)
    loc = G.web_mercator_rect(p - 100.0, p + 100.0, z)
    nw, se = _nw_se(loc)[:2], _nw_se(loc)[2:]
    t = np.linspace(0.05, 0.95, 40)
    w = []
    for s, inside in ((-1e-10, False), (1e-10, True)):
        w += [np.stack([np.full_like(t, nw[0] + s), nw[1] + t * (se[1] - nw[1])], 1), np.stack([nw[0] + t * (se[0] - nw[0]), np.full_like(t, nw[1] + s)], 1),
              np.stack([np.full_like(t, se[0] - s), nw[1] + t * (se[1] - nw[1])], 1), np.stack([nw[0] + t * (se[0] - nw[0]), np.full_like(t, se[1] - s)], 1)]
    w = np.concatenate(w)
    ll = W.to_lat_lng(w, W.oracle())
    e = W.to_ecef(np.stack([ll[:, 0], ll[:, 1], np.linspace(-400.0, 9000.0, len(w))], 1), W.oracle())
    want = W.contains(_nw_se(loc), e, W.oracle())
    assert want.sum() == len(w) // 2
    n = len(e)
    x, y, zz = (np.ascontiguousarray(e[:, k]) for k in range(3))
    rgb = np.zeros((n, 3), np.uint8)
    inten = np.zeros(n, np.float32)
    cl = Cloud(pcv, ctx, str(tmp_path / "edges"), x, y, zz, rgb, inten, e.min(0) - 1.0, e.max(0) + 1.0, 0.0001)
    try:
        got_xyz = _cat(cl.tree.query_points(loc))["xyz"]
        assert np.array_equal(W.contains(_nw_se(loc), got_xyz, W.oracle()), np.ones(len(got_xyz), bool))
        o = _oracle_query(cl.ref, loc)
        assert np.array_equal(_cat(cl.tree.query_points(loc))["xyz"], o["xyz"])
        assert np.array_equal(_cat(cl.dir.query_points(loc))["xyz"], o["xyz"])
        assert np.array_equal(_cat(cl.cloud.query_points(loc))["src"], cl.oracle_s2_points(loc)["src"])
        assert len(o["src"]) == int(W.contains(_nw_se(loc), o["xyz"], W.oracle()).sum()) == len(w) // 2
    finally:
        cl.free()


def test_mixed_batch_counts(scene):
    """Rects, frusta and OBBs in one batch: each location's counts are those of its single-location call."""
    G = scene["G"]
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    ecef_from_local = G.Isometry(W.SLAB_CENTRE, q)
    locs = [scene["rects"]["slab_z21"][1], G.frustum(ecef_from_local, G.Perspective.new_fov(1.0, 1.2, 0.1, 10.0)), scene["rects"]["slab_z19"][1],
            G.obb(ecef_from_local, (50.0, 50.0, 5.0)), scene["rects"]["slab_wrapped_z0"][1], scene["rects"]["slab_strip_z20"][1],
            scene["rects"]["slab_z23"][1], scene["rects"]["slab_strip_z19"][1]]
    cl = scene["slab"]
    for filters in ((), FILTERS):
        for fn in (cl.tree.query_batch_device, cl.dir.query_batch, cl.cloud.query_batch_device):
            counts, tested = fn(locs, filters=filters)
            for i, loc in enumerate(locs):
                c1, t1 = fn([loc], filters=filters)
                assert (int(counts[i]), int(tested[i])) == (int(c1[0]), int(t1[0])), (fn, i)


def test_rect_query_equality_octree_vs_s2(scene):
    """check_web_mercator_rect_query_equality: the zoom-21, 256 x 256 px rect around the slab centre (queries.rs:59-72) streams
    the same indexed points from the octree and from the S2 cloud (main.rs:139-204)."""
    from test_zz7_s2_location_query_gpu import _assert_points_equal, _indexed

    import point_cloud_viewer_b200 as pcv

    loc = scene["rects"]["slab_z21"][1]
    _, _, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    cl = scene["slab"]
    a = _cat(cl.tree.query_points(loc, batch_size=1 << 20))
    b = _cat(cl.cloud.query_points(loc, batch_size=1 << 20))
    _assert_points_equal(_indexed(a["xyz"], a["rgb"]), _indexed(b["xyz"], b["rgb"]), res)


@pytest.mark.parametrize("mn,mx,z", [((0.0, 0.0), (1.0, 1.0), 24), ((-1.0, 0.0), (0.5, 0.5), 0), ((0.0, 0.0), (256.0, 0.5), 0),
                                     ((0.0, 100.0), (0.5, 99.0), 0), ((10.0, 10.0), (11.5, 10.5), 0), ((math.nan, 0.0), (0.5, 0.5), 0)])
def test_constructor_rejects_with_value_error(scene, mn, mx, z):
    with pytest.raises(ValueError):
        scene["G"].web_mercator_rect(mn, mx, z)


@pytest.mark.parametrize("nw_se", [(0.5, 0.5, 0.5, 0.49), (0.5, 0.5, 0.51, 0.5), (1.0, 0.5, 0.5, 0.5), (-0.1, 0.5, 0.5, 0.5), (0.5, math.nan, 0.5, 0.5),
                                   (0.5, 0.5, math.inf, 0.5)])
def test_invalid_kind4_locations_are_rejected(scene, nw_se):
    pcv = scene["pcv"]
    loc = pcv.geometry.Location()
    loc.kind = pcv.geometry.LOC_WEB_MERCATOR_RECT
    loc.aabb_min[0], loc.aabb_min[1], loc.aabb_max[0], loc.aabb_max[1] = nw_se
    cl = scene["slab"]
    calls = [lambda: cl.tree.nodes_in_location(loc), lambda: cl.tree.query_points(loc), lambda: cl.tree.query_batch_device([loc]),
             lambda: cl.dir.nodes_in_location(loc), lambda: cl.dir.query_points(loc), lambda: cl.dir.query_batch([loc]),
             lambda: cl.cloud.cells_in_location(loc), lambda: cl.cloud.query_points(loc), lambda: cl.cloud.query_batch_device([loc])]
    for f in calls:
        with pytest.raises(pcv.PcvError) as e:
            f()
        assert e.value.code == -1


def test_web_mercator_coord(scene):
    """geometry.web_mercator_coord is the point test's map position at zoom z; z > 23 is a ValueError."""
    G = scene["G"]
    e = W.slab_points(1000)
    w, _ = W.coords(e, W.oracle())
    for z in (0, 12, 23):
        got = np.array([G.web_mercator_coord(p, z) for p in e])
        assert np.array_equal(got, w * float(256 << z))
    with pytest.raises(ValueError):
        G.web_mercator_coord(e[0], 24)
