"""Location queries of the S2-cell cloud on the GPU (pcv_s2_cells_in_location, pcv_s2_query_points, pcv_s2_query_cell_union,
pcv_s2_query_batch_device, pcv_s2_query_cell_unions_batch_device) on the 1e6-point slab of test_zz5 (seed 80293751232, split level
20, resolution 0.001):
- the reference's integration test (point_cloud_test/tests/main.rs:87-160) completed: the box, OBB and frustum of queries.rs
  stream the same indexed points from the S2 cloud and from the octree, up to the reference's tolerance;
- exact against the oracle: the cell list is the cells whose numpy point box orc_cached_intersect_aabb does not call Out, in id
  order; the stream is, element for element, the oracle-filtered points of those cells in cell order, and equals the
  brute-force filter of all points (the selection drops nothing);
- filter intervals, cell unions with filters, batched counts over 1, 64 and 2000 frusta (more than one selection chunk), the
  query statistics, and the stream mechanics (batch sizes, cancellation, no colour, directory round trip, build statistics)."""
import ctypes as C

import numpy as np
import pytest

import oracle_api as O
import s2_api as S

pytestmark = pytest.mark.gpu

SEED, LEVEL, N = 80293751232, 20, 1_000_000
SELECT_PAIRS = 1 << 18  # kS2SelectPairs (csrc/s2_api.inl): the (location, cell) pairs of one selection chunk


def _oloc(loc):
    o = O.Location()
    for f, _ in O.Location._fields_:
        setattr(o, f, getattr(loc, f))
    return o


def _indexed(xyz, rgb):  # main.rs:139-140
    idx = (rgb[:, 0].astype(np.int64) << 16) + (rgb[:, 1].astype(np.int64) << 8) + rgb[:, 2].astype(np.int64)
    o = np.argsort(idx, kind="stable")
    return idx[o], xyz[o]


def _assert_points_equal(a, b, resolution, share=0.99):  # main.rs:160-204, the rules of test_zz5_s2_vs_octree_gpu.py
    ia, pa = a
    ib, pb = b
    assert len(ia) and len(ib), "The query returned no points (using streaming)"
    common, ka, kb = np.intersect1d(ia, ib, return_indices=True)
    skipped = (len(ia) - len(common)) + (len(ib) - len(common))
    assert skipped <= -(-min(len(ia), len(ib)) // 100), (skipped, len(ia), len(ib))
    dist = np.linalg.norm(pa[ka] - pb[kb], axis=1)
    thr = np.sqrt(3.0) * 2.0 * resolution
    assert (dist <= thr).mean() >= share and dist.max() <= 2 * thr, ((dist <= thr).mean(), dist.max())


def _cat(batches):
    if not batches:
        return dict(xyz=np.zeros((0, 3)), rgb=np.zeros((0, 3), np.uint8), intensity=np.zeros(0, np.float32), src=np.zeros(0, np.uint64))
    out = {k: np.concatenate([b[k] for b in batches]) for k in ("xyz", "src")}
    out["rgb"] = None if batches[0]["rgb"] is None else np.concatenate([b["rgb"] for b in batches])
    out["intensity"] = None if batches[0]["intensity"] is None else np.concatenate([b["intensity"] for b in batches])
    return out


def _frusta(G, bmin, bmax, count, far, seed=7):  # bench.make_frusta
    rng = np.random.default_rng(seed)
    persp = G.Perspective.new_fov(1.0, 1.2, 0.1, far)
    out = []
    for _ in range(count):
        eye = bmin + rng.random(3) * (bmax - bmin)
        q = rng.random((4, 12)).sum(1) - 6.0
        out.append(G.frustum(G.Isometry(eye, q / np.linalg.norm(q)), persp))
    return out


@pytest.fixture(scope="module")
def scene(ctx):
    import point_cloud_viewer_b200 as pcv

    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED, 0, N)
    inten = (np.arange(N) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    bmin, bmax = np.asarray(bmin, np.float64), np.asarray(bmax, np.float64)
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax)
    cloud = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=LEVEL)
    allp = cloud.query_union(None)  # every point in cell order
    starts = np.concatenate([[0], np.cumsum(cloud.cell_counts)[:-1]]).astype(np.int64)
    assert (cloud.cell_counts > 0).all()
    xyz = allp["xyz"]
    boxes = (np.minimum.reduceat(xyz, starts, axis=0), np.maximum.reduceat(xyz, starts, axis=0))
    G = pcv.geometry
    d = bmax - bmin
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    ecef_from_local = G.Isometry((4157222.543, 664789.307, 4774952.099), q)
    mn, mx = boxes
    k0, k1 = len(starts) // 3, 2 * len(starts) // 3
    locs = {  # test_query_gpu.py::_locations, one location that misses every cell, one whose faces cut through cell boxes
        "all": G.all_points(),
        "aabb": G.aabb(bmin + 0.2 * d, bmin + 0.8 * d),
        "aabb_small": G.aabb(bmin + 0.45 * d, bmin + 0.5 * d),
        "obb": G.obb(ecef_from_local, (50.0, 50.0, 5.0)),
        "frustum": G.frustum(ecef_from_local, G.Perspective.new_fov(1.0, 1.2, 0.1, 10.0)),
        "frustum_far": G.frustum(ecef_from_local * G.Isometry((0, 0, 0), G.quat_from_axis_angle([1, 0.3, 0], 1.3)), G.Perspective.new_fov(1.3, 0.9, 0.5, 150.0)),
        "obb_tilted": G.obb(ecef_from_local * G.Isometry((10, -20, 1), G.quat_from_axis_angle([0.2, 0.5, -0.7], 0.523)), (30.0, 12.0, 4.0)),
        "miss": G.aabb(bmax + 1000.0, bmax + 1100.0),
        "cut": G.aabb(np.minimum(0.5 * (mn[k0] + mx[k0]), 0.5 * (mn[k1] + mx[k1])), np.maximum(0.5 * (mn[k0] + mx[k0]), 0.5 * (mn[k1] + mx[k1]))),
    }
    yield dict(pcv=pcv, G=G, tree=tree, cloud=cloud, allp=allp, starts=starts, boxes=boxes, locs=locs, res=res, bmin=bmin, bmax=bmax,
               x=x, y=y, z=z, rgb=rgb, inten=inten, ecef_from_local=ecef_from_local)
    cloud.free()
    tree.free()


def _selected(s, loc):
    """Indices of the cells the contract selects: every cell for AllPoints, else sat(location, point box) != Out (oracle)."""
    if loc.kind == 0:
        return np.arange(len(s["starts"]))
    L, o = O.lib(), _oloc(loc)
    mn, mx = s["boxes"]
    return np.array([k for k in range(len(mn)) if L.orc_cached_intersect_aabb(C.byref(o), O._d(mn[k]), O._d(mx[k])) != 2], np.int64)


def _passes(s, filters):
    keep = np.ones(len(s["allp"]["src"]), bool)
    v = s["allp"]["intensity"].astype(np.float64)
    for lo, hi in filters:
        keep &= (lo <= v) & (v <= hi)
    return keep


def _expected(s, loc, filters=()):
    """(slots of the expected stream in order, slots of the brute-force filter of all points)."""
    sel = _selected(s, loc)
    counts = s["cloud"].cell_counts.astype(np.int64)
    in_sel = np.zeros(len(s["allp"]["src"]), bool)
    for k in sel:
        in_sel[s["starts"][k]: s["starts"][k] + counts[k]] = True
    ok = O.location_contains(_oloc(loc), s["allp"]["xyz"]) & _passes(s, filters)
    return sel, np.nonzero(in_sel & ok)[0], np.nonzero(ok)[0]


def _assert_stream_is(s, got, slots):
    a = s["allp"]
    assert len(got["src"]) == len(slots)
    assert np.array_equal(got["xyz"].view(np.uint64), a["xyz"][slots].view(np.uint64))
    assert np.array_equal(got["rgb"], a["rgb"][slots])
    assert np.array_equal(got["intensity"].view(np.uint32), a["intensity"][slots].view(np.uint32))
    assert np.array_equal(got["src"], a["src"][slots])


def test_s2_and_octree_location_queries_agree(scene):
    s = scene
    P = np.stack([s["x"], s["y"], s["z"]], 1)
    for name in ("aabb", "obb", "frustum"):  # check_box_query_equality, check_obb_query_equality, check_frustum_query_equality
        loc = s["locs"][name]
        oct_ = _cat(s["tree"].query_points(loc, batch_size=5000 * 40))
        s2 = _cat(s["cloud"].query_points(loc, batch_size=5000 * 40))
        # the S2 side holds the input positions themselves, so every distance below is the octree's own fix-point error: over the
        # whole slab >= 99 % of the points are within 2 sqrt(3) resolution (test_zz5), but inside these locations only 98.5-99 %
        # (measured on an H100), so only the bound that holds for every point, twice that, is kept
        assert np.array_equal(s2["xyz"].view(np.uint64), P[s2["src"].astype(np.int64)].view(np.uint64))
        _assert_points_equal(_indexed(s2["xyz"], s2["rgb"]), _indexed(oct_["xyz"], oct_["rgb"]), s["res"], share=0.0)


def test_cells_and_stream_exact_against_oracle(scene):
    s = scene
    ids = s["cloud"].cell_ids
    for name, loc in s["locs"].items():
        sel, want, brute = _expected(s, loc)
        assert np.array_equal(s["cloud"].cells_in_location(loc), ids[sel]), name
        got = _cat(s["cloud"].query_points(loc, batch_size=100_003))
        _assert_stream_is(s, got, want)
        assert np.array_equal(want, brute), name  # the selection drops no point
        if name == "miss":
            assert len(sel) == 0 and len(want) == 0
        elif name != "cut":
            assert len(want) > 0, name
    mn, mx = s["boxes"]  # the cut location does cut cells: some selected box is not inside it
    cut = s["locs"]["cut"]
    sel = _selected(s, cut)
    inside = (mn[sel] >= np.asarray(cut.aabb_min)).all(1) & (mx[sel] <= np.asarray(cut.aabb_max)).all(1)
    assert len(sel) > 0 and not inside.all()


@pytest.mark.parametrize("filters", [[(100.0, 600.0)], [(100.0, 600.0), (300.0, 900.0)], [(600.0, 100.0)], [(-10.0, -1.0)]],
                         ids=["one", "two", "empty", "excludes_all"])
def test_filters(scene, filters):
    s = scene
    for name in ("all", "aabb", "obb", "frustum_far"):
        loc = s["locs"][name]
        _, want, brute = _expected(s, loc, filters)
        got = _cat(s["cloud"].query_points(loc, filters=filters, batch_size=65536))
        _assert_stream_is(s, got, want)
        assert np.array_equal(want, brute)
        counts, _ = s["cloud"].query_batch_device([loc], filters=filters)
        assert int(counts[0]) == len(want), name
        if filters[0][0] > filters[0][1] or filters[0][1] < 0:
            assert len(want) == 0


def test_filters_need_intensity(scene, ctx):
    import point_cloud_viewer_b200 as pcv

    s = scene
    plain = ctx.build_s2_cloud(s["x"], s["y"], s["z"], s["rgb"], None, split_level=LEVEL)
    try:
        for call in (lambda: plain.query_points(s["locs"]["aabb"], filters=[(0.0, 1.0)]),
                     lambda: plain.query_batch_device([s["locs"]["aabb"]], filters=[(0.0, 1.0)]),
                     lambda: plain.query_points(s["G"].cell_union(plain.cell_ids[:2]), filters=[(0.0, 1.0)])):
            with pytest.raises(pcv.PcvError) as e:
                call()
            assert e.value.code == -1 and "Filter attribute needs to be specified as query attribute." in str(e.value)
    finally:
        plain.free()


def test_cell_unions_with_filters(scene):
    s = scene
    G, cloud = s["G"], s["cloud"]
    centre = np.array([[4157222.543, 664789.307, 4774952.099]])
    cell = int(S.oracle_cell_ids(centre, LEVEL)[0])
    unions = [np.array([cell, S.orc().orc_s2_next(cell)], np.uint64), np.array([S.orc().orc_s2_parent(cell, LEVEL - 2)], np.uint64),
              np.array([int(cloud.cell_ids[3]), int(cloud.cell_ids[-2])], np.uint64)]
    filters = [(100.0, 600.0)]
    for u in unions:
        ref = cloud.query_union(u)
        v = ref["intensity"].astype(np.float64)
        m = (100.0 <= v) & (v <= 600.0)
        got = _cat(cloud.query_points(G.cell_union(u), filters=filters, batch_size=50_000))
        assert 0 < len(got["src"]) < len(ref["src"])
        assert np.array_equal(got["xyz"].view(np.uint64), ref["xyz"][m].view(np.uint64))
        assert np.array_equal(got["src"], ref["src"][m]) and np.array_equal(got["rgb"], ref["rgb"][m])
        nofilt = _cat(cloud.query_points(G.cell_union(u)))
        assert np.array_equal(nofilt["src"], ref["src"])
        assert np.array_equal(cloud.cells_in_location(G.cell_union(u)), cloud.cells_in_union(u))
    counts, tested = cloud.query_batch_device([G.cell_union(u) for u in unions], filters=filters)
    for k, u in enumerate(unions):
        ref = cloud.query_union(u)
        v = ref["intensity"].astype(np.float64)
        assert int(counts[k]) == int(((100.0 <= v) & (v <= 600.0)).sum()) and int(tested[k]) == ref["tested"]
    assert cloud.query_points(G.cell_union([])) == [] and len(cloud.cells_in_location(G.cell_union([]))) == 0
    counts, tested = cloud.query_batch_device([G.cell_union([])])
    assert counts.tolist() == [0] and tested.tolist() == [0]


def test_batches_and_stats(scene):
    s = scene
    G, cloud = s["G"], s["cloud"]
    ncells = len(cloud.cell_ids)
    assert 2000 * ncells > SELECT_PAIRS > 64 * ncells  # 2000 frusta take more than one selection chunk, 64 take one
    F = _frusta(G, s["bmin"], s["bmax"], 2000, 10.0)
    counts64, tested64 = cloud.query_batch_device(F[:64])
    st = cloud.last_query_stats()
    pairs = 0
    for k in range(64):
        got = _cat(cloud.query_points(F[k], batch_size=1 << 20))
        assert int(counts64[k]) == len(got["src"]), k
        cells = cloud.cells_in_location(F[k])
        sel = np.searchsorted(cloud.cell_ids, cells)
        assert int(tested64[k]) == int(cloud.cell_counts[sel].sum()), k
        pairs += len(cells)
    assert counts64.sum() > 0
    assert st["tested_points"] == tested64.sum() and st["returned_points"] == counts64.sum() == st["stored_points"]
    assert st["visited_pairs"] == pairs and st["kernel_launches"] > 0
    assert st["ms_device"] >= st["ms_cull"] > 0 and st["ms_select"] > 0
    assert st["algorithmic_bytes"] == 24 * st["tested_points"] + (24 + 3 + 4) * st["returned_points"]
    c1, t1 = cloud.query_batch_device(F[:1])
    assert c1[0] == counts64[0] and t1[0] == tested64[0]
    call, tall = cloud.query_batch_device(F)
    st = cloud.last_query_stats()
    assert np.array_equal(call[:64], counts64) and np.array_equal(tall[:64], tested64)
    parts = [cloud.query_batch_device(F[i: i + 64]) for i in range(0, 2000, 64)]
    assert np.array_equal(call, np.concatenate([p[0] for p in parts])) and np.array_equal(tall, np.concatenate([p[1] for p in parts]))
    assert st["tested_points"] == tall.sum() and st["returned_points"] == call.sum()
    with pytest.raises(ValueError):
        cloud.query_batch_device([F[0], G.cell_union([int(cloud.cell_ids[0])])])


def test_stream_mechanics(scene, ctx, tmp_path):
    import point_cloud_viewer_b200 as pcv

    s = scene
    cloud, loc = s["cloud"], s["locs"]["aabb"]
    batches = cloud.query_points(loc, batch_size=7777)
    assert len(batches) > 2 and all(len(b["src"]) == 7777 for b in batches[:-1]) and 0 < len(batches[-1]["src"]) <= 7777
    calls = []

    def stop(b):
        calls.append(len(b["src"]))
        return True

    with pytest.raises(pcv.PcvError) as e:
        cloud.query_points(loc, callback=stop, batch_size=1000)
    assert e.value.code == -5 and calls == [1000]
    # a cloud without colour: rgb is None, everything else equal
    nocol = ctx.build_s2_cloud(s["x"], s["y"], s["z"], None, s["inten"], split_level=LEVEL)
    try:
        a, b = _cat(batches), _cat(nocol.query_points(loc, batch_size=7777))
        assert all(bb["rgb"] is None for bb in nocol.query_points(loc, batch_size=100_000))
        assert b["rgb"] is None and np.array_equal(a["xyz"].view(np.uint64), b["xyz"].view(np.uint64)) and np.array_equal(a["src"], b["src"])
        assert np.array_equal(a["intensity"], b["intensity"])
        assert np.array_equal(nocol.query_batch_device([loc])[0], cloud.query_batch_device([loc])[0])
    finally:
        nocol.free()
    # write_dir + load_dir: the same cells and points (the loaded cloud's src is the slot)
    cloud.write_dir(str(tmp_path))
    loaded = ctx.load_s2_dir(str(tmp_path))
    try:
        for name in ("aabb", "obb_tilted", "frustum_far"):
            l = s["locs"][name]
            a, b = _cat(cloud.query_points(l)), _cat(loaded.query_points(l))
            assert np.array_equal(cloud.cells_in_location(l), loaded.cells_in_location(l))
            assert np.array_equal(a["xyz"].view(np.uint64), b["xyz"].view(np.uint64)) and np.array_equal(a["rgb"], b["rgb"])
            assert np.array_equal(a["intensity"], b["intensity"])
            assert np.array_equal(s["allp"]["src"][b["src"].astype(np.int64)], a["src"])
            assert np.array_equal(cloud.query_batch_device([l])[0], loaded.query_batch_device([l])[0])
    finally:
        loaded.free()
    # the build statistics of a fresh cloud do not change with the first location query (the cell tables are built lazily)
    fresh = ctx.build_s2_cloud(s["x"], s["y"], s["z"], s["rgb"], s["inten"], split_level=LEVEL)
    try:
        before = fresh.build_stats()
        fresh.query_points(s["locs"]["obb"])
        fresh.query_batch_device([s["locs"]["frustum"]])
        assert fresh.build_stats() == before
    finally:
        fresh.free()


def test_argument_errors(scene, ctx):
    import point_cloud_viewer_b200 as pcv

    s = scene
    cloud, G = s["cloud"], s["G"]
    bad = G.aabb((0, 0, 0), (1, 1, 1))
    bad.kind = 7
    for call in (lambda: cloud.query_points(bad), lambda: cloud.cells_in_location(bad), lambda: cloud.query_batch_device([bad]),
                 lambda: cloud.query_points(s["locs"]["aabb"], batch_size=0), lambda: cloud.query_points(G.cell_union([2])),
                 lambda: cloud.query_batch_device([G.cell_union([2])])):
        with pytest.raises(pcv.PcvError) as e:
            call()
        assert e.value.code == -1
    counts, tested = cloud.query_batch_device([])
    assert len(counts) == 0 and len(tested) == 0
    empty = ctx.build_s2_cloud(np.zeros(0), np.zeros(0), np.zeros(0), np.zeros((0, 3), np.uint8), np.zeros(0, np.float32))
    try:
        assert empty.query_points(s["locs"]["aabb"]) == [] and len(empty.cells_in_location(s["locs"]["aabb"])) == 0
        assert empty.query_batch_device([s["locs"]["aabb"]])[0].tolist() == [0]
        assert empty.query_points(G.cell_union(cloud.cell_ids[:1])) == []
    finally:
        empty.free()
