"""S2 GPU paths off the slab: the edge fixtures of tests/s2_edges.py (cube corners and edges, the whole globe, cell and face
boundaries with their one-ulp neighbours, face ties, signed zeros, one heavily repeated position) through every S2 entry point,
bit for bit against the oracle and, away from ties, against the exact reference of tests/s2_exact.py:
- cell ids at levels 0, 1, 15, 29 and 30, SoA and AoS;
- the split at levels 0, 1, 7, 20 and 30 (ids, counts, per-cell input order, cell data, a bounding box with negative components);
- streaming to disk at levels 0 and 30 over several batches, byte for byte the in-core directory;
- box, OBB and frustum queries across each cube corner and across the zero planes: cell lists from the oracle's test of the numpy
  point boxes (negative keys of the box reduction), streams equal to the oracle-filtered cells and to the brute force, resident
  and through an S2 directory at two budgets, and batches of 64 frusta at level 30 (one location per selection chunk);
- cell unions of faces, faces with leaves on the neighbouring face, leaves at face edges, and of 255, 256, 257, 4096 and about
  100 000 ids (past the 256 ids the cull kernels stage in shared memory), un-normalised too, through every S2 union entry, the S2
  directory, batches mixing small and large unions, and the octree and octree directory;
- X-ray quadtrees over a corner patch whose leaves hold cells of three faces, resident and from the directory."""
import numpy as np
import pytest

import oracle_api as O
import s2_api as S
import s2_edges as E
import s2_exact as X
from test_octree_dir_query_gpu import _smallest_budget as _octree_dir_smallest_budget
from test_s2_exact_ref import SUBSAMPLE
from test_s2_xray_oracle_points import points_quadtree
from test_zz6_octree_cell_union_gpu import _assert_stream_equal, _stream, _tree_info, _want
from test_zz6_octree_cell_union_gpu import _cat as _octree_cat
from test_zz7_s2_location_query_gpu import _assert_stream_is, _cat, _expected, _frusta, _oloc
from test_zzb_s2_to_dir_gpu import BUDGET_PTS, _files
from test_zzc_s2_dir_xray_gpu import _same
from test_zzd_s2_dir_query_gpu import _smallest_budget

pytestmark = pytest.mark.gpu

SELECT_PAIRS = 1 << 18  # kS2SelectPairs (csrc/s2_api.inl)
CELLS_SHARED = 256      # kCellsShared (csrc/query.cuh): larger unions are read from global memory
QUERY_TILE = 2048       # kQueryTile (csrc/query.cuh)


def _soa(P):
    return [np.ascontiguousarray(P[:, k]) for k in range(3)]


@pytest.fixture(scope="module")
def fx():
    return E.all_fixtures()


@pytest.fixture(scope="module")
def exact(fx):
    """name -> (rows, exact leaf ids, tie mask) over the subsample test_s2_exact_ref walks."""
    out = {}
    for name, P in fx.items():
        rows = np.arange(len(P))[SUBSAMPLE[name]]
        leaf, tie = X.cell_ids(P[rows])
        out[name] = (rows, leaf, tie)
    return out


@pytest.mark.parametrize("level", [0, 1, 15, 29, 30])
def test_cell_ids(ctx, fx, exact, level):
    for name, P in fx.items():
        want = S.oracle_cell_ids(P, level)
        got = ctx.s2_cell_ids(*_soa(P), level)
        assert np.array_equal(got, want), (name, level)
        A = np.ascontiguousarray(P)
        aos = ctx.s2_cell_ids(A.ctypes.data, A.ctypes.data + 8, A.ctypes.data + 16, level, stride=3, n=len(A))
        assert np.array_equal(aos, want), (name, level)
        rows, leaf, tie = exact[name]
        assert np.array_equal(got[rows][~tie], X.parent(leaf, level)[~tie]), (name, level)
        if name == "boundaries":
            assert tie.sum() > 0 and (~tie).sum() > 0


def _check_split(cloud, P, rgb, inten, level):
    want = S.split(P, level)
    assert want["ok"] and cloud.num_points == len(P) and cloud.split_level == level
    assert np.array_equal(cloud.cell_ids, want["ids"]) and np.array_equal(cloud.cell_counts, want["counts"])
    assert np.array_equal(cloud.bbox_min.view(np.uint64), want["bmin"].view(np.uint64))
    assert np.array_equal(cloud.bbox_max.view(np.uint64), want["bmax"].view(np.uint64))
    order = want["order"].astype(np.int64)
    allp = cloud.query_union(None)  # every cell's points, in cell order and input order inside the cell
    assert allp["total"] == len(P) and np.array_equal(allp["src"], want["order"])
    assert np.array_equal(allp["xyz"].view(np.uint64), P[order].view(np.uint64))
    assert np.array_equal(allp["rgb"], rgb[order]) and np.array_equal(allp["intensity"].view(np.uint32), inten[order].view(np.uint32))
    starts = np.concatenate([[0], np.cumsum(want["counts"])]).astype(np.int64)
    big = int(np.argmax(want["counts"]))
    for k in sorted({0, len(want["ids"]) - 1, big, len(want["ids"]) // 2}):
        xyz, c, it, src = cloud.cell_data(want["ids"][k])
        idx = order[starts[k]:starts[k + 1]]
        assert np.array_equal(src, want["order"][starts[k]:starts[k + 1]]) and np.array_equal(xyz.view(np.uint64), P[idx].view(np.uint64))
        assert np.array_equal(c, rgb[idx]) and np.array_equal(it, inten[idx])
    return want


@pytest.mark.parametrize("level", [0, 1, 7, 20, 30])
def test_split(ctx, fx, level):
    for name in ("corners", "edges", "globe", "heavy"):
        P = fx[name]
        rgb, inten = E.attributes(len(P))
        cloud = ctx.build_s2_cloud(*_soa(P), rgb, inten, split_level=level)
        try:
            want = _check_split(cloud, P, rgb, inten, level)
            if name == "globe" and level in (0, 30):  # the extremes: six cells of ~170 000 points, or one point per cell
                import point_cloud_viewer_b200 as pcv

                G = pcv.geometry
                box = G.aabb((-7.0e6, -7.0e6, -7.0e6), (3.0e5, -2.0e5, 1.0e5))
                counts, _ = cloud.query_batch_device([box])
                assert int(counts[0]) == int(O.location_contains(_oloc(box), P).sum()) > 0
                counts, tested = cloud.query_batch_device([G.cell_union([_face_cell(4)])])
                assert int(counts[0]) == int(tested[0]) == int((S.oracle_cell_ids(P, 0) == np.uint64(_face_cell(4))).sum())
        finally:
            cloud.free()
        assert (want["bmin"] < 0).any(), name
        if name == "heavy":
            assert int(want["counts"].max()) >= 10_000 > QUERY_TILE
            if level == 30:
                assert (want["counts"] == 1).sum() > 1000
        if name == "globe":
            assert len(np.unique(want["ids"] >> np.uint64(61))) == 6 and (want["bmin"] < -6e6).all() and (want["bmax"] > 6e6).all()


@pytest.mark.parametrize("level", [0, 30])
def test_stream_to_disk(ctx, fx, tmp_path, level):
    if level == 0:
        P = np.concatenate([fx["globe"], fx["corners"], fx["edges"], fx["heavy"]])
        budget = BUDGET_PTS(300_000)
    else:  # about 10 000 cells: the directory holds three files per cell
        P = np.concatenate([fx["corners"][::80], fx["heavy"], fx["boundaries"][::4]])
        budget = BUDGET_PTS(4096)
    rgb, inten = E.attributes(len(P), 3)
    cloud = ctx.build_s2_cloud(*_soa(P), rgb, inten, split_level=level)
    try:
        cloud.write_dir(str(tmp_path / "core"))
        ncells = cloud.num_cells
    finally:
        cloud.free()
    want = _files(str(tmp_path / "core"))
    info = ctx.build_s2_dir(str(tmp_path / "streamed"), *_soa(P), rgb, inten, split_level=level, max_device_bytes=budget)
    got = _files(str(tmp_path / "streamed"))
    assert info["batches"] > 1 and info["num_points"] == len(P) and info["num_cells"] == ncells
    assert got.keys() == want.keys() and "meta.pb" in got
    for f in want:
        assert got[f] == want[f], f


# ---- location queries ------------------------------------------------------------------------------------------------------
def _scene(cloud):
    allp = cloud.query_union(None)
    counts = cloud.cell_counts.astype(np.int64)
    assert (counts > 0).all()
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    xyz = allp["xyz"]
    boxes = (np.minimum.reduceat(xyz, starts, axis=0), np.maximum.reduceat(xyz, starts, axis=0))
    return dict(cloud=cloud, allp=allp, starts=starts, boxes=boxes)


def _rot(axis, angle):
    import point_cloud_viewer_b200 as pcv

    return pcv.geometry.quat_from_axis_angle(axis, angle)


def _corner_locations(G):
    """A box, an OBB and a frustum across each cube corner (every one cuts the three faces meeting there)."""
    locs = {}
    rng = np.random.default_rng(17)
    for k, d in enumerate(E.corner_directions()):
        c = E.R * d
        locs["aabb%d" % k] = G.aabb(c - (150.0, 120.0, 90.0), c + (110.0, 140.0, 100.0))
        q = G.quat_mul(_rot([0.3, -0.5, 0.8], 0.4 + 0.3 * k), _rot([1, 0, 0], -0.7))
        locs["obb%d" % k] = G.obb(G.Isometry(c + rng.uniform(-20, 20, 3), q), (180.0, 90.0, 45.0))
        # the eye 150 m above the corner, looking down at it (the eye looks along its -z axis), turned about the vertical
        down = G.quat_mul(G.quat_from_axis_angle(np.cross((0.0, 0.0, 1.0), d), np.arccos(d[2])), G.quat_from_axis_angle((0, 0, 1), 0.5 * k))
        locs["frustum%d" % k] = G.frustum(G.Isometry(c + d * 150.0, down), G.Perspective.new_fov(1.1, 1.4, 0.5, 400.0))
    return locs


def _globe_locations(G):
    """Locations across the zero planes of the globe."""
    q = G.quat_mul(_rot([0, 0, 1], 0.6), _rot([0, 1, 0], -0.8))
    h = E.HEAVY_POINT * (E.R / np.linalg.norm(E.HEAVY_POINT))
    return {
        "all": G.all_points(),
        "slab_xy": G.aabb((-2.0e6, -1.5e6, -7.0e6), (1.8e6, 2.2e6, 7.0e6)),
        "slab_yz": G.aabb((-7.0e6, -0.9e6, -1.1e6), (7.0e6, 1.0e6, 0.8e6)),
        "octant": G.aabb((-7.0e6, -7.0e6, -7.0e6), (3.0e5, -2.0e5, 1.0e5)),
        "pole_box": G.aabb((-3.0e5, -E.R_MAX, -2.5e5), (3.5e5, -E.R_MIN + 1.0, 3.0e5)),
        "obb_centre": G.obb(G.Isometry((0.0, 0.0, 0.0), q), (7.0e6, 1.2e6, 0.9e6)),
        "frustum_origin": G.frustum(G.Isometry((0.0, 0.0, 0.0), G.quat_mul(q, _rot([1, 0, 0], 2.0))), G.Perspective.new_fov(1.3, 0.9, 0.1, 7.0e6)),
        "heavy_box": G.aabb(h - 1.0, h + 1.0),
        "miss": G.aabb((0.0, 0.0, 0.0), (1.0e6, 1.0e6, 1.0e6)),
    }


def _check_locations(s, locs, d, ctx, budgets):
    """Resident cells and stream against the oracle, then the same through the S2 directory at each budget."""
    pcv_ids = s["cloud"].cell_ids
    want = {}
    for name, loc in locs.items():
        sel, slots, brute = _expected(s, loc)
        assert np.array_equal(slots, brute), name  # the selection drops no point
        assert np.array_equal(s["cloud"].cells_in_location(loc), pcv_ids[sel]), name
        _assert_stream_is(s, _cat(s["cloud"].query_points(loc, batch_size=100_003)), slots)
        want[name] = (sel, slots)
    counts, tested = s["cloud"].query_batch_device(list(locs.values()))
    cc = s["cloud"].cell_counts.astype(np.int64)
    assert [int(v) for v in counts] == [len(w[1]) for w in want.values()]
    assert [int(v) for v in tested] == [int(cc[w[0]].sum()) for w in want.values()]
    import point_cloud_viewer_b200 as pcv

    for budget in budgets:
        h = pcv.S2Dir(ctx, d, budget)
        try:
            assert np.array_equal(h.cell_ids, pcv_ids) and np.array_equal(h.bbox_min, s["cloud"].bbox_min)
            for name, loc in locs.items():
                sel, slots = want[name]
                assert np.array_equal(h.cells_in_location(loc), pcv_ids[sel]), (name, budget)
                got = _cat(h.query_points(loc, batch_size=65_536))
                assert np.array_equal(got["xyz"].view(np.uint64), s["allp"]["xyz"][slots].view(np.uint64)), (name, budget)
                assert np.array_equal(got["src"].astype(np.int64), slots) and np.array_equal(got["rgb"], s["allp"]["rgb"][slots])
            c2, t2 = h.query_batch(list(locs.values()))
            assert np.array_equal(c2, counts) and np.array_equal(t2, tested)
        finally:
            h.close()
    return want


@pytest.fixture(scope="module")
def corner_cloud(ctx, fx, tmp_path_factory):
    """All eight corner patches in one cloud at level 16 (cells of about 150 m, three faces per patch), and its directory."""
    P = fx["corners"]
    rgb, inten = E.attributes(len(P), 5)
    cloud = ctx.build_s2_cloud(*_soa(P), rgb, inten, split_level=16)
    d = tmp_path_factory.mktemp("corners16")
    cloud.write_dir(str(d))
    yield dict(_scene(cloud), P=P, rgb=rgb, inten=inten, dir=str(d))
    cloud.free()


@pytest.fixture(scope="module")
def world(ctx, fx, tmp_path_factory):
    """The globe with every corner and edge patch and the heavy cell, at level 5 (about 6000 cells), and its directory."""
    P = np.concatenate([fx["globe"], fx["corners"], fx["edges"], fx["heavy"]])
    rgb, inten = E.attributes(len(P), 7)
    cloud = ctx.build_s2_cloud(*_soa(P), rgb, inten, split_level=5)
    d = tmp_path_factory.mktemp("world5")
    cloud.write_dir(str(d))
    s = _scene(cloud)
    s.update(P=P, rgb=rgb, inten=inten, dir=str(d), leaves=S.oracle_cell_ids(s["allp"]["xyz"], 30), leaves_in=S.oracle_cell_ids(P, 30))
    yield s
    cloud.free()


def test_corner_locations(ctx, corner_cloud):
    import point_cloud_viewer_b200 as pcv

    s = corner_cloud
    G = pcv.geometry
    locs = dict(_corner_locations(G), all=G.all_points(), miss=G.aabb((0.0, 0.0, 0.0), (10.0, 10.0, 10.0)))
    hi, _ = _smallest_budget(pcv, ctx, s["dir"])
    want = _check_locations(s, locs, s["dir"], ctx, [0, hi + (1 << 20)])
    faces = s["cloud"].cell_ids >> np.uint64(61)
    for k in range(8):  # every corner location reaches cells of the three faces of its corner
        for kind in ("aabb", "obb", "frustum"):
            sel, slots = want["%s%d" % (kind, k)]
            assert len(slots) > 0 and len(np.unique(faces[sel])) == 3, (kind, k)
    mn, mx = s["boxes"]
    assert ((mn < 0) & (mx > mn)).any(axis=0).all()  # boxes with negative bounds on every axis


def test_globe_locations(ctx, world):
    import point_cloud_viewer_b200 as pcv

    s = world
    G = pcv.geometry
    locs = _globe_locations(G)
    hi, _ = _smallest_budget(pcv, ctx, s["dir"])
    want = _check_locations(s, locs, s["dir"], ctx, [0, 2 * hi])
    mn, mx = s["boxes"]
    for name in ("slab_xy", "slab_yz", "octant", "pole_box", "obb_centre", "frustum_origin", "heavy_box"):
        sel, slots = want[name]
        assert len(slots) > 0, name
    for name in ("slab_xy", "slab_yz", "obb_centre"):  # selected cells on both sides of two zero planes
        sel, _ = want[name]
        c = 0.5 * (mn[sel] + mx[sel])
        assert ((c < 0).any(0) & (c > 0).any(0)).sum() >= 2, name
    assert len(want["miss"][1]) == 0
    sel, slots = want["heavy_box"]  # the heavy cell: several query tiles, all its points inside
    heavy = int(S.oracle_cell_ids(E.HEAVY_POINT[None, :] * (E.R / np.linalg.norm(E.HEAVY_POINT)), 5)[0])
    assert len(slots) >= 10_000 and heavy in [int(v) for v in s["cloud"].cell_ids[sel]]


# ---- cell unions -----------------------------------------------------------------------------------------------------------
def _face_cell(f):
    return (f << 61) | (1 << 60)


def _sample_union(rng, leaves, k, lo=6):
    """k normalised ids: the cells (at levels lo..30) of random points, normalised, then k of them (a subset stays normalised)."""
    pick = rng.choice(len(leaves), min(len(leaves), 3 * k + 1000), replace=False)
    lsb = np.uint64(1) << (2 * (30 - rng.integers(lo, 31, len(pick)))).astype(np.uint64)
    pool = S.normalize((leaves[pick] & ~(lsb - np.uint64(1))) | lsb)
    assert len(pool) >= k
    return np.sort(pool[np.sort(rng.choice(len(pool), k, replace=False))])


@pytest.fixture(scope="module")
def unions(world, fx):
    s = world
    rng = np.random.default_rng(23)
    leaves = s["leaves_in"]
    ng, nc = len(fx["globe"]), len(fx["corners"])
    corner0 = leaves[ng:ng + 40_000]  # the (1, 1, 1) patch: faces 0, 1 and 2
    on1 = corner0[(corner0 >> np.uint64(61)) == 1]
    edge_leaves = leaves[ng + nc: ng + nc + len(fx["edges"])]
    u = {
        "faces": np.array([_face_cell(f) for f in range(6)], np.uint64),
        "face4": np.array([_face_cell(4)], np.uint64),
        "face0_and_leaves_of_face1": np.concatenate([np.array([_face_cell(0)], np.uint64), on1[rng.choice(len(on1), 300, replace=False)]]),
        "edge_leaves": edge_leaves[rng.choice(len(edge_leaves), 600, replace=False)],
    }
    for k in (255, 256, 257, 4096, 100_000):
        u["n%d" % k] = _sample_union(rng, leaves, k, 6 if k < 100_000 else 12)
        assert len(S.normalize(u["n%d" % k])) == k
    raw = u["n4096"][rng.choice(4096, 700, replace=False)]
    nested = [X.parent(raw[j:j + 1], 12)[0] for j in range(5)]
    f, i, j = S.face_ij(int(raw[9]))
    kids = [X.parent(np.array([S.orc().orc_s2_from_face_ij(f, (i & ~((1 << 11) - 1)) + di, (j & ~((1 << 11) - 1)) + dj)], np.uint64), 20)[0]
            for di in (0, 1 << 10) for dj in (0, 1 << 10)]
    u["raw"] = rng.permutation(np.concatenate([raw, raw[:50], nested, kids]).astype(np.uint64))
    assert len(u["raw"]) > CELLS_SHARED and len(S.normalize(u["raw"])) < len(u["raw"])
    return u


def _union_want(s, u):
    un = S.normalize(u)
    inside = S.union_test(un, s["leaves"])[0]
    cells = s["cloud"].cell_ids[S.union_test(un, s["cloud"].cell_ids)[1]]
    return un, inside, cells


def test_cell_unions(ctx, world, unions):
    import point_cloud_viewer_b200 as pcv

    s = world
    G, cloud = pcv.geometry, s["cloud"]
    cc = cloud.cell_counts.astype(np.int64)
    counts_want, tested_want = [], []
    for name, u in unions.items():
        un, inside, cells = _union_want(s, u)
        slots = np.nonzero(inside)[0]
        assert len(slots) > 0, name
        assert np.array_equal(cloud.cells_in_union(u), cells), name
        tested = int(cc[np.searchsorted(cloud.cell_ids, cells)].sum())
        q = cloud.query_union(u)
        assert q["total"] == len(slots) and q["tested"] == tested and np.array_equal(q["src"], s["allp"]["src"][slots]), name
        assert np.array_equal(q["xyz"].view(np.uint64), s["allp"]["xyz"][slots].view(np.uint64)), name
        _assert_stream_is(s, _cat(cloud.query_points(G.cell_union(u), batch_size=300_007)), slots)
        assert np.array_equal(cloud.cells_in_location(G.cell_union(u)), cells), name
        assert np.array_equal(ctx.s2_union_contains(*_soa(s["P"]), u), S.union_test(un, s["leaves_in"])[0]), name
        counts_want.append(len(slots))
        tested_want.append(tested)
        if name == "faces":
            assert len(slots) == len(s["P"])
    assert len(unions["n100000"]) > 100 * CELLS_SHARED
    batch = [G.cell_union(u) for u in unions.values()]  # small and large unions in one batch
    counts, tested = cloud.query_batch_device(batch)
    assert [int(v) for v in counts] == counts_want and [int(v) for v in tested] == tested_want
    counts, tested = cloud.query_batch_device(batch[::-1])
    assert [int(v) for v in counts] == counts_want[::-1] and [int(v) for v in tested] == tested_want[::-1]


def test_cell_unions_directory(ctx, world, unions):
    import point_cloud_viewer_b200 as pcv

    s = world
    G = pcv.geometry
    hi, _ = _smallest_budget(pcv, ctx, s["dir"])
    want = {name: _union_want(s, u) for name, u in unions.items()}
    for budget in (0, hi + (4 << 20)):  # a small budget that still holds the batch's union tables (2.4 MB)
        h = pcv.S2Dir(ctx, s["dir"], budget)
        try:
            for name, u in unions.items():
                _, inside, cells = want[name]
                slots = np.nonzero(inside)[0]
                assert np.array_equal(h.cells_in_union(u), cells), (name, budget)
                got = _cat(h.query_points(G.cell_union(u), batch_size=250_000))
                assert np.array_equal(got["src"].astype(np.int64), slots), (name, budget)
                assert np.array_equal(got["xyz"].view(np.uint64), s["allp"]["xyz"][slots].view(np.uint64))
                assert np.array_equal(got["rgb"], s["allp"]["rgb"][slots]) and np.array_equal(got["intensity"], s["allp"]["intensity"][slots])
            counts, tested = h.query_batch([G.cell_union(u) for u in unions.values()])
            c2, t2 = s["cloud"].query_batch_device([G.cell_union(u) for u in unions.values()])
            assert [int(v) for v in counts] == [int(w[1].sum()) for w in want.values()]
            assert np.array_equal(counts, c2) and np.array_equal(tested, t2)
        finally:
            h.close()


def test_octree_large_unions(fx, tmp_path):
    """The same sizes of union over an octree of the eight corner patches, resident and as a directory."""
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    P = fx["corners"]
    rgb, inten = E.attributes(len(P), 9)
    c = pcv.Context(0)
    try:
        tree = c.build_octree(*_soa(P), rgb, 0.001, P.min(0), P.max(0), intensity=inten)
        s = dict(pcv=pcv, tree=tree, **_tree_info(pcv, tree))  # leaves of the decoded positions
        rng = np.random.default_rng(29)
        cus = {k: _sample_union(rng, s["leaves"], k, 22) for k in (257, 4096, 20_000)}  # coarser cells hold whole patches
        # un-normalised: shuffled, with duplicates and cells that contain others
        cus["raw"] = rng.permutation(np.concatenate([cus[4096][:400], cus[257][:40], X.parent(cus[257][:3], 14)]).astype(np.uint64))
        assert len(cus["raw"]) > CELLS_SHARED
        masks = {}
        for name, cu in cus.items():
            masks[name] = _want(s, cu)
            assert masks[name].sum() > 0, name
            _assert_stream_equal(_octree_cat(_stream(s, cu, 100_000)), s["all"], masks[name])
        counts, tested = tree.query_batch_device([G.cell_union(cu) for cu in cus.values()])
        assert [int(v) for v in counts] == [int(m.sum()) for m in masks.values()]
        d = str(tmp_path / "oct")
        tree.write_dir(d)
        lo, _ = _octree_dir_smallest_budget(c, d)
        for budget in (0, lo + (6 << 20)):
            h = pcv.OctreeDir(c, d, budget)
            try:
                for name, cu in cus.items():
                    got = _octree_cat(h.query_points(G.cell_union(cu), batch_size=50_000))
                    want = _octree_cat(_stream(s, cu, 50_000))
                    assert np.array_equal(got["xyz"].view(np.uint64), want["xyz"].view(np.uint64)), (name, budget)
                    assert np.array_equal(got["rgb"], want["rgb"]) and np.array_equal(got["intensity"], want["intensity"])
                c2, t2 = h.query_batch([G.cell_union(cu) for cu in cus.values()])
                assert np.array_equal(c2, counts) and np.array_equal(t2, tested)
            finally:
                h.close()
        tree.free()
    finally:
        c.close()


# ---- X-ray -----------------------------------------------------------------------------------------------------------------
def test_xray_corner_patch(ctx, fx, tmp_path):
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    P = fx["corners"][:40_000]  # the (1, 1, 1) patch
    rgb, inten = E.attributes(len(P), 11)
    cloud = ctx.build_s2_cloud(*_soa(P), rgb, inten, split_level=16)
    try:
        assert len(np.unique(cloud.cell_ids >> np.uint64(61))) == 3
        box = np.concatenate([cloud.bbox_min, cloud.bbox_max])
        ext = cloud.bbox_max - cloud.bbox_min
        T = 64
        px = float(max(ext[0], ext[1])) / (T * 32)
        c = E.R * E.corner_directions()[0]
        qfg = list(G.Isometry(c, G.quat_mul(_rot([0, 0, 1], 0.785), _rot([1, -1, 0], 0.955))).inverse().as7())
        cloud.write_dir(str(tmp_path))
        for kw in (dict(), dict(query_from_global=qfg)):
            want = points_quadtree(P, rgb, inten, box, T, px, **kw)
            assert want is not None and len(want[1]) > 20
            info, tiles = cloud.xray_quadtree(T, px, **kw)
            _same(info, tiles, want)
            info, tiles = ctx.xray_quadtree_from_s2_dirs(str(tmp_path), T, px, **kw)
            _same(info, tiles, want)
    finally:
        cloud.free()


def test_level30_batches(ctx, fx, corner_cloud, tmp_path):
    """64 frusta over the corners at level 30: more cells than one selection chunk holds pairs, so one location per chunk."""
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    P = fx["corners"]
    cloud = ctx.build_s2_cloud(*_soa(P), None, None, split_level=30)
    try:
        assert cloud.num_cells > SELECT_PAIRS
        F = []
        for k, d in enumerate(E.corner_directions()):
            c = E.R * d
            F += _frusta(G, c - 250.0, c + 250.0, 8, 120.0, seed=100 + k)
        counts, tested = cloud.query_batch_device(F)
        brute = [int(O.location_contains(_oloc(f), P).sum()) for f in F]
        assert [int(v) for v in counts] == brute and sum(brute) > 0
        assert sum(1 for b in brute if b > 0) >= 32
        c16, _ = corner_cloud["cloud"].query_batch_device(F)
        assert np.array_equal(c16, counts)
        cc = cloud.cell_counts.astype(np.int64)
        for k in range(0, 64, 9):
            sel = np.searchsorted(cloud.cell_ids, cloud.cells_in_location(F[k]))
            assert int(tested[k]) == int(cc[sel].sum()), k
            batches = cloud.query_points(F[k])
            assert sum(len(b["src"]) for b in batches) == brute[k] and all(b["rgb"] is None for b in batches)
        cloud.write_dir(str(tmp_path))
    finally:
        cloud.free()
    h = ctx.open_s2_dir(str(tmp_path))
    try:
        assert h.num_cells > SELECT_PAIRS and not h.has_color and not h.has_intensity
        c2, t2 = h.query_batch(F)
        assert np.array_equal(c2, counts) and np.array_equal(t2, tested)
    finally:
        h.close()
