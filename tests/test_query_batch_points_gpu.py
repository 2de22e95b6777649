"""Batched point queries that return their points (pcv_query_batch_points_device, pcv_query_cell_unions_batch_points_device and the
pcv_s2_* forms; Octree / S2Cloud.query_batch_points): for every location, segment [off[i], off[i+1]) of the device arrays is exactly
what query_points streams for it, in order and bit for bit in every field, whatever the other locations of the batch.

On seeded slabs (octree with and without intensity, S2 cloud with and without colour and intensity):
- every location kind and cell unions with In and Cross nodes, with and without filter intervals (including their edges); the
  offsets against query_batch_device's counts; a few locations against the oracle's query;
- empty locations, duplicate and permuted location lists, no locations;
- a batch over more than one slab of tiles (the scan spanning many blocks, a node cut by a slab boundary) and an S2 batch over
  several selection chunks;
- the size query, a capacity one short, NULL fields, the argument contract, the statistics and the torch views."""
import gc

import numpy as np
import pytest

import oracle_api as O

pytestmark = pytest.mark.gpu

SEED, N = 80293751232, 300_000
SLAB_TILES = 1 << 18  # kQbpSlabTiles (csrc/query_batch_points_plan.h)
QUERY_TILE = 2048     # kQueryTile (csrc/query.cuh)
SELECT_PAIRS = 1 << 18  # kS2SelectPairs (csrc/s2_api.inl)
FILTERS = {
    "none": (),
    "band": ((100.0, 250.0),),
    "edges": ((0.0, 0.0),),            # exactly the points of intensity 0
    "top_edge": ((999.0, 999.0),),
    "two": ((100.0, 500.0), (250.0, 900.0)),  # both intervals: [250, 500]
}


def _copy_loc(loc):
    o = O.Location()
    for f, _ in O.Location._fields_:
        setattr(o, f, getattr(loc, f))
    return o


def _parent(cid, level):
    lsb = 1 << (2 * (30 - level))
    return (int(cid) & ~(2 * lsb - 1)) | lsb


@pytest.fixture(scope="module")
def scene():
    import point_cloud_viewer_b200 as pcv

    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED, 0, N)
    inten = (np.arange(N) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    bmin, bmax = np.asarray(bmin, np.float64), np.asarray(bmax, np.float64)
    ctx = pcv.Context(0, max_points_per_node=5000)  # nodes of up to 3 tiles
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    tree_noi = ctx.build_octree(x, y, z, rgb, res, bmin, bmax)
    cloud = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=20)
    cloud_bare = ctx.build_s2_cloud(x, y, z, None, None, split_level=20)
    ref = O.build(x, y, z, rgb.reshape(-1, 3), res, bmin, bmax, intensity=inten, max_points_per_node=5000)
    G = pcv.geometry
    d = bmax - bmin
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    ecef_from_local = G.Isometry((4157222.543, 664789.307, 4774952.099), q)
    mid = np.array([x[N // 2], y[N // 2], z[N // 2]])
    c = np.asarray(G.web_mercator_coord(mid, 19))
    locs = {
        "all": G.all_points(),
        "aabb": G.aabb(bmin + 0.2 * d, bmin + 0.8 * d),
        "aabb_small": G.aabb(bmin + 0.45 * d, bmin + 0.5 * d),
        "obb": G.obb(ecef_from_local, (50.0, 50.0, 5.0)),
        "frustum": G.frustum(ecef_from_local, G.Perspective.new_fov(1.0, 1.2, 0.1, 10.0)),
        "frustum_far": G.frustum(ecef_from_local * G.Isometry((0, 0, 0), G.quat_from_axis_angle([1, 0.3, 0], 1.3)), G.Perspective.new_fov(1.3, 0.9, 0.5, 150.0)),
        "obb_tilted": G.obb(ecef_from_local * G.Isometry((10, -20, 1), G.quat_from_axis_angle([0.2, 0.5, -0.7], 0.523)), (30.0, 12.0, 4.0)),
        "miss": G.aabb(bmax + 1000.0, bmax + 1100.0),
        "mercator": G.web_mercator_rect(c - 150.0, c + 150.0, 19),
    }
    ids = cloud.cell_ids
    unions = {
        "whole": G.cell_union(sorted({_parent(i, 8) for i in ids})),  # holds the root: every node In
        "some": G.cell_union(sorted({_parent(i, 14) for i in ids[:: max(1, len(ids) // 7)]})),  # In and Cross nodes
        "fine": G.cell_union([int(i) for i in ids[len(ids) // 3: len(ids) // 3 + 40]]),
        "empty": G.cell_union([]),
    }
    yield dict(pcv=pcv, G=G, ctx=ctx, tree=tree, tree_noi=tree_noi, cloud=cloud, cloud_bare=cloud_bare, ref=ref, locs=locs, unions=unions,
               bmin=bmin, bmax=bmax)
    for h in (tree, tree_noi, cloud, cloud_bare):
        h.free()
    ctx.close()


def _stream(h, loc, filters=()):
    """query_points(loc) concatenated: dict of numpy arrays (rgb / intensity None when the source has none)."""
    bs = h.query_points(loc, filters=[v for iv in filters for v in iv], batch_size=1 << 22)
    if not bs:
        return None
    out = {k: np.concatenate([b[k] for b in bs]) for k in ("xyz", "src")}
    for k in ("rgb", "intensity"):
        out[k] = None if bs[0][k] is None else np.concatenate([b[k] for b in bs])
    return out


def _host(t):
    return {k: v.cpu().numpy() for k, v in t.items()}


def _assert_segment(got, off, i, want, where):
    a, b = int(off[i]), int(off[i + 1])
    n = 0 if want is None else len(want["src"])
    assert b - a == n, where
    for k, v in got.items():
        seg = v[a:b]
        if n == 0:
            assert len(seg) == 0, (where, k)
        elif k == "xyz":
            assert np.array_equal(seg.view(np.uint64), want["xyz"].view(np.uint64)), where
        elif k == "src":
            assert seg.dtype == np.int64 and np.array_equal(seg.astype(np.uint64), want["src"]), where
        else:
            assert np.array_equal(seg, want[k]), (where, k)


def _check_batch(h, locs, filters=(), fields=None, streams=None):
    """The whole contract over one batch; returns (offsets, host arrays)."""
    f = [v for iv in filters for v in iv]
    off, t = h.query_batch_points(locs, filters=f, fields=fields)
    qs = h.last_query_stats()
    counts, tested = h.query_batch_device(locs, filters=f)
    assert off.dtype == np.uint64 and len(off) == len(locs) + 1 and off[0] == 0
    assert np.array_equal(np.diff(off.astype(np.int64)), counts.astype(np.int64))
    assert qs["returned_points"] == qs["stored_points"] == int(off[-1])
    assert qs["tested_points"] == int(tested.sum())
    got = _host(t)
    for i, loc in enumerate(locs):
        want = streams[i] if streams is not None else _stream(h, loc, filters)
        _assert_segment(got, off, i, want, i)
    return off, got


@pytest.mark.parametrize("fname", sorted(FILTERS))
def test_octree_every_location_kind(scene, fname):
    filters = FILTERS[fname]
    _check_batch(scene["tree"], list(scene["locs"].values()), filters)


@pytest.mark.parametrize("fname", ["none", "band", "edges"])
def test_octree_cell_unions(scene, fname):
    _check_batch(scene["tree"], list(scene["unions"].values()), FILTERS[fname])


def test_octree_without_intensity(scene):
    _check_batch(scene["tree_noi"], list(scene["locs"].values()) + [scene["locs"]["all"]])
    _check_batch(scene["tree_noi"], list(scene["unions"].values()))


@pytest.mark.parametrize("fname", ["none", "band", "two"])
def test_s2_every_location_kind(scene, fname):
    _check_batch(scene["cloud"], list(scene["locs"].values()), FILTERS[fname])
    _check_batch(scene["cloud"], list(scene["unions"].values()), FILTERS[fname])


def test_s2_without_colour_or_intensity(scene):
    h = scene["cloud_bare"]
    off, got = _check_batch(h, list(scene["locs"].values()))
    assert set(got) == {"xyz", "src"}
    _check_batch(h, list(scene["unions"].values()))


def test_against_the_oracle(scene):
    locs = [scene["locs"][k] for k in ("aabb", "obb_tilted", "frustum_far")]
    for filters in ((), (100.0, 250.0)):
        off, t = scene["tree"].query_batch_points(locs, filters=filters)
        got = _host(t)
        for i, loc in enumerate(locs):
            want = scene["ref"].query(_copy_loc(loc), filters=filters, with_intensity=True)
            a, b = int(off[i]), int(off[i + 1])
            assert b - a == len(want["src"]) > 0
            assert np.array_equal(got["src"][a:b].astype(np.uint64), want["src"])
            assert np.array_equal(got["xyz"][a:b].view(np.uint64), want["xyz"].view(np.uint64))
            assert np.array_equal(got["rgb"][a:b], want["rgb"])
            assert np.array_equal(got["intensity"][a:b], want["intensity"])


@pytest.mark.parametrize("source", ["tree", "cloud"])
def test_duplicates_permutations_and_no_locations(scene, source):
    h, L = scene[source], scene["locs"]
    names = ["obb", "miss", "aabb_small", "obb", "frustum", "miss", "aabb_small"]
    streams = {k: _stream(h, L[k], FILTERS["band"]) for k in set(names)}
    off, got = _check_batch(h, [L[k] for k in names], FILTERS["band"], streams=[streams[k] for k in names])
    seg = lambda o, g, i: {k: v[int(o[i]): int(o[i + 1])] for k, v in g.items()}
    for k in ("xyz", "src", "rgb", "intensity"):
        assert np.array_equal(seg(off, got, 0)[k], seg(off, got, 3)[k])
    perm = [4, 2, 0, 6, 1, 5, 3]
    off2, got2 = _check_batch(h, [L[names[p]] for p in perm], FILTERS["band"], streams=[streams[names[p]] for p in perm])
    for j, p in enumerate(perm):
        for k in got:
            assert np.array_equal(seg(off2, got2, j)[k], seg(off, got, p)[k])
    off0, t0 = h.query_batch_points([])
    assert list(off0) == [0] and all(v.shape[0] == 0 for v in t0.values())


def test_many_slabs_and_a_node_cut_by_a_slab(scene):
    """AllPoints repeated until the work list spans more than one slab; a prefix of small boxes moves the first slab boundary
    into a node of several tiles.  A filter keeps the output small."""
    tree, G = scene["tree"], scene["G"]
    nodes = tree.nodes
    tiles_of = lambda names: [-(-nodes[nm]["num_points"] // QUERY_TILE) for nm in names if nodes[nm]["num_points"] > 0]
    all_tiles = tiles_of(tree.order)
    per_all = sum(all_tiles)
    assert max(all_tiles) > 1
    d = scene["bmax"] - scene["bmin"]
    small = G.aabb(scene["bmin"] + 0.45 * d, scene["bmin"] + 0.46 * d)
    small_tiles = sum(tiles_of(tree.nodes_in_location(small)))
    starts = np.concatenate([[0], np.cumsum(all_tiles)])
    for m in range(0, 64):
        r = (SLAB_TILES - m * small_tiles) % per_all
        k = int(np.searchsorted(starts, r, side="right")) - 1
        if starts[k] < r < starts[k + 1]:  # the boundary falls inside node k's tiles
            break
    else:
        pytest.fail("no prefix puts the slab boundary inside a node")
    nall = -(-(2 * SLAB_TILES - m * small_tiles) // per_all) + 1  # past two slab boundaries
    locs = [small] * m + [G.all_points()] * nall
    filters = ((7.0, 7.0),)
    want_all, want_small = _stream(tree, G.all_points(), filters), _stream(tree, small, filters)
    assert m * small_tiles + nall * per_all > 2 * SLAB_TILES
    _check_batch(tree, locs, filters, streams=[want_small] * m + [want_all] * nall)


def test_s2_batch_over_several_selection_chunks(scene):
    h, G = scene["cloud"], scene["G"]
    chunk = max(1, min(SELECT_PAIRS // h.num_cells, 65535))
    rng = np.random.default_rng(3)
    bmin, bmax = scene["bmin"], scene["bmax"]
    boxes = []
    for _ in range(9):
        lo = bmin + rng.random(3) * (bmax - bmin) * 0.9
        boxes.append(G.aabb(lo, lo + (bmax - bmin) * 0.08))
    streams = [_stream(h, b, FILTERS["band"]) for b in boxes]
    order = [k % len(boxes) for k in range(2 * chunk + 5)]  # three chunks, each box in every chunk at a different place
    assert len(order) > 2 * chunk
    _check_batch(h, [boxes[k] for k in order], FILTERS["band"], streams=[streams[k] for k in order])


def _raw(h, fn, locs, filters, off, xyz=None, rgb=None, inten=None, src=None, cap=0):
    from point_cloud_viewer_b200 import _native as N

    arr = (N.Location * len(locs))(*locs)
    f = np.asarray(filters, np.float64).reshape(-1)
    p = lambda t: None if t is None else t.data_ptr()
    return fn(h.h, arr, len(locs), f.ctypes.data if len(f) else None, len(f) // 2, off.ctypes.data, p(xyz), p(rgb), p(inten), p(src), cap)


@pytest.mark.parametrize("source", ["tree", "cloud"])
def test_size_query_capacity_and_null_fields(scene, source):
    import torch
    from point_cloud_viewer_b200 import _native as N

    h = scene[source]
    fn = N.lib().pcv_query_batch_points_device if source == "tree" else N.lib().pcv_s2_query_batch_points_device
    locs = [scene["locs"][k] for k in ("aabb_small", "obb", "miss", "frustum_far")]
    off = np.zeros(len(locs) + 1, np.uint64)
    assert _raw(h, fn, locs, (), off) == 0
    total = int(off[-1])
    assert total > 0
    counts, _ = h.query_batch_device(locs)
    assert np.array_equal(np.diff(off.astype(np.int64)), counts.astype(np.int64))
    full_off, full = h.query_batch_points(locs)
    full = _host(full)
    assert np.array_equal(full_off, off)
    dev = torch.device("cuda", scene["ctx"].device)
    xyz = torch.full((total, 3), -1.0, dtype=torch.float64, device=dev)
    # the size query (no positions) writes nothing, not even the fields it is given
    sentinel = torch.full((total,), -7, dtype=torch.int64, device=dev)
    o2 = np.zeros_like(off)
    assert _raw(h, fn, locs, (), o2, None, None, None, sentinel, total) == 0 and np.array_equal(o2, off)
    assert bool((sentinel == -7).all())
    # one short: PCV_ERR_INVALID naming both numbers, offsets complete
    o3 = np.zeros_like(off)
    assert _raw(h, fn, locs, (), o3, xyz, None, None, None, total - 1) == -1
    msg = N.lib().pcv_last_error().decode()
    assert str(total) in msg and str(total - 1) in msg
    assert np.array_equal(o3, off)
    # position only, then position and provenance
    o4 = np.zeros_like(off)
    assert _raw(h, fn, locs, (), o4, xyz, None, None, None, total) == 0
    assert np.array_equal(xyz.cpu().numpy().view(np.uint64), full["xyz"].view(np.uint64))
    src = torch.zeros(total, dtype=torch.int64, device=dev)
    inten = torch.zeros(total, dtype=torch.float32, device=dev)
    xyz.fill_(0)
    assert _raw(h, fn, locs, (), o4, xyz, None, inten, src, total + 5) == 0
    assert np.array_equal(src.cpu().numpy(), full["src"]) and np.array_equal(inten.cpu().numpy(), full["intensity"])
    assert np.array_equal(xyz.cpu().numpy().view(np.uint64), full["xyz"].view(np.uint64))
    qs = h.last_query_stats()
    assert qs["stored_points"] == qs["returned_points"] == total
    # the Python layer with some of the fields
    o5, part = h.query_batch_points(locs, fields=("src",))
    assert set(part) == {"src"} and np.array_equal(part["src"].cpu().numpy(), full["src"])


def test_fields_the_cloud_lacks_are_invalid(scene):
    import torch
    from point_cloud_viewer_b200 import _native as N

    L = N.lib()
    locs = [scene["locs"]["aabb_small"]]
    dev = torch.device("cuda", scene["ctx"].device)
    buf = torch.zeros((1 << 20, 3), dtype=torch.float64, device=dev)
    f32 = torch.zeros(1 << 20, dtype=torch.float32, device=dev)
    u8 = torch.zeros((1 << 20, 3), dtype=torch.uint8, device=dev)
    off = np.zeros(2, np.uint64)
    assert _raw(scene["tree_noi"], L.pcv_query_batch_points_device, locs, (), off, buf, None, f32, None, 1 << 20) == -1
    assert _raw(scene["cloud_bare"], L.pcv_s2_query_batch_points_device, locs, (), off, buf, None, f32, None, 1 << 20) == -1
    assert _raw(scene["cloud_bare"], L.pcv_s2_query_batch_points_device, locs, (), off, buf, u8, None, None, 1 << 20) == -1
    assert _raw(scene["cloud_bare"], L.pcv_s2_query_batch_points_device, locs, (), off, buf, None, None, None, 1 << 20) == 0
    with pytest.raises(scene["pcv"].PcvError):
        scene["cloud_bare"].query_batch_points(locs, fields=("xyz", "rgb"))


@pytest.mark.parametrize("source", ["tree", "cloud"])
def test_argument_contract(scene, source):
    """As test_query_entry_contract_gpu.py: an unknown kind, a null filter array and filters without intensity are PCV_ERR_INVALID."""
    from point_cloud_viewer_b200 import _native as N

    L, G = N.lib(), scene["G"]
    fn = L.pcv_query_batch_points_device if source == "tree" else L.pcv_s2_query_batch_points_device
    fu = L.pcv_query_cell_unions_batch_points_device if source == "tree" else L.pcv_s2_query_cell_unions_batch_points_device
    h = scene[source]
    off = np.zeros(2, np.uint64)
    assert _raw(h, fn, [G.all_points()], (), off) == 0 and off[1] > 0
    bad = G.all_points()
    bad.kind = 7
    assert _raw(h, fn, [bad], (), off) == -1
    assert fn(h.h, (N.Location * 1)(G.all_points()), 1, None, 1, off.ctypes.data, None, None, None, None, 0) == -1
    cu = scene["unions"]["some"]
    assert fu(h.h, (N.CellUnion * 1)(cu.struct()), 1, None, 1, off.ctypes.data, None, None, None, None, 0) == -1
    assert fn(h.h, (N.Location * 1)(G.all_points()), 1, None, 0, None, None, None, None, None, 0) == -1
    noi = scene["tree_noi"] if source == "tree" else scene["cloud_bare"]
    f = np.array([0.0, 10.0])
    assert fn(noi.h, (N.Location * 1)(G.all_points()), 1, f.ctypes.data, 1, off.ctypes.data, None, None, None, None, 0) == -1
    assert fu(noi.h, (N.CellUnion * 1)(cu.struct()), 1, f.ctypes.data, 1, off.ctypes.data, None, None, None, None, 0) == -1


def test_torch_views(scene):
    import torch

    def run():
        return scene["tree"].query_batch_points([scene["locs"]["obb"], scene["locs"]["aabb_small"]])

    off, t = run()
    gc.collect()
    total = int(off[-1])
    dev = torch.device("cuda", scene["ctx"].device)
    want = {"xyz": (torch.float64, (total, 3)), "rgb": (torch.uint8, (total, 3)), "intensity": (torch.float32, (total,)), "src": (torch.int64, (total,))}
    assert set(t) == set(want)
    for k, (dt, shape) in want.items():
        assert t[k].device == dev and t[k].dtype == dt and tuple(t[k].shape) == shape, k
    # still valid after the call and a collection: the same values as a fresh call
    off2, t2 = run()
    for k in want:
        assert torch.equal(t[k], t2[k]), k
