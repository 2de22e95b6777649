"""Batched point queries that return their points straight from octree and S2 directories (pcv_octree_dir_query_batch_points_device,
pcv_s2_dir_query_batch_points_device and their cell-union forms; OctreeDir / S2Dir.query_batch_points): for every location,
segment [off[i], off[i+1]) of the device arrays is exactly what the handle's query_points streams for it, in order and bit for bit
in xyz, rgb, intensity and src (the slot); the offsets are query_batch's counts; xyz / rgb / intensity equal load_dir (load_s2_dir)
+ the resident query_batch_points; nothing depends on the budget or the chunking.

On seeded slabs written as an octree directory with and without intensity (and one with large nodes, for budgets that split
nodes across chunks) and an S2 directory with and without colour and intensity:
- every location kind and cell unions with In and Cross nodes, with and without filters and filter edges; a few locations
  against the oracle's load_dir query;
- the default budget (one chunk), a budget of several chunks with nodes split across them, a budget too small for the per-tile
  state (PCV_ERR_UNSUPPORTED, the handle still usable);
- the reads: the size query reads the visited nodes' positions (and intensities with filters) once, a one-chunk fill every
  needed file once, a several-chunk fill more than once and at most twice, one location repeated 50 times what it reads alone;
- empty and missed locations, duplicate and permuted lists, no locations, an S2 batch over several selection chunks;
- the size query with a sentinel array, a capacity one short (no writes, no reads beyond the count pass), NULL fields, fields
  the directory lacks, the argument contract, the torch views."""
import gc
import os

import numpy as np
import pytest

import oracle_api as O

pytestmark = pytest.mark.gpu

SEED, N = 80293751232, 300_000
FILTERS = {
    "none": (),
    "band": ((100.0, 250.0),),
    "edges": ((0.0, 0.0),),
    "top_edge": ((999.0, 999.0),),
    "two": ((100.0, 500.0), (250.0, 900.0)),
}
SMALL_BUDGET = 1 << 20
ROOT_N = 1_200_000  # points of the directory of few nodes of many tiles


def _copy_loc(loc):
    o = O.Location()
    for f, _ in O.Location._fields_:
        setattr(o, f, getattr(loc, f))
    return o


def _parent(cid, level):
    lsb = 1 << (2 * (30 - level))
    return (int(cid) & ~(2 * lsb - 1)) | lsb


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED, 0, N)
    inten = (np.arange(N) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    bmin, bmax = np.asarray(bmin, np.float64), np.asarray(bmax, np.float64)
    base = tmp_path_factory.mktemp("dir_batch_points")
    ctx = pcv.Context(0, max_points_per_node=5000)  # nodes of up to 3 tiles
    dirs = {k: str(base / k) for k in ("oct", "oct_noi", "oct_big", "oct_root", "s2", "s2_bare")}
    for k, kw in (("oct", dict(intensity=inten)), ("oct_noi", {})):
        t = ctx.build_octree(x, y, z, rgb, res, bmin, bmax, **kw)
        t.write_dir(dirs[k])
        t.free()
    big = pcv.Context(0, max_points_per_node=100_000)  # nodes larger than a chunk of SMALL_BUDGET
    t = big.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    t.write_dir(dirs["oct_big"])
    t.free()
    big.close()
    big = pcv.Context(0, max_points_per_node=4_000_000)  # few nodes of many tiles
    rx, ry, rz, rrgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED + 1, 0, ROOT_N)
    t = big.build_octree(rx, ry, rz, rrgb, res, bmin, bmax)
    t.write_dir(dirs["oct_root"])
    t.free()
    big.close()
    ctx.build_s2_dir(dirs["s2"], x, y, z, rgb, inten, split_level=20)
    ctx.build_s2_dir(dirs["s2_bare"], x, y, z, None, None, split_level=20)
    h = {k: (pcv.S2Dir if k.startswith("s2") else pcv.OctreeDir)(ctx, d) for k, d in dirs.items()}
    r = {k: (ctx.load_s2_dir(d) if k.startswith("s2") else ctx.load_dir(d)) for k, d in dirs.items()}
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
    ids = r["s2"].cell_ids
    unions = {
        "whole": G.cell_union(sorted({_parent(i, 8) for i in ids})),  # every node In
        "some": G.cell_union(sorted({_parent(i, 14) for i in ids[:: max(1, len(ids) // 7)]})),  # In and Cross nodes
        "fine": G.cell_union([int(i) for i in ids[len(ids) // 3: len(ids) // 3 + 40]]),
        "empty": G.cell_union([]),
    }
    yield dict(pcv=pcv, G=G, ctx=ctx, dirs=dirs, h=h, r=r, locs=locs, unions=unions, bmin=bmin, bmax=bmax)
    for v in h.values():
        v.close()
    for v in r.values():
        v.free()
    ctx.close()


def _stream(h, loc, filters=()):
    """The handle's query_points(loc) concatenated (rgb / intensity None when the directory has none), or None."""
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


def _check_batch(sc, key, locs, filters=(), fields=None, streams=None, h=None):
    """The whole contract over one batch on handle `key` (or h); returns (offsets, host arrays, stats)."""
    h = h or sc["h"][key]
    f = [v for iv in filters for v in iv]
    off, t = h.query_batch_points(locs, filters=f, fields=fields)
    st = h.last_stats()
    counts, tested = h.query_batch(locs, filters=f)
    assert off.dtype == np.uint64 and len(off) == len(locs) + 1 and off[0] == 0
    assert np.array_equal(np.diff(off.astype(np.int64)), counts.astype(np.int64))
    assert st["returned_points"] == int(off[-1]) and st["tested_points"] == int(tested.sum())
    assert 0 < st["peak_device_bytes"] <= st["max_device_bytes"]
    got = _host(t)
    for i, loc in enumerate(locs):
        want = streams[i] if streams is not None else _stream(h, loc, filters)
        _assert_segment(got, off, i, want, i)
    roff, rt = sc["r"][key].query_batch_points(locs, filters=f, fields=[k for k in got if k != "src"] or ["xyz"])
    assert np.array_equal(roff, off)
    rgot = _host(rt)
    for k in got:
        if k == "xyz":
            assert np.array_equal(got[k].view(np.uint64), rgot[k].view(np.uint64))
        elif k != "src":
            assert np.array_equal(got[k], rgot[k]), k
    return off, got, st


def _files(d, names, exts):
    tot = 0
    for nm in names:
        for e in exts:
            p = os.path.join(d, nm + e)
            if os.path.exists(p):
                tot += os.path.getsize(p)
    return tot


def _visited(h, locs):
    return sorted({nm for loc in locs for nm in h.nodes_in_location(loc)})


def _raw(h, fn, locs, filters, off, xyz=None, rgb=None, inten=None, src=None, cap=0):
    from point_cloud_viewer_b200 import _native as N

    arr = (N.Location * len(locs))(*locs)
    f = np.asarray(filters, np.float64).reshape(-1)
    p = lambda t: None if t is None else t.data_ptr()
    return fn(h.h, arr, len(locs), f.ctypes.data if len(f) else None, len(f) // 2, off.ctypes.data, p(xyz), p(rgb), p(inten), p(src), cap)


def _fn(key):
    from point_cloud_viewer_b200 import _native as N

    return N.lib().pcv_s2_dir_query_batch_points_device if key.startswith("s2") else N.lib().pcv_octree_dir_query_batch_points_device


# ---- equality ----


@pytest.mark.parametrize("fname", sorted(FILTERS))
def test_octree_dir_every_location_kind(scene, fname):
    _check_batch(scene, "oct", list(scene["locs"].values()), FILTERS[fname])


@pytest.mark.parametrize("fname", ["none", "band", "edges"])
def test_octree_dir_cell_unions(scene, fname):
    _check_batch(scene, "oct", list(scene["unions"].values()), FILTERS[fname])


def test_octree_dir_without_intensity(scene):
    off, got, _ = _check_batch(scene, "oct_noi", list(scene["locs"].values()) + [scene["locs"]["all"]])
    assert set(got) == {"xyz", "rgb", "src"}
    _check_batch(scene, "oct_noi", list(scene["unions"].values()))


@pytest.mark.parametrize("fname", ["none", "band", "two"])
def test_s2_dir_every_location_kind(scene, fname):
    _check_batch(scene, "s2", list(scene["locs"].values()), FILTERS[fname])
    _check_batch(scene, "s2", list(scene["unions"].values()), FILTERS[fname])


def test_s2_dir_without_colour_or_intensity(scene):
    off, got, _ = _check_batch(scene, "s2_bare", list(scene["locs"].values()))
    assert set(got) == {"xyz", "src"}
    _check_batch(scene, "s2_bare", list(scene["unions"].values()))


def test_against_the_oracle(scene):
    ref = O.load_dir(scene["dirs"]["oct"])
    locs = [scene["locs"][k] for k in ("aabb", "obb_tilted", "frustum_far")]
    for filters in ((), (100.0, 250.0)):
        off, t = scene["h"]["oct"].query_batch_points(locs, filters=filters)
        got = _host(t)
        for i, loc in enumerate(locs):
            want = ref.query(_copy_loc(loc), filters=filters, with_intensity=True)
            a, b = int(off[i]), int(off[i + 1])
            assert b - a == len(want["xyz"]) > 0
            assert np.array_equal(got["xyz"][a:b].view(np.uint64), want["xyz"].view(np.uint64))
            assert np.array_equal(got["rgb"][a:b], want["rgb"])
            assert np.array_equal(got["intensity"][a:b], want["intensity"])


# ---- budgets ----


def _big_batch(sc):
    L = sc["locs"]
    return [L["aabb"], L["all"], L["obb_tilted"], L["frustum_far"], L["all"], L["aabb_small"]]


def test_several_chunks_equal_one_chunk(scene):
    """A budget whose chunks are smaller than the largest nodes: nodes split across chunks, every location's node run crossing
    chunk boundaries; the output is the default budget's (one chunk), bit for bit."""
    pcv, key = scene["pcv"], "oct_big"
    meta = scene["h"][key].meta
    bpc = np.array([{1: 1, 2: 2, 3: 4}.get(int(e), 8) for e in meta["enc"]])
    assert int((meta["num_points"] * (3 * bpc + 7)).max()) > SMALL_BUDGET  # the largest node cannot be one piece
    locs = _big_batch(scene)
    for filters in ((), FILTERS["band"]):
        off1, got1, st1 = _check_batch(scene, key, locs, filters)
        small = pcv.OctreeDir(scene["ctx"], scene["dirs"][key], SMALL_BUDGET)
        try:
            off2, got2, st2 = _check_batch(scene, key, locs, filters, h=small)
        finally:
            small.close()
        assert st1["chunks"] == 2 and st2["chunks"] > 4
        assert st2["peak_device_bytes"] <= st2["max_device_bytes"] == SMALL_BUDGET
        assert np.array_equal(off1, off2)
        for k in got1:
            assert np.array_equal(got1[k], got2[k]), k
        # reads: the one-chunk fill reads every file of every visited node once; several chunks more than once, at most twice
        names = _visited(scene["h"][key], locs)
        every = _files(scene["dirs"][key], names, (".xyz", ".rgb", ".intensity"))
        assert st1["bytes_read"] == every
        assert every < st2["bytes_read"] <= 2 * every


def test_budget_too_small_for_the_tile_state(scene):
    """At the smallest budget under which query_batch counts 200 AllPoints over a directory of few large nodes, the points call
    cannot hold its 4 bytes per work tile: PCV_ERR_UNSUPPORTED, and the handle still answers."""
    pcv, key = scene["pcv"], "oct_root"
    d = scene["dirs"][key]
    meta = scene["h"][key].meta
    n = meta["num_points"][meta["num_points"] > 0]
    tiles = int(((n + 2047) // 2048).sum())
    widest = int(np.bincount(meta["level"]).max())
    # per location: the tile counts against the frontier's room (LocProj 416 B + 8, 24 B per pair of the widest level)
    assert 4 * tiles > 424 + 24 * widest + 64
    many = [scene["locs"]["all"]] * 200

    def counts_fit(b):
        try:
            h = pcv.OctreeDir(scene["ctx"], d, b)
        except pcv.PcvError as e:
            assert e.code == -6
            return False
        try:
            h.query_batch(many)
            return True
        except pcv.PcvError as e:
            assert e.code == -6
            return False
        finally:
            h.close()

    lo, hi = 1 << 16, 256 << 20
    assert counts_fit(hi)
    while hi - lo > 1024:
        mid = (lo + hi) // 2
        if counts_fit(mid):
            hi = mid
        else:
            lo = mid
    h = pcv.OctreeDir(scene["ctx"], d, hi)
    try:
        with pytest.raises(pcv.PcvError) as e:
            h.query_batch_points(many)
        assert e.value.code == -6 and "split the batch" in str(e.value) and "work tiles" in str(e.value)
        counts, _ = h.query_batch(many)  # still usable
        assert int(counts[0]) == ROOT_N
        _check_batch(scene, key, [scene["locs"]["aabb_small"], scene["locs"]["obb"]], h=h)
    finally:
        h.close()


# ---- reads ----


@pytest.mark.parametrize("key", ["oct", "s2"])
def test_size_query_reads_positions_once(scene, key):
    h = scene["h"][key]
    locs = [scene["locs"][k] for k in ("aabb", "obb", "frustum_far")]
    if key == "s2":
        h.query_batch(locs)  # the point boxes are scanned by the first polyhedral call: not part of what this test counts
    for filters in ((), (100.0, 250.0)):
        off = np.zeros(len(locs) + 1, np.uint64)
        assert _raw(h, _fn(key), locs, filters, off) == 0
        st = h.last_stats()
        exts = (".xyz", ".intensity") if filters else (".xyz",)
        if key == "oct":
            names = _visited(h, locs)
        else:
            import point_cloud_viewer_b200 as pcv

            names = sorted({pcv.s2_token(c) for loc in locs for c in h.cells_in_location(loc)})
        assert st["bytes_read"] == _files(scene["dirs"][key], names, exts) > 0
        assert st["chunks"] == 1 and st["returned_points"] == int(off[-1])


def test_one_location_repeated_reads_what_it_reads_alone(scene):
    h = scene["h"]["oct"]
    loc = scene["locs"]["frustum_far"]
    off1, t1 = h.query_batch_points([loc])
    one = h.last_stats()["bytes_read"]
    off50, t50 = h.query_batch_points([loc] * 50)
    assert h.last_stats()["bytes_read"] == one > 0
    n = int(off1[-1])
    assert np.array_equal(np.diff(off50.astype(np.int64)), np.full(50, n))
    for k in t1:
        a, b = t1[k].cpu().numpy(), t50[k].cpu().numpy()
        for i in range(0, 50, 7):
            assert np.array_equal(b[i * n: (i + 1) * n], a), k


# ---- lists ----


@pytest.mark.parametrize("key", ["oct", "s2"])
def test_duplicates_permutations_and_no_locations(scene, key):
    h, L = scene["h"][key], scene["locs"]
    names = ["obb", "miss", "aabb_small", "obb", "frustum", "miss", "aabb_small"]
    streams = {k: _stream(h, L[k], FILTERS["band"]) for k in set(names)}
    off, got, _ = _check_batch(scene, key, [L[k] for k in names], FILTERS["band"], streams=[streams[k] for k in names])
    seg = lambda o, g, i: {k: v[int(o[i]): int(o[i + 1])] for k, v in g.items()}
    for k in got:
        assert np.array_equal(seg(off, got, 0)[k], seg(off, got, 3)[k])
    assert off[2] == off[1]  # the missed location
    perm = [4, 2, 0, 6, 1, 5, 3]
    off2, got2, _ = _check_batch(scene, key, [L[names[p]] for p in perm], FILTERS["band"], streams=[streams[names[p]] for p in perm])
    for j, p in enumerate(perm):
        for k in got:
            assert np.array_equal(seg(off2, got2, j)[k], seg(off, got, p)[k])
    off0, t0 = h.query_batch_points([])
    assert list(off0) == [0] and all(v.shape[0] == 0 for v in t0.values())
    offe, te = h.query_batch_points([scene["unions"]["empty"]])
    assert list(offe) == [0, 0]


def test_s2_batch_over_several_selection_chunks(scene):
    pcv, G = scene["pcv"], scene["G"]
    budget = 8 << 20
    h = pcv.S2Dir(scene["ctx"], scene["dirs"]["s2"], budget)
    try:
        # a selection takes 424 + 8 * cells bytes per location (s2_dir_select_bytes) from what the locations' tables (1112 bytes
        # each) leave: tables over 70 % of the budget leave selections of fewer than a third of the locations
        per_sel, per_table = 424 + 8 * h.num_cells, 1112
        n = int(0.7 * budget / per_table)
        assert n > 3 * (0.3 * budget / per_sel)
        rng = np.random.default_rng(3)
        bmin, bmax = scene["bmin"], scene["bmax"]
        boxes = []
        for _ in range(9):
            lo = bmin + rng.random(3) * (bmax - bmin) * 0.9
            boxes.append(G.aabb(lo, lo + (bmax - bmin) * 0.08))
        streams = [_stream(h, b, FILTERS["band"]) for b in boxes]
        order = [k % len(boxes) for k in range(n)]
        _check_batch(scene, "s2", [boxes[k] for k in order], FILTERS["band"], streams=[streams[k] for k in order], h=h)
    finally:
        h.close()


# ---- size query, capacity and fields ----


@pytest.mark.parametrize("key", ["oct", "s2"])
def test_size_query_capacity_and_null_fields(scene, key):
    import torch
    from point_cloud_viewer_b200 import _native as N

    h, fn = scene["h"][key], _fn(key)
    locs = [scene["locs"][k] for k in ("aabb_small", "obb", "miss", "frustum_far")]
    off = np.zeros(len(locs) + 1, np.uint64)
    assert _raw(h, fn, locs, (), off) == 0
    count_pass = h.last_stats()["bytes_read"]
    total = int(off[-1])
    assert total > 0
    full_off, full = h.query_batch_points(locs)
    full = _host(full)
    assert np.array_equal(full_off, off)
    dev = torch.device("cuda", scene["ctx"].device)
    # the size query writes nothing, not even the fields it is given
    sentinel = torch.full((total,), -7, dtype=torch.int64, device=dev)
    o2 = np.zeros_like(off)
    assert _raw(h, fn, locs, (), o2, None, None, None, sentinel, total) == 0 and np.array_equal(o2, off)
    assert bool((sentinel == -7).all())
    # one short: PCV_ERR_INVALID naming both numbers, offsets complete, the arrays untouched, nothing read after the count pass
    xyz = torch.full((total, 3), -1.0, dtype=torch.float64, device=dev)
    o3 = np.zeros_like(off)
    assert _raw(h, fn, locs, (), o3, xyz, None, None, sentinel, total - 1) == -1
    msg = N.lib().pcv_last_error().decode()
    assert str(total) in msg and str(total - 1) in msg
    assert np.array_equal(o3, off)
    assert bool((xyz == -1.0).all()) and bool((sentinel == -7).all())
    st = h.last_stats()
    assert st["chunks"] == 1 and st["bytes_read"] == _raw_fill_count_bytes(h, fn, locs, total, dev)
    assert st["bytes_read"] >= count_pass
    # position only, then position, intensity and provenance
    o4 = np.zeros_like(off)
    assert _raw(h, fn, locs, (), o4, xyz, None, None, None, total) == 0
    assert np.array_equal(xyz.cpu().numpy().view(np.uint64), full["xyz"].view(np.uint64))
    src = torch.zeros(total, dtype=torch.int64, device=dev)
    inten = torch.zeros(total, dtype=torch.float32, device=dev)
    xyz.fill_(0)
    assert _raw(h, fn, locs, (), o4, xyz, None, inten, src, total + 5) == 0
    assert np.array_equal(src.cpu().numpy(), full["src"]) and np.array_equal(inten.cpu().numpy(), full["intensity"])
    assert np.array_equal(xyz.cpu().numpy().view(np.uint64), full["xyz"].view(np.uint64))
    o5, part = h.query_batch_points(locs, fields=("src",))
    assert set(part) == {"src"} and np.array_equal(part["src"].cpu().numpy(), full["src"])


def _raw_fill_count_bytes(h, fn, locs, total, dev):
    """bytes_read of a fill that needs one chunk: the count pass of the same call, which read every needed file once."""
    import torch

    xyz = torch.zeros((total, 3), dtype=torch.float64, device=dev)
    off = np.zeros(len(locs) + 1, np.uint64)
    assert _raw(h, fn, locs, (), off, xyz, None, None, None, total) == 0
    st = h.last_stats()
    assert st["chunks"] == 2
    return st["bytes_read"]


def test_fields_the_directory_lacks_are_invalid(scene):
    import torch
    from point_cloud_viewer_b200 import _native as N

    L = N.lib()
    locs = [scene["locs"]["aabb_small"]]
    dev = torch.device("cuda", scene["ctx"].device)
    buf = torch.zeros((1 << 20, 3), dtype=torch.float64, device=dev)
    f32 = torch.zeros(1 << 20, dtype=torch.float32, device=dev)
    u8 = torch.zeros((1 << 20, 3), dtype=torch.uint8, device=dev)
    off = np.zeros(2, np.uint64)
    h = scene["h"]
    assert _raw(h["oct_noi"], L.pcv_octree_dir_query_batch_points_device, locs, (), off, buf, None, f32, None, 1 << 20) == -1
    assert _raw(h["s2_bare"], L.pcv_s2_dir_query_batch_points_device, locs, (), off, buf, None, f32, None, 1 << 20) == -1
    assert _raw(h["s2_bare"], L.pcv_s2_dir_query_batch_points_device, locs, (), off, buf, u8, None, None, 1 << 20) == -1
    assert _raw(h["s2_bare"], L.pcv_s2_dir_query_batch_points_device, locs, (), off, buf, None, None, None, 1 << 20) == 0
    with pytest.raises(scene["pcv"].PcvError):
        h["s2_bare"].query_batch_points(locs, fields=("xyz", "rgb"))


@pytest.mark.parametrize("key", ["oct", "s2"])
def test_argument_contract(scene, key):
    """As test_query_batch_points_gpu.py::test_argument_contract: an unknown kind, a null filter array, null offsets and filters
    without intensity are PCV_ERR_INVALID."""
    from point_cloud_viewer_b200 import _native as N

    L, G = N.lib(), scene["G"]
    fn = _fn(key)
    fu = L.pcv_s2_dir_query_cell_unions_batch_points_device if key == "s2" else L.pcv_octree_dir_query_cell_unions_batch_points_device
    h = scene["h"][key]
    off = np.zeros(2, np.uint64)
    assert _raw(h, fn, [G.all_points()], (), off) == 0 and off[1] > 0
    bad = G.all_points()
    bad.kind = 7
    assert _raw(h, fn, [bad], (), off) == -1
    assert fn(h.h, (N.Location * 1)(G.all_points()), 1, None, 1, off.ctypes.data, None, None, None, None, 0) == -1
    cu = scene["unions"]["some"]
    assert fu(h.h, (N.CellUnion * 1)(cu.struct()), 1, None, 1, off.ctypes.data, None, None, None, None, 0) == -1
    assert fn(h.h, (N.Location * 1)(G.all_points()), 1, None, 0, None, None, None, None, None, 0) == -1
    noi = scene["h"]["oct_noi" if key == "oct" else "s2_bare"]
    f = np.array([0.0, 10.0])
    assert fn(noi.h, (N.Location * 1)(G.all_points()), 1, f.ctypes.data, 1, off.ctypes.data, None, None, None, None, 0) == -1
    assert fu(noi.h, (N.CellUnion * 1)(cu.struct()), 1, f.ctypes.data, 1, off.ctypes.data, None, None, None, None, 0) == -1


# ---- front ends ----


def test_torch_views(scene):
    import torch

    def run():
        return scene["h"]["s2"].query_batch_points([scene["locs"]["obb"], scene["locs"]["aabb_small"]])

    off, t = run()
    gc.collect()
    total = int(off[-1])
    dev = torch.device("cuda", scene["ctx"].device)
    want = {"xyz": (torch.float64, (total, 3)), "rgb": (torch.uint8, (total, 3)), "intensity": (torch.float32, (total,)), "src": (torch.int64, (total,))}
    assert set(t) == set(want)
    for k, (dt, shape) in want.items():
        assert t[k].device == dev and t[k].dtype == dt and tuple(t[k].shape) == shape, k
    off2, t2 = run()
    for k in want:
        assert torch.equal(t[k], t2[k]), k


def test_cpp_overloads(tmp_path):
    """pcv::S2CellsDir::query_batch_points run once from C++ (tests/cpp/test_dir_batch_points.cpp); OctreeDir's compiled."""
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_dir_batch_points")
    lib_dir = os.path.join(root, "point_cloud_viewer_b200")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(cuda, "include"), os.path.join(root, "tests", "cpp", "test_dir_batch_points.cpp"), "-o", exe,
                           "-L" + lib_dir, "-l:libpcv_b200.so", "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir])
    r = subprocess.run([exe, str(tmp_path / "s2")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr
