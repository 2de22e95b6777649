"""Point queries straight from an octree directory (pcv_octree_dir_*): node selection, filtered point streaming, batched culls and
the /nodes_data reply must equal the same calls over pcv_octree_load_dir of the directory (and the oracle's load_dir + query),
reading only the visited nodes' files, each once per call, within max_device_bytes."""
import os
import shutil
import sys

import numpy as np
import pytest

import oracle_api as O
from test_query_gpu import _cameras, _copy_loc, _locations

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)  # bench.make_frusta


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    """The 200k-point ECEF slab with intensity, max_points_per_node=3000, written with write_dir; load_dir of it and the oracle's."""
    import point_cloud_viewer_b200 as pcv

    n = 200_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    inten = (np.arange(n) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    c = pcv.Context(0, max_points_per_node=3000)
    d = str(tmp_path_factory.mktemp("slab"))
    tree = c.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    tree.write_dir(d)
    tree.free()
    res_tree = c.load_dir(d)
    everything = _cat(res_tree.query_points(pcv.geometry.all_points(), batch_size=1 << 30))
    yield dict(pcv=pcv, ctx=c, dir=d, res=res_tree, ref=O.load_dir(d), bmin=np.asarray(bmin), bmax=np.asarray(bmax), n=n, all=everything)
    res_tree.free()
    c.close()


def _cat(batches):
    if not batches:
        return dict(xyz=np.zeros((0, 3)), rgb=np.zeros((0, 3), np.uint8), intensity=None, src=np.zeros(0, np.uint64), sizes=[])
    it = [b["intensity"] for b in batches]
    return dict(xyz=np.concatenate([b["xyz"] for b in batches]), rgb=np.concatenate([b["rgb"] for b in batches]),
                intensity=None if it[0] is None else np.concatenate(it), src=np.concatenate([b["src"] for b in batches]), sizes=[len(b["src"]) for b in batches])


def _file_bytes(d, names):
    tot = files = 0
    for nm in names:
        for ext in (".xyz", ".rgb", ".intensity"):
            p = os.path.join(d, nm + ext)
            if os.path.exists(p):
                tot += os.path.getsize(p)
                files += 1
    return tot, files


def _smallest_budget(ctx, d):
    """The smallest budget the handle accepts within 1/64, by a geometric scan, and the largest refused one."""
    import point_cloud_viewer_b200 as pcv

    lo, hi = 1 << 10, 1 << 34
    while hi - lo > lo // 64:
        mid = int((lo * hi) ** 0.5)
        try:
            pcv.OctreeDir(ctx, d, mid).close()
            hi = mid
        except pcv.PcvError as e:
            assert e.code == -6
            lo = mid
    return hi, lo


def _check_stream(h, res_tree, s, loc, filters, bs, budget=None):
    got = h.query_points(loc, filters=filters, batch_size=bs)
    st = h.last_stats()
    want = res_tree.query_points(loc, filters=filters, batch_size=bs)
    g, w = _cat(got), _cat(want)
    assert g["sizes"] == w["sizes"]
    assert np.array_equal(g["xyz"], w["xyz"]) and np.array_equal(g["rgb"], w["rgb"]) and np.array_equal(g["intensity"], w["intensity"])
    # src is the point's slot: the same colour and position as slot s of load_dir
    a = s["all"]
    assert np.array_equal(a["xyz"][g["src"].astype(np.int64)], g["xyz"]) and np.array_equal(a["rgb"][g["src"].astype(np.int64)], g["rgb"])
    visited = [nm for nm in h.nodes_in_location(loc) if res_tree.nodes[nm]["num_points"] > 0]
    nb, nf = _file_bytes(s["dir"], visited)
    assert st["bytes_read"] == nb and st["node_files_read"] == nf
    assert st["returned_points"] == len(g["src"]) and st["tested_points"] == sum(res_tree.nodes[nm]["num_points"] for nm in visited)
    assert st["peak_device_bytes"] <= st["max_device_bytes"]
    if budget:
        assert st["max_device_bytes"] == budget
    return g, st


def test_selection_reads_no_file(scene):
    pcv, ctx = scene["pcv"], scene["ctx"]
    h = ctx.open_dir(scene["dir"])
    assert np.array_equal(h.nodes(), scene["res"].meta)
    for name, loc in _locations(scene).items():
        assert h.nodes_in_location(loc) == scene["res"].nodes_in_location(loc) == scene["ref"].nodes_in_location(_copy_loc(loc)), name
        assert h.last_stats()["node_files_read"] == 0
    some = 0
    for M in _cameras(scene, 50):
        got = h.get_visible_nodes(M)
        assert got == scene["res"].get_visible_nodes(M)
        st = h.last_stats()
        assert st["node_files_read"] == 0 and st["bytes_read"] == 0 and st["peak_device_bytes"] <= st["max_device_bytes"]
        some += len(got)
    assert some > 0
    with pytest.raises(pcv.PcvError) as e:
        h.get_visible_nodes(np.zeros((4, 4)))
    assert e.value.code == -7
    h.close()


def test_query_points_budget_scan(scene):
    pcv, ctx, res_tree = scene["pcv"], scene["ctx"], scene["res"]
    small, refused = _smallest_budget(ctx, scene["dir"])
    with pytest.raises(pcv.PcvError) as e:
        ctx.open_dir(scene["dir"], refused)
    assert e.value.code == -6 and str(refused) in str(e.value)
    whole = sum(os.path.getsize(os.path.join(scene["dir"], f)) for f in os.listdir(scene["dir"]))
    locs = _locations(scene)
    for budget in (small, small * 3, small * 20, 4 * whole):
        h = ctx.open_dir(scene["dir"], budget)
        for name, loc in locs.items():
            for filters in ((), (100.0, 250.0)):
                g, st = _check_stream(h, res_tree, scene, loc, filters, 7777, budget)
                if budget == small and not filters and name == "all":
                    split = sum(1 for m in res_tree.meta if m["num_points"] > 2048)
                    assert split > 0 and st["chunks"] > split  # a chunk holds one tile: nodes of more than 2048 points span chunks
            _check_stream(h, res_tree, scene, loc, (), scene["n"] + 5, budget)
        # the oracle's load_dir + query
        for name, loc in locs.items():
            want = scene["ref"].query(_copy_loc(loc), with_intensity=True)
            g = _cat(h.query_points(loc, batch_size=1 << 20))
            assert np.array_equal(g["xyz"], want["xyz"]) and np.array_equal(g["rgb"], want["rgb"]) and np.array_equal(g["intensity"], want["intensity"]), name
        h.close()
    h = ctx.open_dir(scene["dir"], small)
    _check_stream(h, res_tree, scene, locs["aabb_small"], (), 1, small)
    h.close()


def test_query_points_slots_cover_every_point(scene):
    h = scene["ctx"].open_dir(scene["dir"])
    g = _cat(h.query_points(scene["pcv"].geometry.all_points(), batch_size=1 << 30))
    assert np.array_equal(g["src"], np.arange(scene["n"], dtype=np.uint64))
    h.close()


def test_query_batch(scene):
    import bench

    pcv, ctx, res_tree = scene["pcv"], scene["ctx"], scene["res"]
    G = pcv.geometry
    small = _smallest_budget(ctx, scene["dir"])[0]
    for budget in (0, small * 40):
        h = ctx.open_dir(scene["dir"], budget)
        for far in (10.0, 102.4):
            locs = list(_locations(scene).values()) + bench.make_frusta(G, scene["bmin"], scene["bmax"], 200, far)
            for filters in ((), (100.0, 250.0)):
                counts, tested = h.query_batch(locs, filters=filters)
                st = h.last_stats()
                wc, wt = res_tree.query_batch_device(locs, filters=filters)
                assert np.array_equal(counts, wc) and np.array_equal(tested, wt)
                union = set()
                for loc in locs:
                    union |= {nm for nm in res_tree.nodes_in_location(loc) if res_tree.nodes[nm]["num_points"] > 0}
                nb, nf = _file_bytes(scene["dir"], union)
                assert st["node_files_read"] == nf and st["bytes_read"] == nb  # each visited node read once
                assert st["returned_points"] == int(counts.sum()) and st["tested_points"] == int(tested.sum())
                assert st["peak_device_bytes"] <= st["max_device_bytes"]
        h.close()


def test_cancellation(scene, tmp_path):
    """src/octree/tests.rs:83-136: batch 5000, the consumer errors at >= 13 000 points -> exactly 3 callbacks."""
    pcv = scene["pcv"]
    n = 100001
    x, y, z = np.zeros(n), np.zeros(n), np.zeros(n)
    x[-1], y[-1], z[-1] = -200.0, -40.0, 30.0
    rgb = np.tile(np.array([255, 0, 0], np.uint8), n)
    tree = scene["ctx"].build_octree(x, y, z, rgb, 1.0, (0, 0, 0), (-200, -40, 30))
    tree.write_dir(str(tmp_path))
    tree.free()
    h = scene["ctx"].open_dir(str(tmp_path))
    state = dict(points=0, calls=0)

    def consume(b):
        state["calls"] += 1
        state["points"] += len(b["src"])
        return state["points"] >= 13000

    with pytest.raises(pcv.PcvError) as e:
        h.query_points(pcv.geometry.all_points(), callback=consume, batch_size=5000)
    assert e.value.code == -5 and state["calls"] == 3 and state["points"] == 15000
    assert sum(len(b["src"]) for b in h.query_points(pcv.geometry.all_points(), batch_size=n // 2)) == n
    h.close()


def _equal_to_resident(ctx, d, budget, locs, filters_ok):
    res_tree = ctx.load_dir(d)
    s = dict(dir=d, all=_cat(res_tree.query_points(__import__("point_cloud_viewer_b200").geometry.all_points(), batch_size=1 << 30)))
    h = ctx.open_dir(d, budget)
    for loc in locs:
        _check_stream(h, res_tree, s, loc, (), 50000, budget)
        if filters_ok:
            _check_stream(h, res_tree, s, loc, (0.2, 0.7), 50000, budget)
    counts, tested = h.query_batch(locs)
    wc, wt = res_tree.query_batch_device(locs)
    assert np.array_equal(counts, wc) and np.array_equal(tested, wt)
    st = h.last_stats()
    h.close()
    res_tree.free()
    return st


def test_out_of_core_directory_with_large_leaves(scene, tmp_path):
    """A directory built out of core in several groups from config-2 points, with the 150 000-point coincident cluster."""
    import bench

    pcv = scene["pcv"]
    n = 1_300_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_GAUSS_CLUSTERS, 1, 0, n)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_GAUSS_CLUSTERS)
    inten = np.random.default_rng(4).random(n).astype(np.float32)
    ctx = pcv.Context(0, max_points_per_node=2000)
    info = ctx.build_octree_to_dir(str(tmp_path), x, y, z, rgb, res, bmin, bmax, intensity=inten, max_points_in_core=n // 3)
    assert info["groups"] > 1
    G = pcv.geometry
    d = np.asarray(bmax) - np.asarray(bmin)
    locs = [G.all_points(), G.aabb(np.asarray(bmin) + 0.2 * d, np.asarray(bmin) + 0.7 * d)] + bench.make_frusta(G, np.asarray(bmin), np.asarray(bmax), 6, 102.4)
    big = max(int(m["num_points"]) for m in ctx.load_dir(str(tmp_path)).meta)
    assert big >= 100_000  # the coincident cluster's leaf (the rest of its points went up into its ancestors)
    st = _equal_to_resident(ctx, str(tmp_path), 4 << 20, locs, True)  # a 4 MB budget: the large leaves span many chunks
    assert st["chunks"] > 1
    ctx.close()


def test_float64_and_partial_intensity_directories(scene, tmp_path):
    pcv, ctx = scene["pcv"], scene["ctx"]
    n = 300_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_GAUSS_CLUSTERS, 2, 0, n)
    bmin, bmax, _ = pcv.synth_bbox(pcv.SYNTH_GAUSS_CLUSTERS)
    c2 = pcv.Context(0, max_points_per_node=2000)
    tree = c2.build_octree(x, y, z, rgb, 1e-6, bmin, bmax)  # the upper levels are Float64 encoded
    assert any(int(m["enc"]) == 4 and m["num_points"] > 0 for m in tree.meta)
    tree.write_dir(str(tmp_path / "f64"))
    tree.free()
    G = pcv.geometry
    d = np.asarray(bmax) - np.asarray(bmin)
    locs = [G.all_points(), G.aabb(np.asarray(bmin) + 0.3 * d, np.asarray(bmin) + 0.6 * d)]
    _equal_to_resident(c2, str(tmp_path / "f64"), 2 << 20, locs, False)
    c2.close()
    # some nodes without .intensity: load_dir reads them as zeros
    part = tmp_path / "partial"
    shutil.copytree(scene["dir"], part)
    gone = sorted(f for f in os.listdir(part) if f.endswith(".intensity"))[::3]
    for f in gone:
        os.remove(part / f)
    st = _equal_to_resident(ctx, str(part), 0, list(_locations(scene).values())[:4], True)
    assert st["node_files_read"] > 0


def test_errors(scene, tmp_path):
    pcv, ctx = scene["pcv"], scene["ctx"]
    E = pcv.PcvError

    def copy(name):
        d = tmp_path / name
        shutil.copytree(scene["dir"], d)
        return d

    d = copy("truncated")
    victim = sorted(f for f in os.listdir(d) if f.endswith(".rgb"))[4]
    (d / victim).write_bytes((d / victim).read_bytes()[:-1])
    with pytest.raises(E) as e:
        ctx.open_dir(d)
    assert e.value.code == -4 and victim in str(e.value)
    d = copy("version")
    meta = bytearray((d / "meta.pb").read_bytes())
    assert meta[:2] == b"\x08\x0d"
    meta[1] = 12
    (d / "meta.pb").write_bytes(bytes(meta))
    with pytest.raises(E) as e:
        ctx.open_dir(d)
    assert e.value.code == -1
    # a file that shrinks after open: the call that reads it fails
    d = copy("shrinks")
    h = ctx.open_dir(d)
    victim = max((f for f in os.listdir(d) if f.endswith(".xyz")), key=lambda f: os.path.getsize(d / f))
    (d / victim).write_bytes((d / victim).read_bytes()[:-6])
    with pytest.raises(E) as e:
        h.query_points(pcv.geometry.all_points())
    assert e.value.code == -4 and victim in str(e.value)
    h.close()
    # filters without intensities
    d = copy("no_intensity")
    for f in os.listdir(d):
        if f.endswith(".intensity"):
            os.remove(d / f)
    h = ctx.open_dir(d)
    with pytest.raises(E) as e:
        h.query_points(pcv.geometry.all_points(), filters=(0.0, 1.0))
    assert e.value.code == -1 and "Filter attribute" in str(e.value)
    with pytest.raises(E) as e:
        h.query_batch([pcv.geometry.all_points()], filters=(0.0, 1.0))
    assert e.value.code == -1
    h.close()


def test_nodes_data_blob(scene):
    pcv, ctx, res_tree = scene["pcv"], scene["ctx"], scene["res"]
    h = ctx.open_dir(scene["dir"])
    M = _cameras(scene, 4)[1]
    names = h.get_visible_nodes(M)
    assert names
    got = h.nodes_data_blob(names)
    assert got.tobytes() == res_tree.nodes_data_blob(names).tobytes() == scene["ref"].nodes_data_blob(names)
    st = h.last_stats()
    assert st["node_files_read"] == 2 * len(names)
    with pytest.raises(pcv.PcvError) as e:
        h.nodes_data_blob(names[:1] + ["r" + "7" * 12])
    assert e.value.code == -4
    h.close()
