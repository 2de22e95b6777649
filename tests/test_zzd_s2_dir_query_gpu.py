"""Point queries straight from an S2 directory (pcv_s2_dir_*, Context.open_s2_dir, S2Dir) on the 1e6-point ECEF slab (seed
80293751232) with intensity, written with build_s2_dir at level 20 and at a coarse level whose cells exceed a chunk.  Everything
is compared with load_s2_dir of the same directory and the resident calls (which test_zz7 ties to the oracle): metadata, cell
lists of every location kind, the streamed batches element for element at batch sizes 1, 4097 and 2^30 across a budget scan
from the smallest budget open accepts, batched counts over 1, 64 and 2000 frusta and over cell unions, with and without filters;
the I/O counters (which files a call reads, and that it reads them once), the budget, and every error of the contract."""
import os
import shutil

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SEED, N = 80293751232, 1_000_000
FILT = [(10.0, 60.0)]


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
def scene(ctx, tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED, 0, N)
    inten = np.random.default_rng(3).uniform(0.0, 100.0, N).astype(np.float32)
    base = tmp_path_factory.mktemp("s2q")
    dirs = {}
    for lvl in (20, 10):
        dirs[lvl] = base / ("l%d" % lvl)
        ctx.build_s2_dir(dirs[lvl], x, y, z, rgb, inten, split_level=lvl)
    loaded = {lvl: ctx.load_s2_dir(d) for lvl, d in dirs.items()}
    L = loaded[20]
    bmin, bmax = L.bbox_min, L.bbox_max
    d = bmax - bmin
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    e = G.Isometry((4157222.543, 664789.307, 4774952.099), q)
    c = G.web_mercator_coord(0.5 * (bmin + bmax), 19)
    ids = L.cell_ids
    locs = {
        "all": G.all_points(),
        "aabb": G.aabb(bmin + 0.2 * d, bmin + 0.8 * d),
        "aabb_small": G.aabb(bmin + 0.45 * d, bmin + 0.47 * d),
        "obb": G.obb(e, (50.0, 50.0, 5.0)),
        "frustum": G.frustum(e, G.Perspective.new_fov(1.0, 1.2, 0.1, 10.0)),
        "wm_rect": G.web_mercator_rect((c[0] - 200.0, c[1] - 200.0), (c[0] + 200.0, c[1] + 200.0), 19),
        "miss": G.aabb(bmax + 1000.0, bmax + 1100.0),
        # a level-20 cell and a level-14 ancestor of another (whole cells: no point test), a level-25 descendant (point tests)
        "union": G.cell_union([int(ids[len(ids) // 3]), (int(ids[len(ids) // 2]) & ~((1 << 33) - 1)) | (1 << 32)]),
        "union_fine": G.cell_union([(int(ids[7]) & ~((1 << 11) - 1)) | (1 << 10)]),
    }
    yield dict(pcv=pcv, G=G, ctx=ctx, dirs=dirs, loaded=loaded, locs=locs, bmin=bmin, bmax=bmax, base=base, x=x, y=y, z=z, rgb=rgb, inten=inten)
    for v in loaded.values():
        v.free()


def _cat(batches):
    keys = ("xyz", "rgb", "intensity", "src")
    out = dict(sizes=[len(b["src"]) for b in batches])
    for k in keys:
        parts = [b[k] for b in batches if b[k] is not None]
        out[k] = np.concatenate(parts) if parts else None
        if batches and batches[0][k] is None:
            out[k] = None
    return out


def _smallest_budget(pcv, ctx, d):
    """The smallest budget the handle accepts within 1/64, by a geometric scan (test_octree_dir_query_gpu._smallest_budget)."""
    lo, hi = 1 << 10, 1 << 34
    while hi - lo > lo // 64:
        mid = int((lo * hi) ** 0.5)
        try:
            pcv.S2Dir(ctx, d, mid).close()
            hi = mid
        except pcv.PcvError as e:
            assert e.code == -6
            lo = mid
    return hi, lo


def _selected(cloud, loc):
    """Indices of the cells the loaded cloud selects, in id order."""
    sel = cloud.cells_in_location(loc)
    return np.searchsorted(cloud.cell_ids, sel)


def _bounded(st):
    assert st["peak_device_bytes"] <= st["max_device_bytes"], st


def test_open_and_metadata(scene):
    s = scene
    for lvl, d in s["dirs"].items():
        h = s["ctx"].open_s2_dir(d)
        L = s["loaded"][lvl]
        assert (h.num_cells, h.num_points, h.split_level, h.has_color, h.has_intensity) == (L.num_cells, L.num_points, L.split_level, True, True)
        assert np.array_equal(h.bbox_min, L.bbox_min) and np.array_equal(h.bbox_max, L.bbox_max)
        assert np.array_equal(h.cell_ids, L.cell_ids) and np.array_equal(h.cell_counts, L.cell_counts)
        st = h.last_stats()
        assert st["bytes_read"] == 0 and st["node_files_read"] == 0
        _bounded(st)
        for k in (0, h.num_cells // 2, h.num_cells - 1):
            cid = int(h.cell_ids[k])
            got, want = h.cell_data(cid), L.cell_data(cid)
            for a, b in zip(got, want):
                assert np.array_equal(a, b)
        h.close()


def test_cell_lists(scene):
    s = scene
    G = s["G"]
    L = s["loaded"][20]
    h = s["ctx"].open_s2_dir(s["dirs"][20])
    for key in ("all", "union", "union_fine"):
        assert np.array_equal(h.cells_in_location(s["locs"][key]), L.cells_in_location(s["locs"][key])), key
        assert h.last_stats()["bytes_read"] == 0, key
    assert np.array_equal(h.cells_in_union(None), L.cells_in_union(None)) and h.last_stats()["bytes_read"] == 0
    assert np.array_equal(h.cells_in_union(s["locs"]["union"].ids), L.cells_in_union(s["locs"]["union"].ids))
    assert len(h.cells_in_location(G.cell_union([]))) == 0
    # the first polyhedral call scans every .xyz file once; no later call reads anything
    first = True
    for key in ("aabb", "aabb_small", "obb", "frustum", "wm_rect", "miss"):
        assert np.array_equal(h.cells_in_location(s["locs"][key]), L.cells_in_location(s["locs"][key])), key
        st = h.last_stats()
        _bounded(st)
        if first:
            assert st["bytes_read"] == 24 * N and st["node_files_read"] == h.num_cells, st
            first = False
        else:
            assert st["bytes_read"] == 0 and st["node_files_read"] == 0, (key, st)
    h.close()


def _check_stream(s, h, L, key, filters, bs):
    loc = s["locs"][key]
    got = h.query_points(loc, filters=filters, batch_size=bs)
    st = h.last_stats()
    want = L.query_points(loc, filters=filters, batch_size=bs)
    g, w = _cat(got), _cat(want)
    assert g["sizes"] == w["sizes"], key
    for k in ("xyz", "rgb", "intensity", "src"):
        assert (g[k] is None) == (w[k] is None) and (g[k] is None or np.array_equal(g[k], w[k])), (key, k)
    sel = _selected(L, loc)
    cnt = L.cell_counts[sel].astype(np.int64)
    sel = sel[cnt > 0]
    per = 24 + (3 if L.has_color else 0) + (4 if L.has_intensity else 0)
    assert st["bytes_read"] == per * int(cnt.sum()), (key, st)
    assert st["node_files_read"] == (1 + L.has_color + L.has_intensity) * len(sel), (key, st)
    assert st["tested_points"] == int(cnt.sum()) and st["returned_points"] == sum(g["sizes"]), (key, st)
    _bounded(st)
    return st


@pytest.mark.parametrize("lvl", [20, 10])
def test_stream_across_budgets(scene, lvl):
    s = scene
    pcv, ctx, d, L = s["pcv"], s["ctx"], s["dirs"][lvl], s["loaded"][lvl]
    small, refused = _smallest_budget(pcv, ctx, d)
    with pytest.raises(pcv.PcvError) as e:
        pcv.S2Dir(ctx, d, refused)
    assert e.value.code == -6
    for budget in (small, 8 * small, 0):
        h = ctx.open_s2_dir(d, budget)
        h.cells_in_location(s["locs"]["aabb"])  # the box scan, so that the calls below read only what they select
        for key in ("all", "aabb", "obb", "frustum", "wm_rect", "miss", "union", "union_fine"):
            for filters in ((), FILT):
                st = _check_stream(s, h, L, key, filters, 4097)
                if budget == small and key in ("all", "aabb"):
                    assert st["chunks"] > 8, st  # cells split across many chunks
        for key in ("all", "frustum", "union"):
            _check_stream(s, h, L, key, FILT, 1 << 30)
        _check_stream(s, h, L, "aabb_small", (), 1)
        h.close()


def test_batches(scene):
    s = scene
    pcv, ctx, G, L = s["pcv"], s["ctx"], s["G"], s["loaded"][20]
    h = ctx.open_s2_dir(s["dirs"][20])
    h.cells_in_location(s["locs"]["aabb"])  # the box scan, so that the calls below read only what they select
    ids = L.cell_ids
    unions = [G.cell_union([int(ids[k])]) for k in range(0, len(ids), max(1, len(ids) // 40))] + [s["locs"]["union"], G.cell_union([])]
    for locs in (_frusta(G, s["bmin"], s["bmax"], 1, 60.0), _frusta(G, s["bmin"], s["bmax"], 64, 60.0), _frusta(G, s["bmin"], s["bmax"], 2000, 60.0), unions):
        for filters in ((), FILT):
            counts, tested = h.query_batch(locs, filters=filters)
            st = h.last_stats()
            wc, wt = L.query_batch_device(locs, filters=filters)
            assert np.array_equal(counts, wc) and np.array_equal(tested, wt)
            _bounded(st)
            if len(locs) <= 64:
                cells = set()
                for loc in locs:
                    cells.update(_selected(L, loc).tolist())
                pts = int(L.cell_counts[sorted(cells)].sum()) if cells else 0
                per = 24 + (4 if filters else 0)
                assert st["bytes_read"] == per * pts, st  # each selected cell once, never its .rgb
                assert st["node_files_read"] == (2 if filters else 1) * len(cells), st
    small, _ = _smallest_budget(pcv, ctx, s["dirs"][20])
    hs = ctx.open_s2_dir(s["dirs"][20], small)
    with pytest.raises(pcv.PcvError) as e:
        hs.query_batch(_frusta(G, s["bmin"], s["bmax"], 2000, 60.0))
    assert e.value.code == -6 and "split the batch" in str(e.value)
    hs.close()
    h.close()


def test_attributes_and_cancel(scene, tmp_path):
    s = scene
    pcv, ctx = s["pcv"], s["ctx"]
    n = 200_000
    for name, rgb, inten in (("norgb", None, s["inten"][:n]), ("noint", s["rgb"][: 3 * n], None)):
        d = tmp_path / name
        ctx.build_s2_dir(d, s["x"][:n], s["y"][:n], s["z"][:n], rgb, inten, split_level=20)
        L = ctx.load_s2_dir(d)
        h = ctx.open_s2_dir(d, 1 << 24)
        assert h.has_color == (rgb is not None) and h.has_intensity == (inten is not None)
        h.cells_in_location(s["locs"]["aabb"])  # the box scan
        for key in ("all", "aabb", "union"):
            _check_stream(s, h, L, key, FILT if inten is not None else (), 4097)
        if inten is None:
            for call in (lambda: h.query_points(s["locs"]["aabb"], filters=FILT), lambda: h.query_batch([s["locs"]["aabb"]], filters=FILT)):
                with pytest.raises(pcv.PcvError) as e:
                    call()
                assert e.value.code == -1
        else:
            got = h.query_points(s["locs"]["all"], batch_size=4097)
            assert got and all(b["rgb"] is None for b in got)
        cid = int(h.cell_ids[3])
        for a, b in zip(h.cell_data(cid), L.cell_data(cid)):
            assert (a is None and b is None) or np.array_equal(a, b)
        h.close()
        L.free()
    h = ctx.open_s2_dir(s["dirs"][20])
    seen = []
    with pytest.raises(pcv.PcvError) as e:
        h.query_points(s["locs"]["all"], callback=lambda b: seen.append(len(b["src"])) or len(seen) == 2, batch_size=1000)
    assert e.value.code == -5 and seen == [1000, 1000]
    h.close()


def test_errors(scene, tmp_path):
    s = scene
    pcv, ctx = s["pcv"], s["ctx"]
    src = s["dirs"][20]
    L = s["loaded"][20]
    tok = pcv.s2_token(int(L.cell_ids[5]))

    def fresh(name):
        d = tmp_path / name
        shutil.copytree(src, d)
        return d

    def code(fn):
        with pytest.raises(pcv.PcvError) as e:
            fn()
        return e.value.code

    d = fresh("missing")
    os.remove(d / (tok + ".rgb"))
    assert code(lambda: ctx.open_s2_dir(d)) == -4
    d = fresh("short")
    with open(d / (tok + ".xyz"), "r+b") as f:
        f.truncate(24)
    assert code(lambda: ctx.open_s2_dir(d)) == -4
    d = fresh("shrunk")
    h = ctx.open_s2_dir(d)
    with open(d / (tok + ".intensity"), "r+b") as f:
        f.truncate(4)
    assert code(lambda: h.query_points(s["locs"]["all"])) == -4
    h.close()
    d = fresh("corrupt")
    with open(d / "meta.pb", "wb") as f:
        f.write(b"\xff\xff\xff")
    assert code(lambda: ctx.open_s2_dir(d)) == -1
    os.remove(d / "meta.pb")
    assert code(lambda: ctx.open_s2_dir(d)) == -3
    assert code(lambda: ctx.open_s2_dir(src, 4096)) == -6
