"""The bounded X-ray quadtree driver (pcv_xray_quadtree_bounded) against the oracle's build_xray_quadtree
(xray/src/generation.rs:560-759): node sets and tiles under budgets that give several blocks or the whole tree in one block,
and one leaf per key batch; post-order delivery, cancellation, the budget itself, edge leaves and a deep, sparse quadtree."""
import os

import numpy as np
import pytest

import oracle_api as O

pytestmark = pytest.mark.gpu

WHITE = (255, 255, 255, 255)
TRANSPARENT = (255, 255, 255, 0)


@pytest.fixture(scope="module")
def scene():
    import point_cloud_viewer_b200 as pcv

    n = 150_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    inten = ((np.arange(n) * 7919) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    c = pcv.Context(0, max_points_per_node=4000)
    tree = c.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    ref = O.build(x, y, z, rgb.reshape(-1, 3), res, bmin, bmax, intensity=inten, max_points_per_node=4000)
    yield dict(pcv=pcv, ctx=c, tree=tree, ref=ref, bmin=np.asarray(bmin), bmax=np.asarray(bmax))
    tree.free()
    c.close()


def _post_order_ok(order):
    pos = {k: i for i, k in enumerate(order)}
    assert len(pos) == len(order), "a tile was delivered twice"
    for (l, i), p in pos.items():
        for k in range(4):
            ch = (l + 1, (i << 2) + k)
            if ch in pos:
                assert pos[ch] < p, ("child after parent", ch, (l, i))
    return True


def _run(tree, T, px, budget, **kw):
    order = []
    info, tiles = tree.xray_quadtree(T, px, on_tile=lambda l, i, img: order.append((l, i)) and False, max_device_bytes=budget, **kw)
    assert _post_order_ok(order) and set(order) == set(tiles)
    if budget:
        assert info["max_device_bytes"] == budget and info["peak_device_bytes"] <= budget
    return info, tiles


def _budgets(T):
    tile = T * T * 4
    # small blocks, several blocks, and the default (the whole tree in one block)
    return (tile * 90 + 600_000, tile * 300 + 2_000_000, 0)


@pytest.mark.parametrize("T,depth", [(32, 4), (16, 5)])
def test_xray_strategy_equals_oracle_under_budgets(scene, T, depth):
    tree, ref = scene["tree"], scene["ref"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (2 ** depth * T) * 1.01
    seen_levels = set()
    for bg in (WHITE, TRANSPARENT):
        oinfo, otiles = ref.xray_quadtree(T, px, background=bg)
        assert oinfo["deepest_level"] == depth
        for budget in _budgets(T):
            info, tiles = _run(tree, T, px, budget, background=bg)
            assert set(tiles) == set(otiles), budget
            for k in otiles:
                assert np.array_equal(tiles[k], otiles[k]), (budget, k)
            assert info["num_leaves"] == sum(1 for k in otiles if k[0] == depth)
            assert info["positions_evaluated"] <= 4 * 4 ** depth
            seen_levels.add(info["block_level"])
            if budget == 0:
                assert info["block_level"] == 0 and info["blocks_processed"] == 1
            else:
                assert info["block_level"] > 0 and info["blocks_processed"] > 1
    assert len(seen_levels) >= 2


def test_query_frame_and_sub_root(scene):
    pcv, tree, ref = scene["pcv"], scene["tree"], scene["ref"]
    G = pcv.geometry
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    qfg = G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7()
    T = 32
    oinfo, otiles = ref.xray_quadtree(T, 0.5, query_from_global=qfg)
    for budget in _budgets(T):
        info, tiles = _run(tree, T, 0.5, budget, query_from_global=qfg)
        assert info["deepest_level"] == oinfo["deepest_level"] and set(tiles) == set(otiles)
        assert all(np.array_equal(tiles[k], otiles[k]) for k in otiles)
    sub = sorted(k for k in otiles if k[0] == 2)[0]
    oinfo2, otiles2 = ref.xray_quadtree(T, 0.5, query_from_global=qfg, root=sub)
    info2, tiles2 = _run(tree, T, 0.5, _budgets(T)[0], query_from_global=qfg, root=sub)
    assert set(tiles2) == set(otiles2) and all(np.array_equal(tiles2[k], otiles2[k]) for k in otiles2)
    assert (info2["rect_min_x"], info2["rect_min_y"], info2["rect_edge"]) == (oinfo2["rect_min_x"], oinfo2["rect_min_y"], oinfo2["rect_edge"])


def test_other_strategies_under_a_small_budget(scene):
    pcv, tree, ref = scene["pcv"], scene["tree"], scene["ref"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    T = 32
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (4 * T) * 1.01
    for kw, budget in ((dict(strategy=pcv.XRAY_COLORED), 4 << 20), (dict(strategy=pcv.XRAY_INTENSITY, p0=0.0, p1=1000.0, bin_size=20.0), 24 << 20),
                       (dict(strategy=pcv.XRAY_HEIGHT_STDDEV, p0=1.5, colormap=1), 4 << 20)):
        info, tiles = _run(tree, T, px, budget, background=TRANSPARENT, **kw)
        oinfo, otiles = ref.xray_quadtree(T, px, background=TRANSPARENT, **kw)
        assert set(tiles) == set(otiles)
        for k in (k for k in otiles if k[0] == 2):
            assert np.array_equal(tiles[k][..., 3], otiles[k][..., 3])
            assert np.abs(tiles[k].astype(np.int16) - otiles[k].astype(np.int16)).max() <= 1
        for k in (k for k in tiles if k[0] < 2):
            ch = [tiles.get((k[0] + 1, (k[1] << 2) + j)) for j in range(4)]
            assert np.array_equal(tiles[k], O.build_parent_tile(ch, TRANSPARENT, T)), k


def test_cancel_and_budget_errors(scene):
    pcv, tree = scene["pcv"], scene["tree"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    T = 16
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (16 * T) * 1.01
    full, _ = _run(tree, T, px, _budgets(T)[1])
    for k in (1, 5, full["num_nodes"] - 1):
        seen = []
        with pytest.raises(pcv._native.PcvError) as e:
            tree.xray_quadtree(T, px, on_tile=lambda l, i, img: seen.append((l, i)) or len(seen) >= k, max_device_bytes=_budgets(T)[1])
        assert e.value.code == -5 and len(seen) == k
    again, _ = _run(tree, T, px, _budgets(T)[1])
    assert again["num_nodes"] == full["num_nodes"]
    with pytest.raises(pcv._native.PcvError) as e:
        tree.xray_quadtree(T, px, max_device_bytes=T * T * 4 - 1)
    assert e.value.code == -6


@pytest.mark.parametrize("face", ["min_y", "max_x_obb"])
def test_edge_leaf(face):
    """Every point of one leaf lies exactly on one face of it (power-of-two boxes and a resolution fine enough for float
    position encodings, so the positions decode exactly): no point
    lands on a pixel, but the reference creates the leaf, because its points pass the location test.  The Aabb of a leaf
    is half-open (min <= p < max), so its min-y face is inside it; the Obb under query_from_global is closed, so its max-x
    face is inside it too."""
    import point_cloud_viewer_b200 as pcv

    rng = np.random.default_rng(7)
    n = 4000
    x = rng.uniform(0.0, 64.0, n)
    y = rng.uniform(0.0, 64.0, n)
    z = rng.uniform(0.0, 8.0, n)
    keep = ~((x >= 16) & (x <= 24) & (y >= 16) & (y < 24))  # leaf (16..24, 16..24) of 8 m tiles: only face points
    x, y, z = x[keep], y[keep], z[keep]
    along = 16.0 + 0.125 + np.arange(32) * 0.25
    fx, fy = (along, np.full(32, 16.0)) if face == "min_y" else (np.full(32, 24.0), along)
    x = np.concatenate([x, fx, [0.0, 64.0]])
    y = np.concatenate([y, fy, [0.0, 64.0]])
    z = np.concatenate([z, np.full(32, 4.0), [0.0, 8.0]])
    qfg = None if face == "min_y" else (0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0)
    rgb = np.full((len(x), 3), 200, np.uint8)
    bmin, bmax, res = (0.0, 0.0, 0.0), (64.0, 64.0, 8.0), 1e-9
    c = pcv.Context(0, max_points_per_node=500)
    tree = c.build_octree(x, y, z, rgb.reshape(-1), res, bmin, bmax)
    ref = O.build(x, y, z, rgb, res, bmin, bmax, max_points_per_node=500)
    try:
        for bg in (WHITE, TRANSPARENT):
            oinfo, otiles = ref.xray_quadtree(8, 1.0, background=bg, query_from_global=qfg)
            assert (3, 0b001100) in otiles  # the face-only leaf (x 16..24 -> 2, y 16..24 -> 2)
            for budget in (0, 200_000):
                info, tiles = _run(tree, 8, 1.0, budget, background=bg, query_from_global=qfg)
                assert set(tiles) == set(otiles)
                assert all(np.array_equal(tiles[k], otiles[k]) for k in otiles)
    finally:
        tree.free()
        c.close()


def test_key_batch_split():
    """A shallow octree whose root holds points: every leaf position can hold a large share of the points, so small budgets
    split a block's leaves into several key batches.  Budgets are scanned upwards from one that is refused (a leaf's keys do
    not fit) to one that takes the whole tree in one batch; every run that fits equals the oracle."""
    import point_cloud_viewer_b200 as pcv

    rng = np.random.default_rng(11)
    n = 20_000
    x, y, z = rng.uniform(0.0, 64.0, n), rng.uniform(0.0, 64.0, n), rng.uniform(0.0, 8.0, n)
    x[:3000] = rng.uniform(0.0, 20.0, 3000)  # a dense corner and some empty leaves
    keep = ~((x > 40) & (y > 40))
    x, y, z = x[keep], y[keep], z[keep]
    rgb = np.full((len(x), 3), 90, np.uint8)
    bmin, bmax, res = (0.0, 0.0, 0.0), (64.0, 64.0, 8.0), 1.0 / 256
    c = pcv.Context(0, max_points_per_node=10 ** 6)
    tree = c.build_octree(x, y, z, rgb.reshape(-1), res, bmin, bmax)
    ref = O.build(x, y, z, rgb, res, bmin, bmax, max_points_per_node=10 ** 6)
    try:
        oinfo, otiles = ref.xray_quadtree(8, 1.0)
        budget, refused, runs = 60_000, False, []
        while budget < 64 << 20:
            try:
                info, tiles = _run(tree, 8, 1.0, budget)
            except pcv._native.PcvError as e:
                assert e.code == -6 and not runs  # only budgets below the first that fits are refused
                refused = True
            else:
                assert set(tiles) == set(otiles) and all(np.array_equal(tiles[k], otiles[k]) for k in otiles)
                runs.append(info)
            budget = int(budget * 1.25)
        assert refused and runs
        assert runs[0]["key_batches"] > runs[0]["blocks_processed"]  # some block needed several key batches
        assert runs[-1]["key_batches"] == runs[-1]["blocks_processed"] == 1
        assert all(r["num_leaves"] == sum(1 for k in otiles if k[0] == 3) for r in runs)
    finally:
        tree.free()
        c.close()


def _leaf_set(px, py, rect, deepest):
    """Leaves whose location (Aabb: min <= p < max) holds a point, with the quad_rect_of recurrence (quadtree lib.rs:62-101)."""
    out = set()
    for xv, yv in zip(px.tolist(), py.tolist()):
        stack = [(0, 0, rect[0], rect[1], rect[2])]
        while stack:
            l, i, mx, my, e = stack.pop()
            if not (mx <= xv < mx + e and my <= yv < my + e):
                continue
            if l == deepest:
                out.add(i)
                continue
            h = e / 2.0
            for k in range(4):
                stack.append((l + 1, (i << 2) + k, mx + (h if k & 2 else 0.0), my + (h if k & 1 else 0.0), h))
    return out


def test_deep_sparse_quadtree(scene):
    """deepest - root >= 14 with 8 px tiles (more than 2.6e8 leaf positions, refused before): the created leaves are exactly
    the leaves whose location holds a point, sampled leaves equal pcv_xray_tile, and the positions evaluated stay within a
    small multiple of the created leaves."""
    pcv, tree = scene["pcv"], scene["tree"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    T = 8
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (2 ** 14 * T) * 1.01
    info, tiles = _run(tree, T, px, 256 << 20)
    deepest = info["deepest_level"]
    assert deepest >= 14 and info["blocks_processed"] > 1
    pts = np.concatenate([b["xyz"] for b in tree.query_points(pcv.geometry.all_points(), batch_size=1 << 20)])
    zin = (bmin[2] <= pts[:, 2]) & (pts[:, 2] < bmax[2])  # the Aabb's z range is half-open too
    want = _leaf_set(pts[zin, 0], pts[zin, 1], (info["rect_min_x"], info["rect_min_y"], info["rect_edge"]), deepest)
    got = {i for (l, i) in tiles if l == deepest}
    assert got == want and info["num_leaves"] == len(want)
    assert info["positions_evaluated"] <= 8 * len(want)
    rng = np.random.default_rng(3)
    for i in rng.choice(sorted(got), 24, replace=False).tolist():
        mnx, mny, e = info["rect_min_x"], info["rect_min_y"], info["rect_edge"]
        for lv in range(deepest - 1, -1, -1):
            k = (i >> (2 * lv)) & 3
            e = e / 2.0
            mny += e if k & 1 else 0.0
            mnx += e if k & 2 else 0.0
        _, img, _ = tree.xray_tile((mnx, mny, bmin[2]), (mnx + e, mny + e, bmax[2]), T, T)
        assert np.array_equal(tiles[(deepest, i)], pcv.xray_assign_background(scene["ctx"], img, WHITE)), i


def test_bounded_write_dir(scene, tmp_path):
    from PIL import Image

    tree, ref = scene["tree"], scene["ref"]
    bmin, bmax = scene["bmin"], scene["bmax"]
    T = 16
    px = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1])) / (8 * T) * 1.01
    oinfo, otiles = ref.xray_quadtree(T, px)
    info = tree.xray_quadtree_write_dir(tmp_path, T, px, max_device_bytes=_budgets(T)[0])
    assert info["peak_device_bytes"] <= _budgets(T)[0]
    names = set(os.listdir(tmp_path))
    assert "meta.pb" in names and len(names) == len(otiles) + 1
    for (l, i), img in otiles.items():
        name = "r" + "".join(str((i >> (2 * k)) & 3) for k in range(l - 1, -1, -1)) + ".png"
        got = np.asarray(Image.open(tmp_path / name).convert("RGBA"))
        assert np.array_equal(got, img), name
