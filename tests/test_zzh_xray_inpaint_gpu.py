"""Inpainting X-ray quadtrees on the GPU (pcv_xray_inpaint_quadtree, Context.inpaint_xray_quadtree).  Quadtrees written by
xray_quadtree_write_dir on a transparent background from points with small holes between them and large empty bands; every
output PNG equals the CPU restatement (tests/xray_inpaint_ref.py: leaves through the numpy steps, parents through the
oracle's Lanczos3) pixel for pixel at inpaint distances 0, 1, 3, 8 and 255 and tile sizes 32 and 64, with the file set and
the meta bytes.  Also: a sub-root piece among its neighbour pieces in one directory, copied and in place; budgets; a white
input that comes out unchanged; every error, each leaving no meta."""
import os
import shutil

import numpy as np
import pytest
from PIL import Image

import xray_inpaint_ref as R
import xray_merge_ref as M

pytestmark = pytest.mark.gpu

PX = 0.25
WHITE, TRANSPARENT = (255, 255, 255, 255), (255, 255, 255, 0)


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    base = tmp_path_factory.mktemp("inpaint")
    rng = np.random.default_rng(5)
    n = 40_000
    x, y, z = rng.uniform(0, 100, n), rng.uniform(0, 100, n), rng.uniform(0, 10, n)
    keep = ~((x > 40) & (x < 55)) & ~((y > 70) & (y < 72))  # a wide band and a narrow one without points
    x, y, z = x[keep], y[keep], z[keep]
    x[0], y[0], z[0], x[1], y[1], z[1] = 0.0, 0.0, 0.0, 100.0, 100.0, 10.0
    rgb = rng.integers(0, 256, 3 * len(x), dtype=np.uint8)
    ctx = pcv.Context(0, max_points_per_node=3000)
    tree = ctx.build_octree(x, y, z, rgb, 0.001, (0.0, 0.0, 0.0), (100.0, 100.0, 10.0))
    yield dict(pcv=pcv, ctx=ctx, tree=tree, base=base)
    tree.free()
    ctx.close()


def _build(s, T, name, **kw):
    d = str(s["base"] / ("%s_%d" % (name, T)))
    if not os.path.exists(d):
        s["tree"].xray_quadtree_write_dir(d, T, PX * 32 / T, **kw)
    return d


def _pngs(d):
    return sorted(f for f in os.listdir(d) if f.endswith(".png"))


def _check(out, ref, want_files):
    assert _pngs(out) == sorted(want_files)
    for (l, i), im in ref.items():
        got = R.read_png(os.path.join(out, M.node_name(l, i) + ".png"))
        assert np.array_equal(got, im), (l, i)


def _expected_files(ref):
    return [M.node_name(l, i) + ".png" for (l, i) in ref]


@pytest.mark.parametrize("T", [32, 64])
@pytest.mark.parametrize("k", [0, 1, 3, 8, 255])
def test_inpaint_equals_the_restatement(scene, T, k, tmp_path):
    src = _build(scene, T, "full", background=TRANSPARENT)
    out = str(tmp_path / "out")
    info = scene["ctx"].inpaint_xray_quadtree(src, out, k, background=WHITE)
    ref, adj, holes = R.inpaint_dir(src, k, WHITE)
    _check(out, ref, _expected_files(ref))
    assert open(os.path.join(out, "meta.pb"), "rb").read() == open(os.path.join(src, "meta.pb"), "rb").read()
    meta = M.read_meta(open(os.path.join(src, "meta.pb"), "rb").read())
    assert info["leaves"] == sum(1 for l, _ in meta.nodes if l == meta.deepest) and info["adjacent_leaves"] == 0 == len(adj)
    assert info["hole_pixels_filled"] == holes and (holes > 0) == (k > 0)
    assert info["parents_built"] == len(ref) - info["leaves"] and info["files_copied"] == 1
    assert info["peak_device_bytes"] <= info["max_device_bytes"]
    if k:
        leaves = [im for (l, _), im in ref.items() if l == meta.deepest]
        plain = [R.background(R.read_png(os.path.join(src, M.node_name(l, i) + ".png")), WHITE) for (l, i) in ref if l == meta.deepest]
        assert any(not np.array_equal(a, b) for a, b in zip(leaves, plain))  # something was filled or blended


@pytest.mark.parametrize("in_place", [False, True])
def test_piece_among_neighbour_pieces(scene, in_place, tmp_path):
    T, L = 32, 1
    shared = str(tmp_path / "pieces")
    for i in range(4):
        scene["tree"].xray_quadtree_write_dir(shared, T, PX, background=TRANSPARENT, root=(L, i))
    before = {f: R.read_png(os.path.join(shared, f)) for f in _pngs(shared)}
    for piece in (0, 3):
        src = shared
        if in_place:
            src = str(tmp_path / ("inplace%d" % piece))
            shutil.copytree(shared, src)
        ref, adj, holes = R.inpaint_dir(src, 8, WHITE, root=(L, piece), in_place=in_place)
        out = src if in_place else str(tmp_path / ("out%d" % piece))
        info = scene["ctx"].inpaint_xray_quadtree(src, out, 8, background=WHITE, root=(L, piece))
        assert info["adjacent_leaves"] == len(adj) > 0 and info["hole_pixels_filled"] == holes
        for (l, i), im in ref.items():
            assert np.array_equal(R.read_png(os.path.join(out, M.node_name(l, i) + ".png")), im), (piece, l, i)
        mname = R.meta_name(L, piece)
        if in_place:
            # every other file is as it was
            done = {M.node_name(l, i) + ".png" for (l, i) in ref}
            assert _pngs(out) == sorted(before)
            for f in before:
                if f not in done:
                    assert np.array_equal(R.read_png(os.path.join(out, f)), before[f]), f
            assert not [f for f in os.listdir(out) if f.startswith(".inpaint")]
        else:
            _check(out, ref, _expected_files(ref))  # no adjacent leaf is left
            assert sorted(f for f in os.listdir(out) if f.endswith(".pb")) == [mname]


def test_budgets_give_identical_files(scene, tmp_path):
    src = _build(scene, 64, "full", background=TRANSPARENT)
    outs, need = [], None
    for kk, budget in enumerate((0, None)):
        out = str(tmp_path / ("b%d" % kk))
        info = scene["ctx"].inpaint_xray_quadtree(src, out, 3, background=WHITE, max_device_bytes=budget if budget is not None else need)
        need = info["device_bytes_needed"]
        assert info["peak_device_bytes"] <= info["max_device_bytes"]
        outs.append((out, info))
    assert outs[0][1]["block_depth"] > 0 and outs[1][1]["block_depth"] == 0
    assert outs[1][1]["blocks"] == outs[1][1]["leaves"] and outs[0][1]["blocks"] < outs[1][1]["leaves"]
    assert outs[0][1]["hole_pixels_filled"] == outs[1][1]["hole_pixels_filled"]
    assert _pngs(outs[0][0]) == _pngs(outs[1][0])
    for f in _pngs(outs[0][0]):
        assert np.array_equal(R.read_png(os.path.join(outs[0][0], f)), R.read_png(os.path.join(outs[1][0], f))), f


def test_white_input_leaves_come_out_unchanged(scene, tmp_path):
    src = _build(scene, 32, "white", background=WHITE)
    out = str(tmp_path / "out")
    info = scene["ctx"].inpaint_xray_quadtree(src, out, 8, background=WHITE)
    assert info["hole_pixels_filled"] == 0
    meta = M.read_meta(open(os.path.join(src, "meta.pb"), "rb").read())
    for (l, i) in meta.nodes:
        f = M.node_name(l, i) + ".png"
        if l == meta.deepest:
            assert np.array_equal(R.read_png(os.path.join(out, f)), R.read_png(os.path.join(src, f))), f


def test_errors_leave_no_meta(scene, tmp_path):
    pcv, ctx = scene["pcv"], scene["ctx"]
    src = _build(scene, 32, "full", background=TRANSPARENT)

    def code(inp, name, **kw):
        out = str(tmp_path / ("out_" + name))
        args = dict(background=WHITE)
        args.update(kw)
        k = args.pop("k", 3)
        with pytest.raises(pcv.PcvError) as e:
            ctx.inpaint_xray_quadtree(inp, out, k, **args)
        assert not os.path.exists(out) or not [f for f in os.listdir(out) if f.endswith(".pb")], name
        return e.value.code

    assert code(str(tmp_path / "missing"), "missing") == -4
    assert code(src, "nometa", root=(1, 2)) == -4
    assert code(src, "k", k=256) == -1
    assert code(src, "outside", root=(1, 4)) == -1
    meta = M.read_meta(open(os.path.join(src, "meta.pb"), "rb").read())
    leaf = next(M.node_name(l, i) + ".png" for l, i in meta.nodes if l == meta.deepest)
    for name, fix, want in (("gone", lambda p: os.remove(p), -3), ("corrupt", lambda p: open(p, "r+b").write(b"\x89PNG\r\n\x1a\nxx"), -3),
                            ("size", lambda p: Image.new("RGBA", (34, 34)).save(p), -1)):
        d = str(tmp_path / ("img_" + name))
        shutil.copytree(src, d)
        fix(os.path.join(d, leaf))
        assert code(d, name) == want, name
    odd = str(tmp_path / "odd")
    scene["tree"].xray_quadtree_write_dir(odd, 33, PX, background=TRANSPARENT)
    assert code(odd, "odd") == -6
    need = ctx.inpaint_xray_quadtree(src, str(tmp_path / "ok"), 3)["device_bytes_needed"]
    with pytest.raises(pcv.PcvError) as e:
        ctx.inpaint_xray_quadtree(src, str(tmp_path / "low"), 3, max_device_bytes=need - 1)
    assert e.value.code == -6 and str(need) in str(e.value)
    assert not os.path.exists(str(tmp_path / "low"))
