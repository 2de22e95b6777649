"""Merging partial X-ray quadtrees on the GPU (pcv_xray_merge_quadtrees, Context.merge_xray_quadtrees).  Every sub-root at levels
1 and 2 of three sources - a resident octree, an S2 cloud and two octree directories through xray_quadtree_from_dirs - is built
with its *_write_dir entry, some into directories of their own and the rest into one shared directory, some of them empty; their
merge has the file set, the pixels of every PNG, the node set, levels, tile size and (dyadic scene) the bits of the rect of the
full build, and its parents equal the CPU restatement's merge (tests/xray_merge_ref.py).  Attribute strategies are compared with
that restatement only.  Edge cases: both backgrounds, output into an input directory and into a directory that does not exist,
a single level-0 input, version 2 metas, 1024 px tiles; budgets; every error, each leaving no meta.pb."""
import os
import shutil
import struct

import numpy as np
import pytest
from PIL import Image

import xray_merge_ref as R
from proto_meta import XrayMeta

pytestmark = pytest.mark.gpu

T, PX = 32, 0.25
WHITE, TRANSPARENT = (255, 255, 255, 255), (255, 255, 255, 0)


def _q(v):
    return np.round(np.asarray(v) * 4.0) / 4.0  # multiples of 0.25 m: the box minimum and every rect of the walk are exact


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    base = tmp_path_factory.mktemp("merge")
    rng = np.random.default_rng(11)
    n = 60_000
    x, y, z = _q(rng.uniform(0, 100, n)), _q(rng.uniform(0, 100, n)), _q(rng.uniform(0, 10, n))
    # holes in the quadtree's 128 m square: sub-root 2 at level 1 ([64, 128] x [0, 64]) and sub-root 5 at level 2 ([0, 32] x
    # [96, 128]) hold no point
    keep = ~((x > 60) & (y < 68)) & ~((x < 36) & (y > 92))
    x, y, z = x[keep], y[keep], z[keep]
    x[0], y[0], z[0], x[1], y[1], z[1] = 0.0, 0.0, 0.0, 100.0, 100.0, 10.0
    m = len(x)
    rgb = rng.integers(0, 256, 3 * m, dtype=np.uint8)
    inten = rng.uniform(0, 1000, m).astype(np.float32)
    ctx = pcv.Context(0, max_points_per_node=3000)
    tree = ctx.build_octree(x, y, z, rgb, 0.001, (0.0, 0.0, 0.0), (100.0, 100.0, 10.0), intensity=inten)
    # the octree directories: two halves of the points
    dirs = [str(base / "oct_a"), str(base / "oct_b")]
    for d, sl in zip(dirs, (slice(0, m // 2), slice(m // 2, m))):
        t = ctx.build_octree(x[sl].copy(), y[sl].copy(), z[sl].copy(), rgb.reshape(-1, 3)[sl].reshape(-1).copy(), 0.001, (0.0, 0.0, 0.0),
                             (100.0, 100.0, 10.0), intensity=inten[sl].copy())
        t.write_dir(d)
        t.free()
    sx, sy, sz, srgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 5, 0, 80_000)
    s2 = ctx.build_s2_cloud(_q(sx), _q(sy), _q(sz), srgb, intensity=rng.uniform(0, 1000, 80_000).astype(np.float32))
    writers = {
        "octree": lambda out, **kw: tree.xray_quadtree_write_dir(out, T, PX, **kw),
        "s2": lambda out, **kw: s2.xray_quadtree_write_dir(out, T, PX, **kw),
        "dirs": lambda out, **kw: ctx.xray_quadtree_from_dirs_write_dir(dirs, out, T, PX, **kw),
    }
    yield dict(pcv=pcv, ctx=ctx, base=base, writers=writers, tree=tree)
    tree.free()
    s2.free()
    ctx.close()


def _sub_roots(s, write, tmp, L, own_every=2, **kw):
    """Every sub-root at level L: even indices into directories of their own, odd ones into one shared directory."""
    os.makedirs(tmp, exist_ok=True)
    shared = os.path.join(tmp, "shared")
    dirs = [shared]
    for i in range(4 ** L):
        d = os.path.join(tmp, "own%d" % i) if i % own_every == 0 else shared
        write(d, root=(L, i), **kw)
        if d not in dirs:
            dirs.append(d)
    return dirs


def _pngs(d):
    return sorted(f for f in os.listdir(d) if f.endswith(".png"))


def _read(path):
    return np.asarray(Image.open(path).convert("RGBA"))


def _meta(d, name="meta.pb"):
    return R.read_meta(open(os.path.join(d, name), "rb").read())


def _check_against_ref(merged, inputs, bg):
    meta, parents = R.merge(inputs, bg)
    got = _meta(merged)
    assert sorted(set(got.nodes)) == meta[6]
    assert (got.deepest, got.tile) == meta[1:3]
    assert [v.hex() for v in got.rect] == [v.hex() for v in meta[3]]
    for (l, i), want in parents.items():
        assert np.array_equal(_read(os.path.join(merged, R.node_name(l, i) + ".png")), want), (l, i)
    return meta


@pytest.mark.parametrize("source", ["octree", "s2", "dirs"])
@pytest.mark.parametrize("L", [1, 2])
def test_merge_equals_full_build(scene, source, L, tmp_path):
    s, write = scene, scene["writers"][source]
    full = str(tmp_path / "full")
    write(full)
    inputs = _sub_roots(s, write, str(tmp_path), L)
    out = str(tmp_path / "merged")
    info = s["ctx"].merge_xray_quadtrees(inputs, out)
    full_meta = _meta(full)
    assert info["root_level"] == L and info["deepest_level"] == full_meta.deepest and info["tile_size_px"] == T
    assert info["metas_read"] == 4 ** L and (info["metas_empty"] > 0 or source == "s2")
    assert info["peak_device_bytes"] <= info["device_bytes_needed"] <= info["max_device_bytes"]
    assert _pngs(out) == _pngs(full)
    for f in _pngs(full):
        assert np.array_equal(_read(os.path.join(out, f)), _read(os.path.join(full, f))), f
    got = _meta(out)
    assert set(got.nodes) == set(full_meta.nodes) and len(got.nodes) == len(set(got.nodes))
    assert (got.deepest, got.tile) == (full_meta.deepest, full_meta.tile)
    assert [v.hex() for v in got.rect] == [v.hex() for v in full_meta.rect]
    meta = _check_against_ref(out, inputs, WHITE)
    assert info["parents_built"] == len(meta[5]) and info["roots_decoded"] == len(meta[4])
    assert info["files_copied"] == sum(len(_pngs(d)) for d in inputs)


@pytest.mark.parametrize("strategy", [1, 2, 3])
def test_attribute_strategies_against_the_restatement(scene, strategy, tmp_path):
    kw = dict(strategy=strategy, p0=0.0, p1=1000.0) if strategy != 3 else dict(strategy=3, p0=2.0)
    write = lambda out, **k: scene["tree"].xray_quadtree_write_dir(out, T, PX, **kw, **k)  # noqa: E731
    inputs = _sub_roots(scene, write, str(tmp_path), 2)
    out = str(tmp_path / "merged")
    scene["ctx"].merge_xray_quadtrees(inputs, out)
    _check_against_ref(out, inputs, WHITE)


def test_transparent_output_in_input_and_new_directory(scene, tmp_path):
    s = scene
    write = s["writers"]["octree"]
    full = str(tmp_path / "full")
    write(full, background=TRANSPARENT)
    inputs = _sub_roots(s, lambda d, **kw: write(d, background=TRANSPARENT, **kw), str(tmp_path), 2)
    new = str(tmp_path / "does" / "not" / "exist")
    s["ctx"].merge_xray_quadtrees(inputs, new, background=TRANSPARENT)
    assert _pngs(new) == _pngs(full)
    for f in _pngs(full):
        assert np.array_equal(_read(os.path.join(new, f)), _read(os.path.join(full, f))), f
    # white parents over sub-roots built on a transparent background: only the missing children differ
    white = str(tmp_path / "white")
    s["ctx"].merge_xray_quadtrees(inputs, white, background=WHITE)
    _check_against_ref(white, inputs, WHITE)
    assert not np.array_equal(_read(os.path.join(white, "r.png")), _read(os.path.join(new, "r.png")))
    out = inputs[1]  # one input directory is the output: its images are not copied onto themselves
    info = s["ctx"].merge_xray_quadtrees(inputs, out, background=TRANSPARENT)
    assert info["files_copied"] == sum(len(_pngs(d)) for d in inputs if d != out)
    assert _pngs(out) == _pngs(full)
    for f in _pngs(full):
        assert np.array_equal(_read(os.path.join(out, f)), _read(os.path.join(new, f))), f


def test_single_level0_input_and_v2_metas(scene, tmp_path):
    s = scene
    one = str(tmp_path / "one")
    s["writers"]["octree"](one)
    out = str(tmp_path / "out")
    info = s["ctx"].merge_xray_quadtrees(one, out)
    assert info["root_level"] == 0 and info["parents_built"] == 0 and info["peak_device_bytes"] == 0
    assert _pngs(out) == _pngs(one)
    assert open(os.path.join(out, "meta.pb"), "rb").read() != b"" and set(_meta(out).nodes) == set(_meta(one).nodes)
    # version 2: the sub-roots' metas rewritten with only the deprecated f32 fields (the scene's rects are exact in f32)
    inputs = _sub_roots(s, s["writers"]["octree"], str(tmp_path / "v2"), 1)
    full = str(tmp_path / "full")
    s["writers"]["octree"](full)
    for d in inputs:
        for f in os.listdir(d):
            if f.startswith("meta") and f.endswith(".pb"):
                m = XrayMeta.FromString(open(os.path.join(d, f), "rb").read())
                r = m.bounding_rect
                x, y, e = r.min.x, r.min.y, r.edge_length
                assert struct.unpack("f", struct.pack("f", x))[0] == x and struct.unpack("f", struct.pack("f", e))[0] == e
                r.ClearField("min")
                r.ClearField("edge_length")
                r.deprecated_min.x, r.deprecated_min.y, r.deprecated_edge_length = x, y, e
                m.version = 2
                open(os.path.join(d, f), "wb").write(m.SerializeToString())
    out2 = str(tmp_path / "out2")
    s["ctx"].merge_xray_quadtrees(inputs, out2)
    assert [v.hex() for v in _meta(out2).rect] == [v.hex() for v in _meta(full).rect]
    assert _pngs(out2) == _pngs(full)


def test_1024_px_tiles(scene, tmp_path):
    tree = scene["tree"]
    write = lambda out, **kw: tree.xray_quadtree_write_dir(out, 1024, 0.05, **kw)  # noqa: E731
    full = str(tmp_path / "full")
    write(full)
    inputs = _sub_roots(scene, write, str(tmp_path), 1)
    out = str(tmp_path / "merged")
    scene["ctx"].merge_xray_quadtrees(inputs, out)
    for f in _pngs(full):
        assert np.array_equal(_read(os.path.join(out, f)), _read(os.path.join(full, f))), f


def test_budgets(scene, tmp_path):
    s = scene
    inputs = _sub_roots(s, s["writers"]["octree"], str(tmp_path), 2)
    outs = []
    need = None
    for k, budget in enumerate((0, 1 << 26, None)):
        out = str(tmp_path / ("m%d" % k))
        if budget is None:
            budget = need
        info = s["ctx"].merge_xray_quadtrees(inputs, out, max_device_bytes=budget)
        need = info["device_bytes_needed"]
        assert info["peak_device_bytes"] <= info["max_device_bytes"]
        outs.append(out)
    for f in _pngs(outs[0]):
        a = open(os.path.join(outs[0], f), "rb").read()
        assert all(open(os.path.join(o, f), "rb").read() == a for o in outs[1:]), f
    low = str(tmp_path / "low")
    with pytest.raises(s["pcv"].PcvError) as e:
        s["ctx"].merge_xray_quadtrees(inputs, low, max_device_bytes=need - 1)
    assert e.value.code == -6 and str(need) in str(e.value)
    assert not os.path.exists(os.path.join(low, "meta.pb")) and _pngs(low) == []


def test_errors(scene, tmp_path):
    s = scene
    pcv, ctx = s["pcv"], s["ctx"]
    base = str(tmp_path / "in")
    inputs = _sub_roots(s, s["writers"]["octree"], base, 1, own_every=1)

    def code(dirs, name):
        out = str(tmp_path / ("out_" + name))
        with pytest.raises(pcv.PcvError) as e:
            ctx.merge_xray_quadtrees(dirs, out)
        assert not os.path.exists(os.path.join(out, "meta.pb")), name
        return e.value.code

    assert code([str(tmp_path / "missing")], "missing") == -4
    afile = str(tmp_path / "afile")
    open(afile, "w").close()
    assert code([afile], "afile") == -1
    empty = str(tmp_path / "empty")
    os.makedirs(empty)
    assert code([empty], "nometa") == -4
    own = [d for d in inputs if os.path.isdir(d)]
    assert code(own + [own[1]], "twice") == -1  # the same root twice
    other = str(tmp_path / "other_level")
    s["writers"]["octree"](other, root=(2, 1))
    assert code(own + [other], "levels") == -1
    other_t = str(tmp_path / "other_tile")
    s["tree"].xray_quadtree_write_dir(other_t, 64, PX / 2, root=(1, 3))
    assert code(own[:3] + [other_t], "tiles") == -1
    bad = str(tmp_path / "badmeta")
    shutil.copytree(own[0], bad)
    metaf = [f for f in os.listdir(bad) if f.endswith(".pb")][0]
    open(os.path.join(bad, metaf), "wb").write(b"\x08\x04")  # version 4
    assert code([bad] + own[1:], "version") == -1
    # sub-root images: missing, corrupt, wrongly sized
    for name, fix, want in (("gone", lambda p: os.remove(p), -4), ("corrupt", lambda p: open(p, "r+b").write(b"\x89PNG\r\n\x1a\nxx"), -1),
                            ("size", lambda p: Image.new("RGBA", (T + 1, T + 1)).save(p), -1)):
        d = str(tmp_path / ("img_" + name))
        shutil.copytree(own[0], d)
        pngs = [f for f in os.listdir(d) if f.endswith(".png") and len(f) == len("r0.png")]
        assert pngs
        fix(os.path.join(d, pngs[0]))
        assert code([d] + own[1:], name) == want
