"""S2-cell clouds streamed straight to an S2 directory (pcv_s2_build_to_dir, pcv_s2_build_from_file_to_dir): every directory equals
the in-core build's write_dir file for file and byte for byte, meta.pb included, at every budget, split level, layout and
attribute set; plus errors, rewrites of an existing directory and the info counters."""
import os

import numpy as np
import pytest

import s2_api as S
from ply_util import write_ply

pytestmark = pytest.mark.gpu

SEED = 80293751232
# a budget that plans batches of about `b` host points (whole 4096-point granules; see csrc/s2_stream_plan.h)
BUDGET_PTS = lambda b: (2 << 20) + b * 262  # noqa: E731


def _files(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


def _points(n, seed=SEED):
    import point_cloud_viewer_b200 as pcv

    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, seed, 0, n)
    inten = ((np.arange(n) * 13) % 511).astype(np.float32)
    return x, y, z, rgb, inten


def _in_core(ctx, d, x, y, z, rgb, inten, level, stride=1, n=None):
    c = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=level, stride=stride, n=n)
    c.write_dir(d)
    c.free()
    return _files(d)


def _check_info(info, n, files, budget):
    assert info["num_points"] == n and info["num_cells"] == sum(f.endswith(".xyz") for f in files)
    assert info["batches"] == -(-n // info["largest_batch"])
    assert info["bytes_written"] == sum(len(v) for f, v in files.items() if f != "meta.pb")
    if budget:
        assert info["max_device_bytes"] == budget and info["peak_device_bytes"] <= budget
    assert info["ms_total"] > 0 and info["ms_split"] > 0


@pytest.mark.parametrize("level", [10, 20, 30])
def test_stream_equals_in_core_soa_aos_pageable_pinned(ctx, tmp_path, level):
    import torch

    n = 300_000 if level < 30 else 20_000
    x, y, z, rgb, inten = _points(n)
    want = _in_core(ctx, str(tmp_path / "ref"), x, y, z, rgb, inten, level)
    P = np.ascontiguousarray(np.stack([x, y, z], 1))
    pinned = {k: torch.from_numpy(v).pin_memory() for k, v in (("x", x), ("y", y), ("z", z), ("rgb", rgb), ("i", inten), ("P", P))}
    budgets = [0, BUDGET_PTS(-(-n // 8)), BUDGET_PTS(4096)]
    for bi, budget in enumerate(budgets):
        for layout in ("soa", "aos", "soa_pinned", "aos_pinned"):
            if bi == 2 and layout != "soa":
                continue
            d = str(tmp_path / ("s%d_%s" % (bi, layout)))
            if layout == "soa":
                info = ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=level, max_device_bytes=budget)
            elif layout == "aos":
                info = ctx.build_s2_dir(d, P.ctypes.data, P.ctypes.data + 8, P.ctypes.data + 16, rgb, inten, split_level=level, max_device_bytes=budget,
                                        stride=3, n=n)
            else:
                t = pinned
                if layout == "soa_pinned":
                    info = ctx.build_s2_dir(d, t["x"].data_ptr(), t["y"].data_ptr(), t["z"].data_ptr(), t["rgb"].data_ptr(), t["i"].data_ptr(),
                                            split_level=level, max_device_bytes=budget, n=n)
                else:
                    p0 = t["P"].data_ptr()
                    info = ctx.build_s2_dir(d, p0, p0 + 8, p0 + 16, t["rgb"].data_ptr(), t["i"].data_ptr(), split_level=level, max_device_bytes=budget,
                                            stride=3, n=n)
            got = _files(d)
            assert got.keys() == want.keys(), (level, budget, layout)
            assert got == want, (level, budget, layout)
            _check_info(info, n, got, budget)
            assert info["h2d_bytes"] == n * 31 and info["d2h_bytes"] == n * 31
            if bi == 0:
                assert info["batches"] == 1
            elif bi == 1:
                assert (6 if n >= 8 * 8192 else 4) <= info["batches"] <= 10  # whole 4096-point granules
            else:  # batches of one or two granules
                assert info["largest_batch"] <= 8192 and info["batches"] >= n // 8192
                if level <= 20:  # every cell is appended to by several batches (at level 30 every point is its own cell)
                    assert info["file_writes"] > 3 * info["num_cells"]
                if level == 10:  # and the largest cell is larger than a batch
                    cells = ctx.load_s2_dir(d)
                    assert int(cells.cell_counts.max()) > info["largest_batch"]
                    cells.free()


@pytest.mark.parametrize("attrs", ["none", "rgb", "intensity"])
def test_stream_without_colour_or_intensity(ctx, tmp_path, attrs):
    n = 100_000
    x, y, z, rgb, inten = _points(n, SEED + 1)
    rgb = rgb if attrs == "rgb" else None
    inten = inten if attrs == "intensity" else None
    want = _in_core(ctx, str(tmp_path / "ref"), x, y, z, rgb, inten, 20)
    for budget in (0, BUDGET_PTS(16384)):
        d = str(tmp_path / ("s%d" % budget))
        info = ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=20, max_device_bytes=budget)
        got = _files(d)
        assert got == want
        _check_info(info, n, got, budget)
        per = 24 + (3 if rgb is not None else 0) + (4 if inten is not None else 0)
        assert info["h2d_bytes"] == n * per and info["file_writes"] >= info["num_cells"]


def test_stream_against_the_oracle_split_and_queries(ctx, tmp_path):
    """test_zz3's checks against the oracle's S.split, on a streamed directory, independently of the in-core build."""
    import point_cloud_viewer_b200 as pcv
    from proto_meta import Meta

    n = 60_000
    x, y, z, rgb, inten = _points(n)
    P = np.stack([x, y, z], 1)
    rgb3 = rgb.reshape(-1, 3)
    want = S.split(P, 21)
    d = str(tmp_path / "s2")
    ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=21, max_device_bytes=BUDGET_PTS(8192))
    m = Meta.FromString(open(os.path.join(d, "meta.pb"), "rb").read())
    assert m.version == 13 and m.WhichOneof("data") == "s2"
    assert {c.id: c.num_points for c in m.s2.cells} == {int(i): int(c) for i, c in zip(want["ids"], want["counts"])}
    bb = m.bounding_box
    assert [bb.min.x, bb.min.y, bb.min.z] == list(want["bmin"]) and [bb.max.x, bb.max.y, bb.max.z] == list(want["bmax"])
    assert set(os.listdir(d)) == {"meta.pb"} | {pcv.s2_token(i) + e for i in want["ids"] for e in (".xyz", ".rgb", ".intensity")}
    o = 0
    for cid, cnt in zip(want["ids"], want["counts"]):
        idx = want["order"][o:o + int(cnt)].astype(np.int64)
        o += int(cnt)
        stem = os.path.join(d, S.token(cid))
        assert np.array_equal(np.fromfile(stem + ".xyz", "<f8").reshape(-1, 3), P[idx])
        assert np.array_equal(np.fromfile(stem + ".rgb", np.uint8).reshape(-1, 3), rgb3[idx])
        assert np.array_equal(np.fromfile(stem + ".intensity", "<f4"), inten[idx])
    back = ctx.load_s2_dir(d)
    cloud = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=21)
    centre = int(S.oracle_cell_ids(P[n // 2:n // 2 + 1], 20)[0])
    u = np.array([centre, S.orc().orc_s2_next(centre)], np.uint64)
    a, b = cloud.query_union(u), back.query_union(u)
    assert a["total"] == b["total"] > 0 and all(np.array_equal(a[k], b[k]) for k in ("xyz", "rgb", "intensity"))
    back.free()
    cloud.free()


PLY_LAYOUTS = [
    [("float", "x"), ("float", "y"), ("float", "z"), ("uchar", "red"), ("uchar", "green"), ("uchar", "blue")],
    [("double", "x"), ("double", "y"), ("double", "z"), ("uchar", "r"), ("uchar", "g"), ("uchar", "b"), ("uchar", "alpha"), ("float", "intensity")],
    [("uchar", "red"), ("short", "junk"), ("float", "z"), ("uchar", "green"), ("int", "y"), ("ushort", "x"), ("uchar", "blue"), ("float", "intensity")],
    [("int", "x"), ("int", "y"), ("double", "z")],
]


@pytest.mark.parametrize("li", range(len(PLY_LAYOUTS)))
def test_ply_stream_equals_in_core_build_of_the_file(ctx, tmp_path, li):
    rng = np.random.default_rng(li)
    n = 150_000
    props = PLY_LAYOUTS[li]
    path = str(tmp_path / "p.ply")
    from ply_util import NP_TYPES

    # coordinates within 100 m of the offset, in each property's own type
    cols = {nm: (rng.random(n) * 100).astype(NP_TYPES[t]) for t, nm in props if nm in ("x", "y", "z")}
    write_ply(path, n, props, rng, offset=(4.2e6, 6.6e5, 4.75e6), comments=("made by a test",), columns=cols)
    pp = ctx.load_ply(path)
    c = ctx.build_s2_cloud(pp.x.ptr, pp.y.ptr, pp.z.ptr, pp.rgb.ptr if pp.rgb else None, pp.intensity.ptr if pp.intensity else None, split_level=20,
                           n=n, device=True)
    ref = str(tmp_path / "ref")
    c.write_dir(ref)
    c.free()
    want = _files(ref)
    for budget in (0, 16 << 20):
        d = str(tmp_path / ("s%d" % budget))
        info = ctx.build_s2_dir_from_file(path, d, split_level=20, max_device_bytes=budget)
        got = _files(d)
        assert got == want, (li, budget)
        _check_info(info, n, got, budget)
        assert info["h2d_bytes"] == n * int(pp.info.record_bytes)
        if budget:
            assert info["batches"] > 1
    # a truncated body: PCV_ERR_IO and no meta.pb
    import point_cloud_viewer_b200 as pcv

    cut = str(tmp_path / "cut.ply")
    write_ply(cut, 1000, props, rng, body_cut=7)
    d = str(tmp_path / "cut")
    with pytest.raises(pcv.PcvError) as e:
        ctx.build_s2_dir_from_file(cut, d)
    assert e.value.code == -3 and "truncated" in str(e.value)
    assert not os.path.exists(os.path.join(d, "meta.pb"))


def test_errors_invalid_nan_empty_budget(ctx, tmp_path):
    import point_cloud_viewer_b200 as pcv

    n = 50_000
    x, y, z, rgb, inten = _points(n)
    # an invalid point in a late batch: the in-core message, and no meta.pb even where the directory held one
    bad = x.copy()
    bad[n - 100] = 1.0
    by, bz = y.copy(), z.copy()
    by[n - 100] = 2.0
    bz[n - 100] = 3.0
    with pytest.raises(pcv.PcvError) as e_ref:
        ctx.build_s2_cloud(bad, by, bz, rgb, inten, split_level=20)
    d = str(tmp_path / "bad")
    ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=20)
    assert os.path.exists(os.path.join(d, "meta.pb"))
    with pytest.raises(pcv.PcvError) as e:
        ctx.build_s2_dir(d, bad, by, bz, rgb, inten, split_level=20, max_device_bytes=BUDGET_PTS(8192))
    assert str(e.value) == str(e_ref.value) and "is not a valid ECEF point" in str(e.value)
    assert not os.path.exists(os.path.join(d, "meta.pb"))
    # a NaN position passes the radius check in both
    nx = x.copy()
    nx[n // 3] = np.nan
    want = _in_core(ctx, str(tmp_path / "nan_ref"), nx, y, z, rgb, inten, 20)
    ctx.build_s2_dir(str(tmp_path / "nan"), nx, y, z, rgb, inten, split_level=20, max_device_bytes=BUDGET_PTS(8192))
    assert _files(str(tmp_path / "nan")) == want
    # empty input: the in-core error, and nothing written
    e0 = ctx.build_s2_cloud(x[:0], y[:0], z[:0], split_level=20)
    with pytest.raises(pcv.PcvError) as e_ref:
        e0.write_dir(str(tmp_path / "e_ref"))
    e0.free()
    with pytest.raises(pcv.PcvError) as e:
        ctx.build_s2_dir(str(tmp_path / "empty"), x[:0], y[:0], z[:0], split_level=20)
    assert str(e.value) == str(e_ref.value) and not os.path.exists(tmp_path / "empty")
    # arguments and budget
    with pytest.raises(pcv.PcvError) as e:
        ctx.build_s2_dir(str(tmp_path / "l31"), x, y, z, split_level=31)
    assert e.value.code == -1
    with pytest.raises(pcv.PcvError) as e:
        ctx.build_s2_dir(str(tmp_path / "small"), x, y, z, rgb, inten, max_device_bytes=1 << 20)
    assert e.value.code == -6 and "cannot hold one batch" in str(e.value) and str(1 << 20) in str(e.value)


def test_rewrite_of_a_larger_cloud(ctx, tmp_path):
    x, y, z, rgb, inten = _points(200_000, SEED + 7)
    d = str(tmp_path / "d")
    ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=20)
    m = 50_000
    want = _in_core(ctx, str(tmp_path / "ref"), x[:m], y[:m], z[:m], rgb[:3 * m], inten[:m], 20)
    ctx.build_s2_dir(d, x[:m], y[:m], z[:m], rgb[:3 * m], inten[:m], split_level=20, max_device_bytes=BUDGET_PTS(8192))
    got = _files(d)
    for f, v in want.items():
        assert got[f] == v, f
    back = ctx.load_s2_dir(d)
    assert back.num_points == m
    back.free()


def test_at_scale_many_batches(ctx, tmp_path):
    n = 200_000_000
    x, y, z, rgb = _points(n)[:4]
    ref, d = str(tmp_path / "ref"), str(tmp_path / "s")
    want_cloud = ctx.build_s2_cloud(x, y, z, rgb, None, split_level=20)
    want_cloud.write_dir(ref)
    want_cloud.free()
    info = ctx.build_s2_dir(d, x, y, z, rgb, None, split_level=20, max_device_bytes=4 << 30)
    assert info["batches"] >= 8 and info["peak_device_bytes"] <= 4 << 30
    a, b = sorted(os.listdir(ref)), sorted(os.listdir(d))
    assert a == b
    for f in a:
        with open(os.path.join(ref, f), "rb") as fa, open(os.path.join(d, f), "rb") as fb:
            while True:
                ca, cb = fa.read(1 << 26), fb.read(1 << 26)
                assert ca == cb, f
                if not ca:
                    break
