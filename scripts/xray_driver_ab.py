"""A/B of two builds of the library on the bounded X-ray quadtree driver, e.g. a build of the parent commit against the tree's
own: every source (resident octree, octree directory, several octree directories, S2 cloud, one or several S2 directories) on the
seeded scenes of its GPU tests, at the smallest and the default budgets those tests use and, for the directory lists, budgets
that make the windows reuse the previous block's nodes, all four strategies with and without query_from_global, a sub-root, a run cancelled from
on_tile, budgets too small to run and write_dir.  Each library runs in its own process.  Every tile is hashed as it is
delivered, so the two runs must agree on every tile's bytes and on the delivery order; they must also agree on every field of
the info dict except the ms_* timings, on every error's code and message, and on every file write_dir writes.  Library A runs
twice: a case whose tiles differ between those two runs (the float atomics of XRAY_COLORED's sums) has to agree on everything
but the tile bytes.

    python scripts/xray_driver_ab.py --lib-a /path/to/parent/libpcv_b200.so [--lib-b in-tree] [--out result.json]
"""
import argparse
import hashlib
import json
import os
import pickle
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WHITE, TRANSPARENT = (255, 255, 255, 255), (255, 255, 255, 0)


def record(fn, *a, cancel_after=0, **kw):
    """The delivered tiles (level, index, sha256) in order, the info dict without its timings, or the error."""
    from point_cloud_viewer_b200 import _native as N

    order = []

    def on_tile(level, index, img):
        order.append((level, index, hashlib.sha256(img.tobytes()).hexdigest()))
        return cancel_after and len(order) >= cancel_after

    try:
        info, _ = fn(*a, on_tile=on_tile, keep_tiles=False, **kw)
        return dict(order=order, info={k: v for k, v in info.items() if not k.startswith("ms_")})
    except N.PcvError as e:
        return dict(order=order, error=(e.code, str(e)))


def record_dir(fn, *a, **kw):
    """write_dir into a fresh directory: the info dict without its timings and the sha256 of every file, or the error."""
    from point_cloud_viewer_b200 import _native as N

    with tempfile.TemporaryDirectory() as d:
        try:
            info = fn(d, *a, **kw)
        except N.PcvError as e:
            return dict(error=(e.code, str(e)))
        files = {f: hashlib.sha256(open(os.path.join(d, f), "rb").read()).hexdigest() for f in sorted(os.listdir(d))}
    return dict(files=files, info={k: v for k, v in info.items() if not k.startswith("ms_")})


def strategies(pcv):
    return {"xray": {}, "colored": dict(strategy=pcv.XRAY_COLORED), "intensity": dict(strategy=pcv.XRAY_INTENSITY, p0=0.0, p1=1000.0),
            "intensity_binned": dict(strategy=pcv.XRAY_INTENSITY, p0=0.0, p1=1000.0, bin_size=20.0),
            "stddev": dict(strategy=pcv.XRAY_HEIGHT_STDDEV, p0=1.5, colormap=1)}


def slab_qfg(pcv):
    G = pcv.geometry
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    return list(G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7())


def octree_cases(pcv, out, tmp):
    """test_xray_bounded_gpu.py's and test_xray_dir_gpu.py's scene: 1.5e5 slab points, 4000 per node, with intensity."""
    import numpy as np

    n = 150_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    inten = ((np.arange(n) * 7919) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    ctx = pcv.Context(0, max_points_per_node=4000)
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    d = os.path.join(tmp, "octree")
    os.makedirs(d)
    tree.write_dir(d)
    ext = float(max(bmax[0] - bmin[0], bmax[1] - bmin[1]))
    qfg = slab_qfg(pcv)
    octree_bytes = int(tree.xyz_bytes) + 3 * n
    from_dir = lambda *a, **kw: ctx.xray_quadtree_from_dir(d, *a, **kw)

    def smallest(T, px, **kw):  # test_xray_dir_gpu.py's scan upwards from an eighth of the octree's bytes; every attempt is recorded
        b = octree_bytes // 8
        while b < 64 << 20:
            r = out["dir/scan/%s/%d" % (json.dumps(kw, sort_keys=True), b)] = record(from_dir, T, px, max_device_bytes=b, **kw)
            if "error" not in r:
                return b
            b = int(b * 1.2)
        return 0

    for T, depth in ((32, 4), (16, 5)):
        px = ext / (2 ** depth * T) * 1.01
        tile = T * T * 4
        for bg in (WHITE, TRANSPARENT):
            for budget in (tile * 90 + 600_000, tile * 300 + 2_000_000, 0):
                out["octree/T%d/bg%d/%d" % (T, bg[3], budget)] = record(tree.xray_quadtree, T, px, background=bg, max_device_bytes=budget)
            small = smallest(T, px, background=bg)
            for budget in (small, 2 * small, 4 * small, 0):
                out["dir/T%d/bg%d/%d" % (T, bg[3], budget)] = record(from_dir, T, px, background=bg, max_device_bytes=budget)
    T = 32
    for name, kw in strategies(pcv).items():
        for q in (None, qfg):
            px = 0.5 if q else ext / (4 * T) * 1.01
            kw2 = dict(kw, background=TRANSPARENT, query_from_global=q)
            for budget in (4 << 20, 24 << 20, 0):
                out["octree/%s/q%d/%d" % (name, q is not None, budget)] = record(tree.xray_quadtree, T, px, max_device_bytes=budget, **kw2)
            for budget in (smallest(T, px, **kw2), 24 << 20, 0):
                out["dir/%s/q%d/%d" % (name, q is not None, budget)] = record(from_dir, T, px, max_device_bytes=budget, **kw2)
    full = out["octree/xray/q1/0"]["order"]
    sub = sorted((l, i) for l, i, _ in full if l == 2)[0]
    for budget in (T * T * 4 * 90 + 600_000, 0):
        out["octree/subroot/%d" % budget] = record(tree.xray_quadtree, T, 0.5, query_from_global=qfg, root=sub, max_device_bytes=budget)
        out["dir/subroot/%d" % budget] = record(from_dir, T, 0.5, query_from_global=qfg, root=sub, max_device_bytes=budget)
    px = ext / (16 * T) * 1.01
    for k in (1, 5, 40):
        out["octree/cancel/%d" % k] = record(tree.xray_quadtree, T, px, cancel_after=k, max_device_bytes=T * T * 4 * 300 + 2_000_000)
        out["dir/cancel/%d" % k] = record(from_dir, T, px, cancel_after=k, max_device_bytes=4 << 20)
    out["octree/too_small"] = record(tree.xray_quadtree, T, px, max_device_bytes=T * T * 4 - 1)
    out["dir/too_small"] = record(from_dir, T, px, max_device_bytes=700_000)
    for budget in (T * T * 4 * 90 + 600_000, 0):
        out["octree/write_dir/%d" % budget] = record_dir(tree.xray_quadtree_write_dir, T, px, max_device_bytes=budget)
        out["dir/write_dir/%d" % budget] = record_dir(lambda o, *a, **kw: ctx.xray_quadtree_from_dir_write_dir(d, o, *a, **kw), T, px, max_device_bytes=budget)
    tree.free()
    ctx.close()


def s2_cases(pcv, out):
    """test_zz8_s2_xray_quadtree_gpu.py's scene: the 1e6-point slab split at level 20, 64 px tiles over five levels."""
    import numpy as np

    ctx = pcv.Context(0)
    n = 1_000_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    inten = np.random.default_rng(3).uniform(0.0, 100.0, n).astype(np.float32)
    cloud = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=20)
    d = cloud.bbox_max - cloud.bbox_min
    T, px, qfg = 64, float(max(d[0], d[1])) / (64 * 32), slab_qfg(pcv)
    for name, kw in strategies(pcv).items():
        for q in (None, qfg):
            for budget in (3 << 20, 0):
                out["s2/%s/q%d/%d" % (name, q is not None, budget)] = record(cloud.xray_quadtree, T, px, query_from_global=q, background=TRANSPARENT,
                                                                             max_device_bytes=budget, **kw)
    out["s2/subroot"] = record(cloud.xray_quadtree, T, px, query_from_global=qfg, root=(2, 6))
    out["s2/white"] = record(cloud.xray_quadtree, T, px, query_from_global=qfg)
    for f in ([(10.0, 60.0)], [(0.0, 20.0), (30.0, 40.0)]):
        out["s2/filters/%s" % f] = record(cloud.xray_quadtree, T, px, filter_intervals=f)
    out["s2/too_small"] = record(cloud.xray_quadtree, T, px, query_from_global=qfg, max_device_bytes=64 << 10)
    for budget in [int(v) for v in np.geomspace(16 << 10, 4 << 20, 40)]:  # test_budgets: the smallest budgets and several key batches
        out["s2/small/%d" % budget] = record(cloud.xray_quadtree, 16, px * 8, query_from_global=qfg, max_device_bytes=budget)
    for k in (1, 5, 40):
        out["s2/cancel/%d" % k] = record(cloud.xray_quadtree, T, px, cancel_after=k)
    for budget in (3 << 20, 0):
        out["s2/write_dir/%d" % budget] = record_dir(cloud.xray_quadtree_write_dir, T, px, query_from_global=qfg, max_device_bytes=budget)
    cloud.free()
    ctx.close()


def dirs_common(pcv, out, name, run, run_dir, T, px, qfg, filters):
    """The cases every list of directories runs: a budget scan, the strategies, a sub-root, filters, cancels, a budget too small
    and write_dir.  run(T, px, **kw) / run_dir(out_dir, T, px, **kw) call the entry over the scene's directories."""
    import numpy as np

    for b in [int(v) for v in np.geomspace(256 << 10, 48 << 20, 12)] + [0]:
        out["%s/scan/%d" % (name, b)] = record(run, T, px, query_from_global=qfg, max_device_bytes=b)
    for sname, kw in strategies(pcv).items():
        for budget in (3 << 20, 0):
            out["%s/%s/%d" % (name, sname, budget)] = record(run, T, px, background=TRANSPARENT, max_device_bytes=budget, **kw)
    for budget in (3 << 20, 0):
        out["%s/subroot/%d" % (name, budget)] = record(run, T, px, query_from_global=qfg, root=(1, 2), max_device_bytes=budget)
        out["%s/filters/%d" % (name, budget)] = record(run, T, px, filter_intervals=filters, max_device_bytes=budget)
    for k in (1, 5, 40):
        out["%s/cancel/%d" % (name, k)] = record(run, T, px, cancel_after=k, max_device_bytes=3 << 20)
    out["%s/too_small" % name] = record(run, T, px, max_device_bytes=64 << 10)
    for budget in (3 << 20, 0):
        out["%s/write_dir/%d" % (name, budget)] = record_dir(run_dir, T, px, query_from_global=qfg, max_device_bytes=budget)


def octree_dirs_cases(pcv, out, tmp):
    """test_zzf_xray_octree_dirs_gpu.py's four directories: two overlapping parts of the slab at 4000 and 1500 points per node,
    clusters beside it written by build_octree_to_dir at 2500, and a part of the slab without intensities."""
    import numpy as np

    n = 150_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    xyz = np.stack([x, y, z], 1)
    rgb = np.asarray(rgb).reshape(-1, 3)
    inten = ((np.arange(n) * 7919) % 1000).astype(np.float32)
    _, _, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    m = 40_000
    cx, cy, cz, crgb = pcv.synth_points_host(pcv.SYNTH_GAUSS_CLUSTERS, 7, 0, m)
    c = np.stack([cx, cy, cz], 1)
    c = (c - c.min(0)) / np.ptp(c, 0).max()
    ext = xyz.max(0) - xyz.min(0)
    cxyz = xyz.max(0) + np.array([0.05, -0.3, -0.5]) * ext + c * 0.4 * ext
    cinten = ((np.arange(m) * 31) % 1000).astype(np.float32)
    col = lambda p, k: np.ascontiguousarray(p[:, k])  # noqa: E731
    dirs = [os.path.join(tmp, "dirs_" + name) for name in ("a", "b", "c", "bare")]
    for d, (lo, hi), mppn, with_i in ((dirs[0], (0, 90_000), 4000, True), (dirs[1], (60_000, n), 1500, True), (dirs[3], (20_000, 70_000), 4000, False)):
        bc = pcv.Context(0, max_points_per_node=mppn)
        p = xyz[lo:hi]
        t = bc.build_octree(col(p, 0), col(p, 1), col(p, 2), rgb[lo:hi].reshape(-1).copy(), res, p.min(0), p.max(0),
                            intensity=inten[lo:hi].copy() if with_i else None)
        t.write_dir(d)
        t.free()
        bc.close()
    bc = pcv.Context(0, max_points_per_node=2500)
    bc.build_octree_to_dir(dirs[2], col(cxyz, 0), col(cxyz, 1), col(cxyz, 2), np.asarray(crgb).reshape(-1).copy(), res, cxyz.min(0), cxyz.max(0),
                           intensity=cinten, max_points_in_core=15_000)
    bc.close()
    ctx = pcv.Context(0)
    hs = [ctx.open_dir(d) for d in dirs[:3]]
    box = np.concatenate([np.min([h.bbox_min for h in hs], 0), np.max([h.bbox_max for h in hs], 0)])
    for h in hs:
        h.close()
    T = 32
    px = float(max(box[3] - box[0], box[4] - box[1])) / (T * 2 ** 5)
    for name, ds in (("dirs3", dirs[:3]), ("dirs4", dirs), ("dirs4_permuted", [dirs[k] for k in (3, 1, 0, 2)])):
        run = lambda *a, ds=ds, **kw: ctx.xray_quadtree_from_dirs(ds, *a, **kw)  # noqa: E731
        run_dir = lambda o, *a, ds=ds, **kw: ctx.xray_quadtree_from_dirs_write_dir(ds, o, *a, **kw)  # noqa: E731
        if name == "dirs4":  # intensity strategies and filters are refused with the directory without intensities
            out["%s/scan/0" % name] = record(run, T, px, query_from_global=slab_qfg(pcv), max_device_bytes=0)
            out["%s/scan/small" % name] = record(run, T, px, query_from_global=slab_qfg(pcv), max_device_bytes=3 << 20)
            out["%s/filters" % name] = record(run, T, px, filter_intervals=[(100.0, 600.0)])
            continue
        dirs_common(pcv, out, name, run, run_dir, T, px, slab_qfg(pcv), [(100.0, 600.0), (700.0, 800.0)])
    ctx.close()


def s2_dirs_cases(pcv, out, tmp):
    """test_zzc_s2_dir_xray_gpu.py's scene: the 1e6-point slab written with build_s2_dir at level 20, as one directory and as
    three overlapping parts."""
    import numpy as np

    ctx = pcv.Context(0)
    n = 1_000_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    rgb = np.asarray(rgb).reshape(-1, 3)
    inten = np.random.default_rng(3).uniform(0.0, 100.0, n).astype(np.float32)
    one = os.path.join(tmp, "s2_l20")
    ctx.build_s2_dir(one, x, y, z, rgb.reshape(-1).copy(), inten, split_level=20)
    parts = []
    for k, (a, b) in enumerate([(0, int(0.45 * n)), (int(0.3 * n), int(0.75 * n)), (int(0.6 * n), n)]):
        parts.append(os.path.join(tmp, "s2_part%d" % k))
        ctx.build_s2_dir(parts[-1], x[a:b].copy(), y[a:b].copy(), z[a:b].copy(), rgb[a:b].reshape(-1).copy(), inten[a:b].copy(), split_level=20)
    h = ctx.open_s2_dir(one)
    ext = h.bbox_max - h.bbox_min
    h.close()
    T = 64
    px = float(max(ext[0], ext[1])) / (T * 32)
    for name, ds in (("s2dir", [one]), ("s2dirs3", parts), ("s2dirs3_permuted", parts[::-1])):
        run = lambda *a, ds=ds, **kw: ctx.xray_quadtree_from_s2_dirs(ds, *a, **kw)  # noqa: E731
        run_dir = lambda o, *a, ds=ds, **kw: ctx.xray_quadtree_from_s2_dirs_write_dir(ds, o, *a, **kw)  # noqa: E731
        dirs_common(pcv, out, name, run, run_dir, T, px, slab_qfg(pcv), [(10.0, 60.0), (70.0, 80.0)])
    ctx.close()


def child(path):
    sys.path.insert(0, ROOT)
    import point_cloud_viewer_b200 as pcv

    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        octree_cases(pcv, out, tmp)
        octree_dirs_cases(pcv, out, tmp)
        s2_dirs_cases(pcv, out, tmp)
    s2_cases(pcv, out)
    with open(path, "wb") as f:
        pickle.dump(out, f)


def what_differs(x, y):
    """The parts of two records of one case that differ: the info fields (with both values), the tile bytes, the delivery order,
    the files, the error."""
    if not x or not y:
        return dict(missing="a" if not x else "b")
    out = {}
    xi, yi = x.get("info") or {}, y.get("info") or {}
    out.update({"info." + k: (xi.get(k), yi.get(k)) for k in sorted(set(xi) | set(yi)) if xi.get(k) != yi.get(k)})
    if [t[:2] for t in x.get("order", ())] != [t[:2] for t in y.get("order", ())]:
        out["order"] = True
    elif x.get("order") != y.get("order"):
        out["tile_bytes"] = True
    for k in ("files", "error"):
        if x.get(k) != y.get(k):
            out[k] = (str(x.get(k))[:200], str(y.get(k))[:200])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", required=True)
    ap.add_argument("--lib-b", default="in-tree")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args.child)
    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, lib in (("a", args.lib_a), ("b", args.lib_b), ("a2", args.lib_a)):
            env = dict(os.environ)
            if lib != "in-tree":
                env["PCV_B200_LIB"] = os.path.abspath(lib)
            p = os.path.join(tmp, name + ".pkl")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--lib-a", "-", "--child", p], env=env)
            with open(p, "rb") as f:
                runs[name] = pickle.load(f)
    a, b, a2 = runs["a"], runs["b"], runs["a2"]
    keys = set(a) | set(b) | set(a2)
    unstable = sorted(k for k in keys if a.get(k) != a2.get(k))
    shape = lambda r: r and dict(r, order=[(l, i) for l, i, _ in r.get("order", ())])  # without the tiles' bytes
    equal = [k for k in keys if a.get(k) == b.get(k)]
    differ = sorted(k for k in keys if a.get(k) != b.get(k) and (k not in unstable or shape(a.get(k)) != shape(b.get(k))))
    res = dict(cases=len(keys), equal=len(equal), unstable_in_a=len(unstable), unstable_equal_but_bytes=len(unstable) - len(set(unstable) & set(differ)),
               errors=sum("error" in v for v in a.values()), tiles=sum(len(v.get("order", v.get("files", ()))) for v in a.values()),
               unstable=unstable[:30], differ=differ[:20])
    for k in differ[:40]:
        res["diff/" + k] = what_differs(a.get(k), b.get(k))
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0 if not differ else 1


if __name__ == "__main__":
    sys.exit(main())
