"""A/B of two builds of the library on the directory query handles, e.g. a build of the parent commit against the tree's own:
OctreeDir and S2Dir on the seeded scenes of their GPU tests (test_octree_dir_query_gpu.py's 200k-point slab at 3000 points per
node; test_zzd_s2_dir_query_gpu.py's 1e6-point slab at split levels 20 and 10).  query_points over a box, a small box, an OBB,
frustums and a cell union, with and without filters, at the smallest budget each handle accepts (nodes and cells cut across
chunks), a few times it and 4 GiB; query_batch over the same locations, many frustums and cell unions; a batch too large
for the smallest budget.  Each library runs in its own process.  Every batch is hashed in delivery order (positions, colours,
intensities, slots), so the two runs must agree on every point, its batch and its order; they must also agree on every batched
count, on last_stats without the ms_* timings and on every error's code and message.

    python scripts/dir_query_ab.py --lib-a /path/to/parent/libpcv_b200.so [--lib-b in-tree] [--out result.json]
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


def stats(h):
    return {k: v for k, v in h.last_stats().items() if not k.startswith("ms_")}


def record(h, fn, *a, **kw):
    """fn's batches as (size, sha256 of every array) in order, or its (counts, tested) hashed, and the handle's stats; or the
    error."""
    from point_cloud_viewer_b200 import _native as N

    try:
        r = fn(*a, **kw)
    except N.PcvError as e:
        return dict(error=(e.code, str(e)))
    if isinstance(r, tuple):  # query_batch
        return dict(counts=hashlib.sha256(r[0].tobytes() + r[1].tobytes()).hexdigest(), total=int(r[0].sum()), stats=stats(h))
    batches = []
    for b in r:
        hs = hashlib.sha256()
        for k in ("xyz", "rgb", "intensity", "src"):
            hs.update(k.encode() + (b"-" if b[k] is None else b[k].tobytes()))
        batches.append((len(b["src"]), hs.hexdigest()))
    return dict(batches=batches, stats=stats(h))


def smallest_budget(open_fn):
    """The smallest budget the handle accepts within 1/64 (the tests' geometric scan)."""
    import point_cloud_viewer_b200 as pcv

    lo, hi = 1 << 10, 1 << 34
    while hi - lo > lo // 64:
        mid = int((lo * hi) ** 0.5)
        try:
            open_fn(mid).close()
            hi = mid
        except pcv.PcvError:
            lo = mid
    return hi


def frusta(G, bmin, bmax, count, far, seed=7):  # bench.make_frusta
    import numpy as np

    rng = np.random.default_rng(seed)
    persp = G.Perspective.new_fov(1.0, 1.2, 0.1, far)
    out = []
    for _ in range(count):
        eye = bmin + rng.random(3) * (bmax - bmin)
        q = rng.random((4, 12)).sum(1) - 6.0
        out.append(G.frustum(G.Isometry(eye, q / np.linalg.norm(q)), persp))
    return out


def locations(G, bmin, bmax, ids):
    d = bmax - bmin
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    e = G.Isometry((4157222.543, 664789.307, 4774952.099), q)
    return {
        "all": G.all_points(),
        "aabb": G.aabb(bmin + 0.2 * d, bmin + 0.8 * d),
        "aabb_small": G.aabb(bmin + 0.45 * d, bmin + 0.47 * d),
        "obb": G.obb(e, (50.0, 50.0, 5.0)),
        "obb_tilted": G.obb(e * G.Isometry((10, -20, 1), G.quat_from_axis_angle([0.2, 0.5, -0.7], 0.523)), (30.0, 12.0, 4.0)),
        "frustum": G.frustum(e, G.Perspective.new_fov(1.0, 1.2, 0.1, 10.0)),
        "frustum_far": G.frustum(e * G.Isometry((0, 0, 0), G.quat_from_axis_angle([1, 0.3, 0], 1.3)), G.Perspective.new_fov(1.3, 0.9, 0.5, 150.0)),
        # a level-20 cell and a level-14 ancestor of another, and a level-25 descendant (point tests)
        "union": G.cell_union([int(ids[len(ids) // 3]), (int(ids[len(ids) // 2]) & ~((1 << 33) - 1)) | (1 << 32)]),
        "union_fine": G.cell_union([(int(ids[7]) & ~((1 << 11) - 1)) | (1 << 10)]),
    }


def handle_cases(out, name, open_fn, G, bmin, bmax, ids, filt):
    locs = locations(G, bmin, bmax, ids)
    unions = [G.cell_union([int(ids[k])]) for k in range(0, len(ids), max(1, len(ids) // 40))] + [locs["union"], G.cell_union([])]
    small = smallest_budget(open_fn)
    for budget in (small, 3 * small, 40 * small, 4 << 30):  # explicit budgets: the default one follows the device's free memory
        h = open_fn(budget)
        for key, loc in locs.items():
            for filters in ((), filt):
                out["%s/%d/points/%s/%s" % (name, budget, key, filters)] = record(h, h.query_points, loc, filters=filters, batch_size=7777)
        out["%s/%d/points/one" % (name, budget)] = record(h, h.query_points, locs["aabb_small"], batch_size=1)
        for bname, batch in (("locs", [v for k, v in locs.items() if not k.startswith("union")]), ("frusta64", frusta(G, bmin, bmax, 64, 60.0)), ("frusta2000", frusta(G, bmin, bmax, 2000, 60.0)),
                             ("unions", unions)):
            for filters in ((), filt):
                out["%s/%d/batch/%s/%s" % (name, budget, bname, filters)] = record(h, h.query_batch, batch, filters=filters)
        h.close()


def child(path):
    sys.path.insert(0, ROOT)
    import numpy as np
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        n = 200_000
        x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
        inten = (np.arange(n) % 1000).astype(np.float32)
        bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
        c = pcv.Context(0, max_points_per_node=3000)
        d = os.path.join(tmp, "octree")
        os.makedirs(d)
        tree = c.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
        tree.write_dir(d)
        tree.free()
        s2 = os.path.join(tmp, "cells_for_unions")
        c.build_s2_dir(s2, x, y, z, rgb, inten, split_level=20)
        h = c.open_s2_dir(s2)
        ids = h.cell_ids.copy()
        h.close()
        handle_cases(out, "octree", lambda b: pcv.OctreeDir(c, d, b), G, np.asarray(bmin), np.asarray(bmax), ids, (100.0, 250.0))
        c.close()

        ctx = pcv.Context(0)
        n = 1_000_000
        x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
        inten = np.random.default_rng(3).uniform(0.0, 100.0, n).astype(np.float32)
        for lvl in (20, 10):
            d = os.path.join(tmp, "s2_l%d" % lvl)
            ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=lvl)
            h = ctx.open_s2_dir(d)
            bmin, bmax = h.bbox_min.copy(), h.bbox_max.copy()
            if lvl == 20:  # the cell unions of both levels are built from the level-20 cells, as the tests build them
                ids = h.cell_ids.copy()
            h.close()
            handle_cases(out, "s2_l%d" % lvl, lambda b, d=d: pcv.S2Dir(ctx, d, b), G, bmin, bmax, ids, [(10.0, 60.0)])
        ctx.close()
    with open(path, "wb") as f:
        pickle.dump(out, f)


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
        for name, lib in (("a", args.lib_a), ("b", args.lib_b)):
            env = dict(os.environ)
            if lib != "in-tree":
                env["PCV_B200_LIB"] = os.path.abspath(lib)
            p = os.path.join(tmp, name + ".pkl")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--lib-a", "-", "--child", p], env=env)
            with open(p, "rb") as f:
                runs[name] = pickle.load(f)
    a, b = runs["a"], runs["b"]
    keys = set(a) | set(b)
    differ = sorted(k for k in keys if a.get(k) != b.get(k))
    res = dict(cases=len(keys), equal=len(keys) - len(differ), errors=sum("error" in v for v in a.values()),
               batches=sum(len(v.get("batches", ())) for v in a.values()), points=sum(n for v in a.values() for n, _ in v.get("batches", ())),
               differ=differ[:20])
    for k in differ[:20]:
        x, y = a.get(k) or {}, b.get(k) or {}
        res["diff/" + k] = {f: (str(x.get(f))[:200], str(y.get(f))[:200]) for f in ("batches", "counts", "error") if x.get(f) != y.get(f)}
        res["diff/" + k].update({"stats." + f: (x["stats"].get(f), y["stats"].get(f)) for f in x.get("stats", {}) if x["stats"].get(f) != y.get("stats", {}).get(f)})
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0 if not differ else 1


if __name__ == "__main__":
    sys.exit(main())
