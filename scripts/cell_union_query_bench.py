"""Octree queries by S2 cell union on the GPU: 1e8 config-1 slab points resident (SYNTH_SLAB_ECEF), unions of 1, 64 and 4096 cells.

Per union size one JSON line: ms_select and ms_cull of the batched form (pcv_last_query_stats, CUDA events; median of --reps),
tested and returned points, Gpoints/s tested in the cull, the wall time of the streaming form (pcv_query_cell_union, points to
the host), and the same run's baseline - the AllPoints stream to the host masked with pcv_s2_union_contains - with a parity
verdict.  Then one line for an octree directory of the same points (pcv_octree_dir_query_cell_union, pcv_octree_dir_last_stats).
Every line carries the card and its power limit, read in the same run.  Progress goes to stderr."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from xray_dir_bench import card  # noqa: E402

CENTRE = (4157222.543, 664789.307, 4774952.099)  # the slab's origin (csrc/synth.cuh)


def log(*a):
    print("[cell_union_query_bench]", *a, file=sys.stderr, flush=True)


def cat(batches, key):
    return np.concatenate([b[key] for b in batches]) if batches else np.zeros(0)


def unions_for(ctx, x, y, z, rng):
    """The slab spans ~240 m.  1 cell: the level-20 cell of its origin (the reference's own union, queries.rs:49-53, without the
    successor); 64 and 4096 cells: distinct level-22 / level-24 cells (~2 m / ~0.5 m) of sampled points."""
    c = np.array(CENTRE)
    out = {1: ctx.s2_cell_ids(c[:1].copy(), c[1:2].copy(), c[2:3].copy(), 20)}
    for k, level in ((64, 22), (4096, 24)):
        ids = np.zeros(0, np.uint64)
        for _ in range(20):
            pick = rng.integers(0, len(x), 4 * k)
            ids = np.unique(np.concatenate([ids, ctx.s2_cell_ids(x[pick], y[pick], z[pick], level)]))
            if len(ids) >= k:
                break
        if len(ids) < k:
            raise RuntimeError("only %d distinct level-%d cells found" % (len(ids), level))
        out[k] = rng.choice(ids, k, replace=False)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=float, default=1e8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--tmp", default=None)
    ap.add_argument("--no-dir", action="store_true")
    a = ap.parse_args()
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    name, power = card()
    n = int(a.points)
    ctx = pcv.Context(0)
    kind = pcv.SYNTH_SLAB_ECEF
    bmin, bmax, res = pcv.synth_bbox(kind)
    log("generating %d points on the host" % n)
    x, y, z, rgb = pcv.synth_points_host(kind, 80293751232, 0, n)
    t = time.perf_counter()
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax)
    log("built %d nodes in %.1f s" % (len(tree.meta), time.perf_counter() - t))
    rng = np.random.default_rng(1)
    unions = unions_for(ctx, x, y, z, rng)
    del x, y, z, rgb
    common = dict(card=name, power_limit=power, points=n, nodes=int(len(tree.meta)))
    # the baseline's first half does not depend on the union: one AllPoints stream to the host
    t = time.perf_counter()
    allb = tree.query_points(G.all_points(), batch_size=1 << 26)
    all_s = time.perf_counter() - t
    axyz, asrc = cat(allb, "xyz"), cat(allb, "src")
    del allb
    log("AllPoints stream: %.2f s" % all_s)
    for k, ids in unions.items():
        log("union of %d cells" % k)
        cu = G.cell_union(ids)
        stats = []
        for _ in range(a.reps):
            counts, tested = tree.query_batch_device([cu])
            stats.append(tree.last_query_stats())
        ms_sel = float(np.median([s["ms_select"] for s in stats]))
        ms_cull = float(np.median([s["ms_cull"] for s in stats]))
        t = time.perf_counter()
        got = tree.query_points(cu, batch_size=1 << 26)
        stream_s = time.perf_counter() - t
        t = time.perf_counter()
        keep = ctx.s2_union_contains(np.ascontiguousarray(axyz[:, 0]), np.ascontiguousarray(axyz[:, 1]), np.ascontiguousarray(axyz[:, 2]), ids)
        mask_s = time.perf_counter() - t
        parity = bool(np.array_equal(cat(got, "src"), asrc[keep]))
        out = dict(common, union_cells=k, ms_select=ms_sel, ms_cull=ms_cull, tested_points=int(tested[0]), returned_points=int(counts[0]),
                   gpoints_per_s_tested=(int(tested[0]) / (ms_cull * 1e-3) / 1e9) if ms_cull > 0 else None,
                   stream_s=stream_s, baseline_s=all_s + mask_s, baseline_all_points_s=all_s, baseline_mask_s=mask_s, parity=parity)
        print(json.dumps(out), flush=True)
    if not a.no_dir:
        tmp = tempfile.mkdtemp(prefix="cell_union_bench_", dir=a.tmp)
        try:
            d = os.path.join(tmp, "octree")
            t = time.perf_counter()
            tree.write_dir(d)
            log("wrote the directory in %.1f s" % (time.perf_counter() - t))
            h = pcv.OctreeDir(ctx, d)
            for k, ids in unions.items():
                cu = G.cell_union(ids)
                t = time.perf_counter()
                got = h.query_points(cu, batch_size=1 << 26)
                wall = time.perf_counter() - t
                st = h.last_stats()
                ref = tree.query_points(cu, batch_size=1 << 26)
                parity = bool(np.array_equal(cat(got, "xyz"), cat(ref, "xyz")))
                print(json.dumps(dict(common, directory=True, union_cells=k, wall_s=wall, parity=parity, **st)), flush=True)
            h.close()
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    tree.free()
    ctx.close()


if __name__ == "__main__":
    main()
