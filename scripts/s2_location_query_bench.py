"""Location queries of the S2-cell cloud on the GPU: 1e8 config-1 slab points (SYNTH_SLAB_ECEF) split at level 20 and resident.

One JSON line per query:
- the Aabb, Obb and Frustum of point_cloud_test/src/queries.rs: the batched form's ms_select / ms_cull (pcv_last_query_stats, CUDA
  events, median of --reps), tested and returned points, Gpoints/s tested in the cull, algorithmic_bytes / ms_cull against 3.35
  TB/s (HBM3 of the H100 SXM data sheet: 24 B per tested position dominate), the wall time of the stream to the host
  (pcv_s2_query_points) and two baselines of the same run: the host workaround (the AllPoints stream to the host, pcv_s2_query_union,
  then the oracle's point test, orc_location_contains_n, with a parity verdict) and the octree's batched query over the same points;
- bench.make_frusta frusta (1000 at far 10, 2000 at far 102.4) through pcv_s2_query_batch_device, with the octree's
  pcv_query_batch_device over the same frusta.
Every line carries the card and its power limit, read in the same run.  Progress goes to stderr."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import make_frusta  # noqa: E402
from xray_dir_bench import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, HBM3


def log(*a):
    print("[s2_location_query_bench]", *a, file=sys.stderr, flush=True)


def cat(batches, key):
    return np.concatenate([b[key] for b in batches]) if batches else np.zeros(0)


def batch_stats(q, locs, reps):
    """Median stats of `reps` batched calls (after one warm-up), with the counts of the last."""
    q.query_batch_device(locs[:1])
    stats = []
    for _ in range(reps):
        counts, tested = q.query_batch_device(locs)
        stats.append(q.last_query_stats())
    med = {k: float(np.median([s[k] for s in stats])) for k in ("ms_device", "ms_select", "ms_cull")}
    st = stats[-1]
    ms = med["ms_cull"]
    return dict(med, tested_points=int(tested.sum()), returned_points=int(counts.sum()), algorithmic_bytes=int(st["algorithmic_bytes"]),
                kernel_launches=int(st["kernel_launches"]),
                gpoints_per_s_tested=int(tested.sum()) / (ms * 1e-3) / 1e9 if ms > 0 else None,
                hbm_fraction=(st["algorithmic_bytes"] / (ms * 1e-3)) / HBM_BYTES_PER_S if ms > 0 else None), counts


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=float, default=1e8)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import oracle_api as O
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    name, power = card()
    n = int(a.points)
    ctx = pcv.Context(0)
    kind = pcv.SYNTH_SLAB_ECEF
    bmin, bmax, res = pcv.synth_bbox(kind)
    bmin, bmax = np.asarray(bmin, np.float64), np.asarray(bmax, np.float64)
    log("generating %d points on the host" % n)
    x, y, z, rgb = pcv.synth_points_host(kind, 80293751232, 0, n)
    t = time.perf_counter()
    cloud = ctx.build_s2_cloud(x, y, z, rgb, None, split_level=20)
    log("S2 cloud: %d cells in %.1f s (device %.1f ms)" % (cloud.num_cells, time.perf_counter() - t, cloud.build_stats()["ms_device"]))
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax)
    log("octree: %d nodes" % len(tree.meta))
    del x, y, z, rgb
    common = dict(card=name, power_limit=power, points=n, cells=int(cloud.num_cells), hbm_peak_bytes_per_s=HBM_BYTES_PER_S)
    d = bmax - bmin
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    ecef_from_local = G.Isometry((4157222.543, 664789.307, 4774952.099), q)
    shapes = {  # point_cloud_test/src/queries.rs at the slab pose
        "aabb": G.aabb(bmin + 0.2 * d, bmin + 0.8 * d),
        "obb": G.obb(ecef_from_local, (50.0, 50.0, 5.0)),
        "frustum": G.frustum(ecef_from_local, G.Perspective.new_fov(1.0, 1.2, 0.1, 10.0)),
    }
    # the host workaround's first half does not depend on the location: every point to the host once
    t = time.perf_counter()
    allp = cloud.query_union(None)
    all_s = time.perf_counter() - t
    log("AllPoints to the host: %.2f s" % all_s)
    for label, loc in shapes.items():
        log(label)
        st, counts = batch_stats(cloud, [loc], a.reps)
        t = time.perf_counter()
        got = cloud.query_points(loc, batch_size=1 << 26)
        stream_s = time.perf_counter() - t
        oloc = O.Location()
        for f, _ in O.Location._fields_:
            setattr(oloc, f, getattr(loc, f))
        t = time.perf_counter()
        keep = O.location_contains(oloc, allp["xyz"])
        mask_s = time.perf_counter() - t
        parity = bool(np.array_equal(cat(got, "src"), allp["src"][keep]) and int(counts[0]) == int(keep.sum()))
        oct_st, _ = batch_stats(tree, [loc], a.reps)
        print(json.dumps(dict(common, query=label, **st, stream_s=stream_s, host_workaround_s=all_s + mask_s, host_all_points_s=all_s,
                              host_point_test_s=mask_s, parity_with_host_workaround=parity,
                              octree_batch={k: oct_st[k] for k in ("ms_select", "ms_cull", "tested_points", "returned_points")})), flush=True)
    del allp
    for count, far in ((1000, 10.0), (2000, 102.4)):
        log("%d frusta, far %g" % (count, far))
        locs = make_frusta(G, bmin, bmax, count, far)
        st, _ = batch_stats(cloud, locs, a.reps)
        oct_st, _ = batch_stats(tree, locs, a.reps)
        print(json.dumps(dict(common, query="frusta", frusta=count, far=far, **st,
                              octree_batch={k: oct_st[k] for k in ("ms_device", "ms_select", "ms_cull", "tested_points", "returned_points",
                                                                   "gpoints_per_s_tested")})), flush=True)
    cloud.free()
    tree.free()
    ctx.close()


if __name__ == "__main__":
    main()
