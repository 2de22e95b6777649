"""Web Mercator rect queries on the GPU: 1e8 config-1 slab points (SYNTH_SLAB_ECEF) as a resident octree and as a resident S2
cloud (split level 20).

One JSON line per (zoom, number of locations, location kind, source): 1 and 1000 rects of 256 x 256 px at zoom 21, 19 and 17 whose
centres are slab points, and OBBs of the same footprints (centred on the rect's centre, east / north / up axes, half extents of
half the rect's metric width and height and 300 m, so that the box spans the tilted slab's column as the rect does), through the
batched form (query_batch_device).  Each line has ms_select and ms_cull (pcv_last_query_stats, CUDA events, median of --reps calls after one warm-up), the points tested and
returned, and Gpoints/s tested in the cull.  The rect's point test is an FP64 ECEF -> WGS84 -> Web Mercator conversion per point;
the OBB's is one rigid transform.  Every line carries the card and its power limit, read in the same run.  Progress goes to
stderr."""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from xray_dir_bench import card  # noqa: E402

WGS84_A = 6378137.0


def log(*a):
    print("[web_mercator_query_bench]", *a, file=sys.stderr, flush=True)


def batch_stats(q, locs, reps):
    q.query_batch_device(locs[:1])
    q.query_batch_device(locs)
    stats = []
    for _ in range(reps):
        counts, tested = q.query_batch_device(locs)
        stats.append(q.last_query_stats())
    med = {k: float(np.median([s[k] for s in stats])) for k in ("ms_select", "ms_cull")}
    ms = med["ms_cull"]
    return dict(med, tested_points=int(tested.sum()), returned_points=int(counts.sum()),
                gpoints_per_s_tested=int(tested.sum()) / (ms * 1e-3) / 1e9 if ms > 0 else None)


def enu_quaternion(lat, lng):
    """The unit quaternion (i, j, k, w) of the rotation whose columns are east, north and up at (lat, lng)."""
    sl, cl, so, co = math.sin(lat), math.cos(lat), math.sin(lng), math.cos(lng)
    m = np.array([[-so, -sl * co, cl * co], [co, -sl * so, cl * so], [0.0, cl, sl]])
    w = math.sqrt(max(0.0, 1.0 + m[0, 0] + m[1, 1] + m[2, 2])) / 2.0
    x = math.copysign(math.sqrt(max(0.0, 1.0 + m[0, 0] - m[1, 1] - m[2, 2])) / 2.0, m[2, 1] - m[1, 2])
    y = math.copysign(math.sqrt(max(0.0, 1.0 - m[0, 0] + m[1, 1] - m[2, 2])) / 2.0, m[0, 2] - m[2, 0])
    z = math.copysign(math.sqrt(max(0.0, 1.0 - m[0, 0] - m[1, 1] + m[2, 2])) / 2.0, m[1, 0] - m[0, 1])
    q = np.array([x, y, z, w])
    return q / np.linalg.norm(q)


def footprints(G, centres, zoom, half_px=128.0):
    """The rect of +-half_px around each centre's map position at `zoom`, and the OBB of its footprint."""
    rects, obbs = [], []
    for p in centres:
        c = np.array(G.web_mercator_coord(p, zoom))
        rects.append(G.web_mercator_rect(c - half_px, c + half_px, zoom))
        # geodetic latitude / longitude of the centre, and the metric size of the rect there (Mercator is conformal)
        lng = math.atan2(p[1], p[0])
        lat = math.atan2(p[2], math.hypot(p[0], p[1]) * (1.0 - 0.00669437999014))
        half_m = half_px * 2.0 * math.pi * WGS84_A * math.cos(lat) / float(256 << zoom)
        obbs.append(G.obb(G.Isometry(tuple(p), enu_quaternion(lat, lng)), (half_m, half_m, 300.0)))
    return rects, obbs


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=float, default=1e8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--many", type=int, default=1000)
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
    rng = np.random.default_rng(5)
    pick = rng.integers(0, n, a.many)
    centres = np.stack([x[pick], y[pick], z[pick]], 1)
    t = time.perf_counter()
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax)
    cloud = ctx.build_s2_cloud(x, y, z, rgb, None, split_level=20)
    log("octree and S2 cloud in %.1f s" % (time.perf_counter() - t))
    del x, y, z, rgb
    common = dict(card=name, power_limit=power, points=n)
    for zoom in (21, 19, 17):
        for count in (1, a.many):
            rects, obbs = footprints(G, centres[:count], zoom)
            for label, locs in (("web_mercator_rect", rects), ("obb", obbs)):
                for src, q in (("octree", tree), ("s2", cloud)):
                    log("zoom %d, %d x %s, %s" % (zoom, count, label, src))
                    print(json.dumps(dict(common, zoom=zoom, locations=count, location=label, source=src, **batch_stats(q, locs, a.reps))), flush=True)
    cloud.free()
    tree.free()
    ctx.close()


if __name__ == "__main__":
    main()
