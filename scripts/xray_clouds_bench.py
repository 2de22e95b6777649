"""python scripts/xray_clouds_bench.py [--points N] [--clouds K] [--tile-px T] [--leaves-per-side L] [--repeats R]

The X-ray quadtree of several clouds at once against one cloud of the same points: N config-1 slab points (the ECEF slab
generator, seed 1; default 1e8) built as K resident octrees of N / K consecutive points each (default 4, each with its own box)
and as one octree on the union of their boxes, then Context.xray_quadtree_clouds over the K and over the one (the same quadtree
frame), with T-px tiles (default 256) in the slab's
local frame, at the pixel size that puts about L leaves (default 64) along the longer side of the local box.  The same for K
S2 clouds (level-20 cells) against one.  Prints one JSON line: per run the device ms of the leaves and of the parents, leaves,
tiles, points read (info.leaf_points), Gpoints/s read over the leaves' device time, peak device bytes and an all-tiles
checksum, as the median and the spread (min, max) over R calls (default 5) after one warm-up call; and the card's name and
power limit read in the same run.  Progress goes to stderr."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED = 1


def card():
    """(name, power limit) of GPU 0, read in the same run as the measurement."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:
        return None, "unknown (%s)" % str(e)[:80]


def log(*a):
    print("[xray_clouds_bench]", *a, file=sys.stderr, flush=True)


def measure(fn, repeats):
    """One warm-up call, then `repeats` calls: the median and spread of the device times, the counters and a tile checksum."""
    import numpy as np

    runs, sums = [], set()
    for r in range(repeats + 1):
        h = hashlib.sha256()

        def on_tile(level, index, img):
            h.update(bytes([level]) + int(index).to_bytes(8, "little") + img.tobytes())

        info = fn(on_tile)
        if r:
            runs.append(info)
            sums.add(h.hexdigest()[:16])
    leaves = np.array([i["ms_leaves"] for i in runs])
    parents = np.array([i["ms_parents"] for i in runs])
    i0 = runs[0]
    med = float(np.median(leaves))
    return dict(ms_leaves=round(med, 3), ms_leaves_min=round(float(leaves.min()), 3), ms_leaves_max=round(float(leaves.max()), 3),
                ms_parents=round(float(np.median(parents)), 3), ms_parents_min=round(float(parents.min()), 3), ms_parents_max=round(float(parents.max()), 3),
                leaves=i0["num_leaves"], tiles=i0["num_nodes"], points_read=i0["leaf_points"],
                gpoints_per_s_read=round(i0["leaf_points"] / max(med, 1e-9) / 1e6, 3), peak_device_bytes=max(i["peak_device_bytes"] for i in runs),
                blocks=i0["blocks_processed"], key_batches=i0["key_batches"], checksums=sorted(sums))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=100_000_000)
    ap.add_argument("--clouds", type=int, default=4)
    ap.add_argument("--tile-px", type=int, default=256)
    ap.add_argument("--leaves-per-side", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch

    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    n, T, K = a.points, a.tile_px, a.clouds
    kind = pcv.SYNTH_SLAB_ECEF
    _, _, res = pcv.synth_bbox(kind)
    ctx = pcv.Context(0)
    x, y, z = (torch.empty(n, dtype=torch.float64, device="cuda") for _ in range(3))
    rgb = torch.empty(3 * n, dtype=torch.uint8, device="cuda")
    ctx.synth_points_device(kind, SEED, 0, n, x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr())
    log("%d points generated" % n)
    cuts = [n * k // K for k in range(K + 1)]
    parts = []
    for lo, hi in zip(cuts, cuts[1:]):
        pmin = np.array([float(v[lo:hi].min()) for v in (x, y, z)])
        pmax = np.array([float(v[lo:hi].max()) for v in (x, y, z)])
        ptr = lambda t, size: t.data_ptr() + size * lo
        parts.append((ptr(x, 8), ptr(y, 8), ptr(z, 8), ptr(rgb, 3), hi - lo, pmin, pmax))
    out = dict(points=n, clouds=K, tile_px=T)
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    local_from_ecef = G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse()  # the slab's local frame (csrc/synth.cuh)
    kw = dict(query_from_global=list(local_from_ecef.as7()), keep_tiles=False)

    def pixel_size(clouds):
        lo = np.min([c.bbox_min for c in clouds], 0)
        hi = np.max([c.bbox_max for c in clouds], 0)
        corners = [[(hi if k & (1 << ax) else lo)[ax] for ax in range(3)] for k in range(8)]
        local = np.array([local_from_ecef.transform_point(np.array(c)) for c in corners])
        return float(max(np.ptp(local[:, 0]), np.ptp(local[:, 1]))) / (T * a.leaves_per_side) * 1.01

    for what in ("octree", "s2"):
        if what == "octree":
            many = [ctx.build_octree(px_, py_, pz_, pc_, res, pmin, pmax, n=m, device=True) for px_, py_, pz_, pc_, m, pmin, pmax in parts]
            # on the union of the parts' boxes, so that both runs lay the quadtree over the same box
            umin, umax = np.min([p[5] for p in parts], 0), np.max([p[6] for p in parts], 0)
            one = [ctx.build_octree(x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr(), res, umin, umax, n=n, device=True)]
        else:
            many = [ctx.build_s2_cloud(px_, py_, pz_, pc_, None, split_level=20, n=m, device=True) for px_, py_, pz_, pc_, m, _, _ in parts]
            one = [ctx.build_s2_cloud(x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr(), None, split_level=20, n=n, device=True)]
        log("%s: %d clouds and one built" % (what, K))
        px = pixel_size(one)
        res_many = measure(lambda cb: ctx.xray_quadtree_clouds(many, T, px, on_tile=cb, **kw)[0], a.repeats)
        res_one = measure(lambda cb: ctx.xray_quadtree_clouds(one, T, px, on_tile=cb, **kw)[0], a.repeats)
        out[what] = dict(pixel_size_m=px, many=res_many, one=res_one)
        log(what, json.dumps(out[what]))
        for c in many + one:
            c.free()
        torch.cuda.empty_cache()
    out["gpu"], out["power_limit"] = card()
    print(json.dumps(out), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
