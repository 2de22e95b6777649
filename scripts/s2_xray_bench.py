"""python scripts/s2_xray_bench.py [--points N] [--tile-px T] [--leaves-per-side L] [--repeats R]

The X-ray quadtree of an S2 cloud at scale: N config-1 slab points (the ECEF slab generator, seed 1; default 1e8) split into
level-20 cells on the device, then S2Cloud.xray_quadtree with T-px tiles (default 256) in the slab's local frame
(query_from_global), at the pixel size that puts about L leaves (default 64) along the longer side of the local box.  Prints
one JSON line: device ms of the leaves and of the parents, leaves, tiles and points read (info.leaf_points), Gpoints/s read
over the leaves' device time, the peak of the call's device memory and an all-tiles checksum; beside it, for scale only, the
same quadtree parameters through Octree.xray_quadtree over an octree of the same points (its positions are quantised, so its
tiles differ); and the card's name and power limit read in the same run.  The best of R calls (default 3) after one warm-up
call is reported.  Progress goes to stderr."""
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
    print("[s2_xray_bench]", *a, file=sys.stderr, flush=True)


def measure(fn, repeats):
    """One warm-up call, then the call with the least leaf + parent device time of `repeats`; (info, checksum)."""
    best = None
    for r in range(repeats + 1):
        h = hashlib.sha256()

        def on_tile(level, index, img):
            h.update(bytes([level]) + int(index).to_bytes(8, "little") + img.tobytes())

        info = fn(on_tile)
        if r and (best is None or info["ms_leaves"] + info["ms_parents"] < best[0]["ms_leaves"] + best[0]["ms_parents"]):
            best = (info, h.hexdigest()[:16])
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=100_000_000)
    ap.add_argument("--tile-px", type=int, default=256)
    ap.add_argument("--leaves-per-side", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch

    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    n, T = a.points, a.tile_px
    kind = pcv.SYNTH_SLAB_ECEF
    bmin, bmax, res = pcv.synth_bbox(kind)
    ctx = pcv.Context(0)
    x, y, z = (torch.empty(n, dtype=torch.float64, device="cuda") for _ in range(3))
    rgb = torch.empty(3 * n, dtype=torch.uint8, device="cuda")
    ctx.synth_points_device(kind, SEED, 0, n, x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr())
    log("%d points generated" % n)
    cloud = ctx.build_s2_cloud(x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr(), None, split_level=20, n=n, device=True)
    log("S2 cloud: %d cells" % cloud.num_cells)
    tree = ctx.build_octree(x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr(), res, bmin, bmax, n=n, device=True)
    log("octree built")
    del x, y, z, rgb
    torch.cuda.empty_cache()
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    local_from_ecef = G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse()  # the slab's local frame (csrc/synth.cuh)
    qfg = list(local_from_ecef.as7())
    corners = [[(cloud.bbox_max if k & (1 << ax) else cloud.bbox_min)[ax] for ax in range(3)] for k in range(8)]
    local = np.array([local_from_ecef.transform_point(np.array(c)) for c in corners])
    extent = float(max(local[:, 0].max() - local[:, 0].min(), local[:, 1].max() - local[:, 1].min()))
    px = extent / (T * a.leaves_per_side) * 1.01
    kw = dict(query_from_global=qfg, keep_tiles=False)
    s2, s2_sum = measure(lambda cb: cloud.xray_quadtree(T, px, on_tile=cb, **kw)[0], a.repeats)
    log("S2 quadtree: %d tiles" % s2["num_nodes"])
    oc, oc_sum = measure(lambda cb: tree.xray_quadtree(T, px, on_tile=cb, **kw)[0], a.repeats)
    name, power = card()
    out = dict(
        points=n, tile_px=T, pixel_size_m=px, cells=cloud.num_cells, deepest_level=s2["deepest_level"],
        ms_leaves=round(s2["ms_leaves"], 3), ms_parents=round(s2["ms_parents"], 3), leaves=s2["num_leaves"], tiles=s2["num_nodes"],
        points_read=s2["leaf_points"], gpoints_per_s_read=round(s2["leaf_points"] / max(s2["ms_leaves"], 1e-9) / 1e6, 3),
        peak_device_bytes=s2["peak_device_bytes"], blocks=s2["blocks_processed"], key_batches=s2["key_batches"], checksum=s2_sum,
        octree_for_scale=dict(ms_leaves=round(oc["ms_leaves"], 3), ms_parents=round(oc["ms_parents"], 3), leaves=oc["num_leaves"], tiles=oc["num_nodes"],
                              points_read=oc["leaf_points"], peak_device_bytes=oc["peak_device_bytes"], checksum=oc_sum),
        gpu=name, power_limit=power)
    print(json.dumps(out), flush=True)
    cloud.free()
    tree.free()
    ctx.close()


if __name__ == "__main__":
    main()
