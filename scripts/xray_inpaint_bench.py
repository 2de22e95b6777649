"""Inpainting X-ray quadtrees (Context.inpaint_xray_quadtree) on one GPU.

A config-2 octree of --points points is built resident and written per tile size with xray_quadtree_write_dir on a transparent
background; the pixel size is chosen so that the deepest level is --deepest-256 (256 px) or --deepest-big (larger tiles), small
enough per pixel that the points leave holes.  The quadtree is then inpainted with k = --k into a fresh directory.  For every
tile size one JSON line gives the card and its power limit (read in the same run), the leaves, hole pixels filled, blocks and
block depth, the time split (tile decode and PNG encode summed over host threads; kernels and parents by CUDA events; the
call's wall time) and the peak device bytes."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED = 1  # bench.py's generator seed


def card():
    """(name, power limit) of GPU 0, read in the same run as the measurement."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:
        return None, "unknown (%s)" % str(e)[:80]


def log(*a):
    print("[xray_inpaint_bench]", *a, file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=float, default=2e7)
    ap.add_argument("--tiles", default="256,4096")
    ap.add_argument("--deepest-256", type=int, default=5)
    ap.add_argument("--deepest-big", type=int, default=2)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--tmp", default=None)
    a = ap.parse_args()
    import point_cloud_viewer_b200 as pcv

    name, power = card()
    ctx = pcv.Context(0)
    kind = pcv.SYNTH_GAUSS_CLUSTERS
    bmin, bmax, res = pcv.synth_bbox(kind)
    n = int(a.points)
    log("generating %d points on the host" % n)
    x, y, z, rgb = pcv.synth_points_host(kind, SEED, 0, n)
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax)
    del x, y, z, rgb
    ext = max(bmax[0] - bmin[0], bmax[1] - bmin[1])
    tmp = tempfile.mkdtemp(prefix="xray_inpaint_bench_", dir=a.tmp)
    try:
        for T in [int(v) for v in a.tiles.split(",")]:
            deepest = a.deepest_256 if T <= 256 else a.deepest_big
            px = ext / T / 2 ** deepest * 0.999
            src, out = os.path.join(tmp, "src%d" % T), os.path.join(tmp, "out%d" % T)
            t = time.perf_counter()
            tree.xray_quadtree_write_dir(src, T, px, background=pcv.TRANSPARENT)
            build_s = time.perf_counter() - t
            log("T=%d: built in %.1f s, inpainting" % (T, build_s))
            t = time.perf_counter()
            info = ctx.inpaint_xray_quadtree(src, out, a.k, background=pcv.WHITE)
            wall = time.perf_counter() - t
            rec = dict(card=name, power_limit=power, points=n, tile_px=T, pixel_size_m=px, k=a.k, build_s=round(build_s, 3), inpaint_wall_s=round(wall, 3))
            rec.update({kk: (round(v, 3) if isinstance(v, float) else v) for kk, v in info.items()})
            print(json.dumps(rec), flush=True)
            shutil.rmtree(src, ignore_errors=True)
            shutil.rmtree(out, ignore_errors=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        tree.free()
        ctx.close()


if __name__ == "__main__":
    main()
