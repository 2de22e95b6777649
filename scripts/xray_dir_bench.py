"""python scripts/xray_dir_bench.py [--dir OCTREE_DIR | --points N] [--dirs K] [--tile-px T] [--pixel-m PX] [--budget BYTES] [--tmp PARENT]

The X-ray quadtree straight from an on-disk octree.  With --dir, the octree directory given is X-rayed; otherwise N config-2
points (the benchmark's generator, seed 1) are built with build_octree_to_dir into a temporary directory under PARENT, which is
removed afterwards.  The quadtree (T-px tiles, default 256; pixel size PX, default with --points: 2^-6 of the generator's extent per tile) is built
by xray_quadtree_from_dir under max_device_bytes = BYTES (default: a quarter of the directory's node data), every tile handed to
a callback that keeps nothing.  Prints one JSON line: the card and its power limit, the directory's points, nodes and bytes, the
budget, wall seconds of the build and of the X-ray call, the occupancy pass and window phases, bytes read and uploaded, windows,
nodes reused and re-read, the peak of device memory, tiles and leaves.  Progress goes to stderr.

With --dirs K > 1 (and --points), the N points are split into K interleaved directories over the same area (point i goes to
directory i mod K, as survey runs over one area), each built with build_octree_to_dir, plus one directory of all N points.
The JSON line then times xray_quadtree_from_dirs over the K directories (default budget: a quarter of their node data) against
load_dir of each plus xray_quadtree_clouds, and against xray_quadtree_from_dir over the one directory of all the points under
the same budget, with the phases, bytes read, windows and peak of the directory calls, and whether the three agree in tiles."""
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
    print("[xray_dir_bench]", *a, file=sys.stderr, flush=True)


def dir_size(d):
    nodes = size = 0
    for f in os.listdir(d):
        if f.endswith(".xyz"):
            nodes += 1
        size += os.path.getsize(os.path.join(d, f))
    return nodes, size


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--dir", default=None)
    ap.add_argument("--points", type=float, default=2e8)
    ap.add_argument("--tile-px", type=int, default=256)
    ap.add_argument("--pixel-m", type=float, default=0.0)
    ap.add_argument("--budget", type=float, default=0)
    ap.add_argument("--tmp", default=None)
    ap.add_argument("--dirs", type=int, default=1)
    a = ap.parse_args()
    if a.dirs > 1:
        if a.dir is not None:
            raise SystemExit("--dirs K > 1 splits --points into K directories; it takes no --dir")
        return main_dirs(a)
    import point_cloud_viewer_b200 as pcv

    name, power = card()
    ctx = pcv.Context(0)
    tmp, build_s, n = None, None, None
    d = a.dir
    if d is None:
        n = int(a.points)
        kind = pcv.SYNTH_GAUSS_CLUSTERS
        bmin, bmax, res = pcv.synth_bbox(kind)
        log("generating %d points on the host" % n)
        x, y, z, rgb = pcv.synth_points_host(kind, SEED, 0, n)
        if a.pixel_m <= 0:
            a.pixel_m = max(bmax[0] - bmin[0], bmax[1] - bmin[1]) / a.tile_px / 64.0
        tmp = tempfile.mkdtemp(prefix="xray_dir_bench_", dir=a.tmp)
        d = os.path.join(tmp, "octree")
        t = time.perf_counter()
        ctx.build_octree_to_dir(d, x, y, z, rgb, res, bmin, bmax)
        build_s = time.perf_counter() - t
        del x, y, z, rgb
        log("built the octree into %s in %.1f s" % (d, build_s))
    try:
        nodes, size = dir_size(d)
        budget = int(a.budget) if a.budget else size // 4
        T, px = a.tile_px, a.pixel_m
        if px <= 0:
            raise SystemExit("--pixel-m is needed with --dir")
        ntiles = [0]

        def on_tile(level, index, img):
            ntiles[0] += 1
            return False

        log("X-ray from disk: %d px tiles, %.6g m per pixel, budget %d bytes (directory %d bytes)" % (T, px, budget, size))
        t = time.perf_counter()
        info, _ = ctx.xray_quadtree_from_dir(d, T, px, on_tile=on_tile, keep_tiles=False, max_device_bytes=budget)
        xs = time.perf_counter() - t
        out = dict(card=name, power_limit=power, points=n, dir_nodes=nodes, dir_bytes=size, max_device_bytes=budget, build_s=build_s, xray_s=round(xs, 3),
                   ms_occupancy=round(info["ms_occupancy"], 1), ms_windows=round(info["ms_windows"], 1), ms_leaves=round(info["ms_leaves"], 1),
                   ms_parents=round(info["ms_parents"], 1), bytes_read=info["bytes_read"], node_files_read=info["node_files_read"],
                   bytes_uploaded=info["bytes_uploaded"], windows=info["windows_loaded"], nodes_reused=info["nodes_reused"], nodes_reread=info["nodes_reread"],
                   largest_window_bytes=info["largest_window_bytes"], peak_device_bytes=info["peak_device_bytes"], block_level=info["block_level"],
                   deepest_level=info["deepest_level"], tiles=ntiles[0], leaves=info["num_leaves"], occupied_leaves=info["occupied_leaves"],
                   peak_within_budget=info["peak_device_bytes"] <= budget, dir_larger_than_budget=size > budget)
        print(json.dumps(out), flush=True)
    finally:
        if tmp:
            shutil.rmtree(tmp, ignore_errors=True)
        ctx.close()


def _digest(tiles):
    """(level, index) -> hash of the tile's bytes, for comparing quadtrees without keeping them."""
    import hashlib

    return {k: hashlib.sha1(v.tobytes()).hexdigest() for k, v in tiles.items()}


def main_dirs(a):
    import numpy as np

    import point_cloud_viewer_b200 as pcv

    name, power = card()
    ctx = pcv.Context(0)
    n, K = int(a.points), a.dirs
    kind = pcv.SYNTH_GAUSS_CLUSTERS
    bmin, bmax, res = pcv.synth_bbox(kind)
    log("generating %d points on the host" % n)
    x, y, z, rgb = pcv.synth_points_host(kind, SEED, 0, n)
    rgb = np.asarray(rgb).reshape(-1, 3)
    T = a.tile_px
    px = a.pixel_m if a.pixel_m > 0 else max(bmax[0] - bmin[0], bmax[1] - bmin[1]) / T / 64.0
    tmp = tempfile.mkdtemp(prefix="xray_dir_bench_", dir=a.tmp)
    try:
        dirs = [os.path.join(tmp, "part%d" % k) for k in range(K)]
        t = time.perf_counter()
        for k, d in enumerate(dirs):
            ctx.build_octree_to_dir(d, *(np.ascontiguousarray(v[k::K]) for v in (x, y, z)), np.ascontiguousarray(rgb[k::K]).reshape(-1), res, bmin, bmax)
        build_s = time.perf_counter() - t
        whole = os.path.join(tmp, "all")
        ctx.build_octree_to_dir(whole, x, y, z, rgb.reshape(-1), res, bmin, bmax)
        del x, y, z, rgb
        log("built %d directories and the one of all points in %s" % (K, tmp))
        sizes = [dir_size(d) for d in dirs]
        size = sum(s for _, s in sizes)
        budget = int(a.budget) if a.budget else size // 4
        ntiles = [0]

        def on_tile(level, index, img):
            ntiles[0] += 1
            return False

        log("X-ray from %d directories: %d px tiles, %.6g m per pixel, budget %d bytes (directories %d bytes)" % (K, T, px, budget, size))
        t = time.perf_counter()
        info, tiles = ctx.xray_quadtree_from_dirs(dirs, T, px, on_tile=on_tile, max_device_bytes=budget)
        xs = time.perf_counter() - t
        got = _digest(tiles)
        del tiles
        log("load_dir x %d + xray_quadtree_clouds" % K)
        t = time.perf_counter()
        clouds = [ctx.load_dir(d) for d in dirs]
        load_s = time.perf_counter() - t
        t = time.perf_counter()
        cinfo, ctiles = ctx.xray_quadtree_clouds(clouds, T, px)
        clouds_s = time.perf_counter() - t
        for c in clouds:
            c.free()
        same_clouds = _digest(ctiles) == got
        del ctiles
        log("one directory of all the points")
        t = time.perf_counter()
        winfo, wtiles = ctx.xray_quadtree_from_dir(whole, T, px, max_device_bytes=budget)
        whole_s = time.perf_counter() - t
        same_whole = _digest(wtiles) == got
        del wtiles
        phases = lambda i: dict(ms_occupancy=round(i["ms_occupancy"], 1), ms_windows=round(i["ms_windows"], 1), ms_leaves=round(i["ms_leaves"], 1),  # noqa: E731
                                ms_parents=round(i["ms_parents"], 1), bytes_read=i["bytes_read"], bytes_uploaded=i["bytes_uploaded"],
                                windows=i["windows_loaded"], nodes_reused=i["nodes_reused"], nodes_reread=i["nodes_reread"],
                                largest_window_bytes=i["largest_window_bytes"], peak_device_bytes=i["peak_device_bytes"], block_level=i["block_level"])
        out = dict(card=name, power_limit=power, points=n, dirs=K, dir_nodes=sum(v for v, _ in sizes), dir_bytes=size, max_device_bytes=budget,
                   build_s=round(build_s, 1), xray_s=round(xs, 3), **phases(info), tiles=ntiles[0], leaves=info["num_leaves"],
                   occupied_leaves=info["occupied_leaves"], peak_within_budget=info["peak_device_bytes"] <= budget,
                   loaded_load_s=round(load_s, 3), loaded_clouds_s=round(clouds_s, 3), loaded_peak_device_bytes=cinfo["peak_device_bytes"],
                   same_tiles_as_loaded=same_clouds, whole_dir_s=round(whole_s, 3), whole=phases(winfo), same_tiles_as_whole=same_whole)
        print(json.dumps(out), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        ctx.close()


if __name__ == "__main__":
    main()
