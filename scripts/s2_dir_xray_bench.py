"""python scripts/s2_dir_xray_bench.py [--points N] [--tile-px T] [--leaves-per-side L]

The X-ray quadtree straight from an S2 directory at scale: N config-1 slab points (the ECEF slab generator on the host, seed 1;
default 1e8) with colour and intensity, written by Context.build_s2_dir at level 20 into a temporary directory (about 31 B per
point on disk), then Context.xray_quadtree_from_s2_dirs with T-px tiles (default 256) in the slab's local frame at the pixel
size that puts about L leaves (default 64) along the longer side of the local box, as scripts/s2_xray_bench.py does.  Two
budgets: the default (most of the free memory) and a small one: an eighth of the directory's size, doubled until one leaf's
window fits (the budgets refused on the way are reported with their errors); each call is repeated once and both are reported.
For comparison, load_s2_dir + S2Cloud.xray_quadtree on the same directory, also twice.  The directory was just
written, so its files were likely in the page cache: the reads are the page cache's, not the disk's (dropping caches is a
system-wide setting and is not done here).  Prints one JSON line: per call the wall time, ms_occupancy (the scan pass),
ms_windows, the device leaf and parent time, bytes read and uploaded, windows loaded and cells reused, the peak, and an
all-tiles checksum; the card's name and power limit read in the same run.  Progress goes to stderr."""
import argparse
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

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
    print("[s2_dir_xray_bench]", *a, file=sys.stderr, flush=True)


def timed(fn):
    """fn(on_tile) -> info; returns (wall ms, info, checksum of the set of tiles: every (level, index, RGBA), in any order, and
    the checksum of the delivery order)."""
    digests, order = [], hashlib.sha256()

    def on_tile(level, index, img):
        key = bytes([level]) + int(index).to_bytes(8, "little")
        digests.append(hashlib.sha256(key + img.tobytes()).digest())
        order.update(key)

    t = time.perf_counter()
    info = fn(on_tile)
    wall = (time.perf_counter() - t) * 1e3
    info["order_checksum"] = order.hexdigest()[:16]
    return wall, info, hashlib.sha256(b"".join(sorted(digests))).hexdigest()[:16]


def row(wall, info, checksum):
    keys = ("ms_occupancy", "ms_windows", "ms_leaves", "ms_parents", "bytes_read", "bytes_uploaded", "windows_loaded", "nodes_reused", "nodes_reread",
            "largest_window_points", "occupied_leaves", "peak_device_bytes", "max_device_bytes", "num_nodes", "blocks_processed")
    out = dict(wall_ms=round(wall, 1), checksum=checksum, order_checksum=info["order_checksum"])
    out.update({k: (round(info[k], 1) if isinstance(info[k], float) else info[k]) for k in keys if k in info})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=100_000_000)
    ap.add_argument("--tile-px", type=int, default=256)
    ap.add_argument("--leaves-per-side", type=int, default=64)
    a = ap.parse_args()
    import numpy as np

    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    n, T = a.points, a.tile_px
    ctx = pcv.Context(0)
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED, 0, n)
    inten = np.random.default_rng(SEED).uniform(0.0, 100.0, n).astype(np.float32)
    log("%d points generated" % n)
    tmp = tempfile.mkdtemp(prefix="s2_dir_xray_bench_")
    try:
        d = os.path.join(tmp, "s2")
        t = time.perf_counter()
        ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=20)
        log("directory written in %.1f s" % (time.perf_counter() - t))
        del x, y, z, rgb, inten
        size = sum(os.path.getsize(os.path.join(d, f)) for f in os.listdir(d))
        cells = sum(1 for f in os.listdir(d) if f.endswith(".xyz"))
        probe = ctx.load_s2_dir(d)
        bmin, bmax = probe.bbox_min.copy(), probe.bbox_max.copy()
        probe.free()
        q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
        local_from_ecef = G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse()  # the slab's local frame (csrc/synth.cuh)
        corners = [[(bmax if k & (1 << ax) else bmin)[ax] for ax in range(3)] for k in range(8)]
        local = np.array([local_from_ecef.transform_point(np.array(c)) for c in corners])
        extent = float(max(local[:, 0].max() - local[:, 0].min(), local[:, 1].max() - local[:, 1].min()))
        px = extent / (T * a.leaves_per_side) * 1.01
        kw = dict(query_from_global=list(local_from_ecef.as7()), keep_tiles=False)
        runs = {}
        # an eighth of the directory, doubled until one leaf's window fits (the error of each budget that does not is reported)
        refused = []
        small = size // 8
        while True:
            try:
                ctx.xray_quadtree_from_s2_dirs(d, T, px, max_device_bytes=small, **kw)
                break
            except pcv.PcvError as e:
                if e.code != -6 or small >= size:
                    raise
                refused.append(dict(max_device_bytes=small, error=str(e)))
                log("budget %d refused: %s" % (small, e))
                small *= 2
        for name, budget in (("default", 0), ("small", small)):
            runs[name] = []
            for _ in range(2):
                wall, info, cs = timed(lambda cb: ctx.xray_quadtree_from_s2_dirs(d, T, px, on_tile=cb, max_device_bytes=budget, **kw)[0])
                runs[name].append(row(wall, info, cs))
                log(name, runs[name][-1])
        runs["load_s2_dir"] = []
        for _ in range(2):
            def load_and_xray(cb):
                t0 = time.perf_counter()
                cloud = ctx.load_s2_dir(d)
                ms_load = (time.perf_counter() - t0) * 1e3
                try:
                    info = cloud.xray_quadtree(T, px, on_tile=cb, **kw)[0]
                finally:
                    cloud.free()
                info["ms_load"] = ms_load
                return info

            wall, info, cs = timed(load_and_xray)
            r = row(wall, info, cs)
            r["ms_load"] = round(info["ms_load"], 1)
            runs["load_s2_dir"].append(r)
            log("load_s2_dir", r)
        same = len({r["checksum"] for v in runs.values() for r in v}) == 1
        same_order = len({r["order_checksum"] for v in runs.values() for r in v}) == 1
        gpu, power = card()
        last = runs["small"][-1]
        out = dict(points=n, cells=cells, directory_bytes=size, tile_px=T, pixel_size_m=px, page_cache="likely warm: the directory was just written",
                   same_tiles=same, same_order=same_order, small_budget=small, small_budget_over_directory=round(small / size, 3), refused_budgets=refused, runs=runs,
                   # the scan reads 24 B per point and uploads them; the device passes are timed separately (ms_leaves, ms_parents)
                   scan_gb_per_s=round(24 * n / max(last["ms_occupancy"], 1e-9) / 1e6, 2),
                   bound=("file reads and host-to-device copies (ms_occupancy + ms_windows >> ms_leaves + ms_parents)"
                          if last["ms_occupancy"] + last["ms_windows"] > 2 * (last["ms_leaves"] + last["ms_parents"]) else "the device passes"),
                   not_run="clouds above 2^32 points or above device memory", gpu=gpu, power_limit=power)
        print(json.dumps(out), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        ctx.close()


if __name__ == "__main__":
    main()
