"""python scripts/ooc_bench.py [--points N] [--dir PARENT]

Out-of-core build_octree on one GPU: N config-2 points (the benchmark's generator, seed 1) in pageable host memory ->
pcv_build_octree_to_dir with the default group budget (pcv_in_core_capacity) -> a temporary directory under PARENT (default:
the system temporary directory), removed afterwards.  Prints one JSON line: k, groups, per-phase ms, end-to-end Gpoints/s, the
host -> device bytes over the histogram + selection time, the card and its power limit, the directory, and a verdict from the
written files alone: the points of meta.pb sum to N, every node's files have the sizes meta.pb implies, and the 2^24-bin histogram
of every .rgb colour equals the generator's.  Progress goes to stderr."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

SEED = 1  # bench.py's generator seed


def card():
    """(name, power limit) of GPU 0, read in the same run as the measurement."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:
        return None, "unknown (%s)" % str(e)[:80]


def run(n, base_dir):
    import numpy as np
    import torch

    import point_cloud_viewer_b200 as pcv
    from proto_meta import parse_meta

    kind = pcv.SYNTH_GAUSS_CLUSTERS
    bmin, bmax, res = pcv.synth_bbox(kind)
    need_ram = 27 * n + (1 << 31)
    avail_ram = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail_ram < need_ram:
        return {"n": n, "error": "needs %.1f GB of free host memory, have %.1f GB" % (need_ram / 1e9, avail_ram / 1e9)}
    base_dir = base_dir or tempfile.gettempdir()
    need_disk = 14 * n
    free_disk = shutil.disk_usage(base_dir).free
    if free_disk < need_disk:
        return {"n": n, "error": "needs %.1f GB of free disk under %s, have %.1f GB" % (need_disk / 1e9, base_dir, free_disk / 1e9)}
    ctx = pcv.Context(0)
    x, y, z = (np.empty(n, np.float64) for _ in range(3))
    rgb = np.empty(3 * n, np.uint8)
    want_hist = np.zeros(1 << 24, np.int64)
    step = 100_000_000
    dx, dy, dz = (torch.empty(step, dtype=torch.float64, device="cuda") for _ in range(3))
    drgb = torch.empty(3 * step, dtype=torch.uint8, device="cuda")
    for first in range(0, n, step):  # the generator on the device, slice by slice into host memory
        m = min(step, n - first)
        ctx.synth_points_device(kind, SEED, first, m, dx.data_ptr(), dy.data_ptr(), dz.data_ptr(), drgb.data_ptr())
        for h, d in ((x, dx), (y, dy), (z, dz)):
            torch.from_numpy(h[first:first + m]).copy_(d[:m])
        torch.from_numpy(rgb[3 * first:3 * (first + m)]).copy_(drgb[:3 * m])
        c = drgb[:3 * m].view(m, 3).to(torch.int64)
        want_hist += torch.bincount(c[:, 0] | (c[:, 1] << 8) | (c[:, 2] << 16), minlength=1 << 24).cpu().numpy()
        del c
    del dx, dy, dz, drgb
    torch.cuda.empty_cache()
    ctx.release_cached_memory()
    capacity = ctx.in_core_capacity()
    print("[ooc_bench] %d points generated in host memory; in-core capacity %d" % (n, capacity), file=sys.stderr, flush=True)
    d = tempfile.mkdtemp(prefix="pcv_ooc_", dir=base_dir)
    try:
        name, power = card()
        w0 = time.perf_counter()
        info = ctx.build_octree_to_dir(d, x, y, z, rgb, res, bmin, bmax)
        wall = time.perf_counter() - w0
        del x, y, z, rgb
        print("[ooc_bench] built %d points in %.1f s: %s" % (n, wall, info), file=sys.stderr, flush=True)
        # verdict from the directory alone: every .rgb file into one buffer, its colour histogram on the GPU in slices
        meta = parse_meta(open(os.path.join(d, "meta.pb"), "rb").read())
        total = sum(v[0] for v in meta["nodes"].values())
        sizes_ok = True
        colours = np.empty(3 * total, np.uint8)
        o = 0
        for (hi, lo), (num, enc) in meta["nodes"].items():
            stem = os.path.join(d, pcv.node_name(hi, lo))
            if num == 0:
                sizes_ok = sizes_ok and not os.path.exists(stem + ".rgb") and not os.path.exists(stem + ".xyz")
                continue
            sizes_ok = sizes_ok and os.path.getsize(stem + ".xyz") == num * 3 * pcv.ENC_BYTES[enc] and os.path.getsize(stem + ".rgb") == num * 3
            with open(stem + ".rgb", "rb") as f:
                o += f.readinto(memoryview(colours)[o:o + 3 * num])
        got_hist = np.zeros(1 << 24, np.int64)
        for first in range(0, total, step):
            c = torch.from_numpy(colours[3 * first:3 * min(total, first + step)]).cuda().view(-1, 3).to(torch.int64)
            got_hist += torch.bincount(c[:, 0] | (c[:, 1] << 8) | (c[:, 2] << 16), minlength=1 << 24).cpu().numpy()
            del c
        del colours
        hist_ok = bool(np.array_equal(got_hist, want_hist))
        sel = info["ms_histogram"] + info["ms_select"]
        return {"n": n, "prefix_levels": info["prefix_levels"], "groups": info["groups"], "largest_group": info["largest_group"], "in_core_capacity": capacity,
                "nodes": info["num_nodes"], "phases_ms": {k: info["ms_" + k] for k in ("histogram", "select", "build", "write", "top", "total")},
                "wall_s": wall, "gpoints_per_s": n / wall / 1e9, "h2d_bytes": info["h2d_bytes"],
                "h2d_GBps_over_histogram_and_select": info["h2d_bytes"] / (sel * 1e-3) / 1e9 if sel > 0 else None,
                "gpu": name, "power_limit": power, "directory": d, "input": "pageable host SoA (numpy), config-2 generator",
                "verdict": {"ok": total == n and sizes_ok and hist_ok, "points_sum_equals_n": total == n, "file_sizes_match_meta": sizes_ok,
                            "colour_histogram_equal": hist_ok}}
    finally:
        shutil.rmtree(d, ignore_errors=True)
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=float, default=1.2e9, help="host points to build out of core (default 1.2e9: more than one 80 GB H100 builds in core)")
    ap.add_argument("--dir", default=None, help="parent of the temporary output directory (default: the system temporary directory)")
    args = ap.parse_args()
    print(json.dumps({"out_of_core": run(int(args.points), args.dir)}))


if __name__ == "__main__":
    main()
