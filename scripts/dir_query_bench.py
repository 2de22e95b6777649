"""python scripts/dir_query_bench.py [--dir OCTREE_DIR | --points N] [--budget BYTES] [--frusta K] [--tmp PARENT]

Point queries straight from an on-disk octree.  With --dir, the octree directory given is queried; otherwise N config-2 points (the
benchmark's generator, seed 1) are built with build_octree_to_dir into a temporary directory under PARENT, which is removed
afterwards.  The directory is opened with max_device_bytes = BYTES (default: a quarter of its node bytes) and three workloads run:
  batch    the K + K frusta of bench.make_frusta (far 10 and 102.4) through query_batch
  points   20 of them through query_points, batch size 500 000, every batch consumed
  blob     visible_nodes + nodes_data_blob for 20 cameras (the same frusta's matrices)
Each workload runs twice in the same process ("first read", then "repeat"); nothing drops the page cache, so the repeat is probably
served from it when the directory is smaller than host RAM (reported).  One JSON line per run: the card and its power limit, the
directory's size, the budget and the peak, bytes read and uploaded, wall seconds split into ms_select / ms_read_wait / ms_cull,
points tested per second, and a parity verdict against load_dir + the resident calls whenever the directory fits on the device.
Progress goes to stderr."""
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

from xray_dir_bench import SEED, card, dir_size  # noqa: E402


def log(*a):
    print("[dir_query_bench]", *a, file=sys.stderr, flush=True)


def host_ram():
    try:
        return os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES")
    except (ValueError, OSError):
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--dir", default=None)
    ap.add_argument("--points", type=float, default=1e8)
    ap.add_argument("--budget", type=float, default=0)
    ap.add_argument("--frusta", type=int, default=1000)
    ap.add_argument("--tmp", default=None)
    a = ap.parse_args()
    import torch  # noqa: F401  (device memory query)

    import bench
    import point_cloud_viewer_b200 as pcv

    name, power = card()
    ctx = pcv.Context(0)
    tmp, build_s, n = None, None, None
    d = a.dir
    G = pcv.geometry
    if d is None:
        n = int(a.points)
        kind = pcv.SYNTH_GAUSS_CLUSTERS
        bmin, bmax, res = pcv.synth_bbox(kind)
        log("generating %d points on the host" % n)
        x, y, z, rgb = pcv.synth_points_host(kind, SEED, 0, n)
        tmp = tempfile.mkdtemp(prefix="dir_query_bench_", dir=a.tmp)
        d = os.path.join(tmp, "octree")
        t = time.perf_counter()
        ctx.build_octree_to_dir(d, x, y, z, rgb, res, bmin, bmax)
        build_s = time.perf_counter() - t
        del x, y, z, rgb
        log("built the octree into %s in %.1f s" % (d, build_s))
    try:
        nodes, size = dir_size(d)
        budget = int(a.budget) if a.budget else size // 4
        h = ctx.open_dir(d, budget)
        bmin, bmax = h.bbox_min, h.bbox_max
        frusta = bench.make_frusta(G, bmin, bmax, a.frusta, 10.0) + bench.make_frusta(G, bmin, bmax, a.frusta, 102.4)
        cams = [np.array(f.clip_from_query).reshape(4, 4).T for f in frusta[:: max(1, len(frusta) // 20)][:20]]
        free, _ = torch.cuda.mem_get_info(0)
        resident = ctx.load_dir(d) if size * 2 < free else None  # parity against load_dir whenever the directory fits
        ram = host_ram()
        common = dict(card=name, power_limit=power, points=h.num_points, build_s=build_s, dir_nodes=nodes, dir_bytes=size, host_ram_bytes=ram,
                      dir_smaller_than_host_ram=(ram is not None and size < ram), max_device_bytes=budget)

        def run_batch():
            counts, tested = h.query_batch(frusta)
            sts = [h.last_stats()]
            ok = None
            if resident is not None:
                wc, wt = resident.query_batch_device(frusta)
                ok = bool(np.array_equal(counts, wc) and np.array_equal(tested, wt))
            return sts, ok

        def run_points():
            sts, ok = [], resident is not None
            for loc in frusta[:20]:
                got = []
                h.query_points(loc, callback=lambda b: got.append((len(b["src"]), b["xyz"][:1].copy())) and False, batch_size=500_000)
                sts.append(h.last_stats())
                if resident is not None:
                    want = []
                    resident.query_points(loc, callback=lambda b: want.append((len(b["src"]), b["xyz"][:1].copy())) and False, batch_size=500_000)
                    ok = ok and [g[0] for g in got] == [w[0] for w in want] and all(np.array_equal(g[1], w[1]) for g, w in zip(got, want))
            return sts, (ok if resident is not None else None)

        def run_blob():
            sts, ok = [], resident is not None
            for M in cams:
                names = h.get_visible_nodes(M)
                s1 = h.last_stats()
                blob = h.nodes_data_blob(names) if names else np.zeros(0, np.uint8)
                s2 = h.last_stats() if names else dict(s1)
                both = dict(s2)
                for k in ("ms_select", "ms_total"):
                    both[k] = s1[k] + s2[k]
                both["peak_device_bytes"] = max(s1["peak_device_bytes"], s2["peak_device_bytes"])
                sts.append(both)
                if resident is not None:
                    ok = ok and names == resident.get_visible_nodes(M) and (not names or blob.tobytes() == resident.nodes_data_blob(names).tobytes())
            return sts, (ok if resident is not None else None)

        for wl, fn in (("batch", run_batch), ("points", run_points), ("blob", run_blob)):
            for run in ("first read", "repeat"):
                t = time.perf_counter()
                sts, ok = fn()
                wall = time.perf_counter() - t
                tot = lambda k: sum(s[k] for s in sts)  # noqa: E731
                out = dict(common, workload=wl, run=run, calls=len(sts), wall_s=round(wall, 4), peak_device_bytes=max(s["peak_device_bytes"] for s in sts),
                           bytes_read=tot("bytes_read"), bytes_uploaded=tot("bytes_uploaded"), node_files_read=tot("node_files_read"), chunks=tot("chunks"),
                           ms_total=round(tot("ms_total"), 2), ms_select=round(tot("ms_select"), 2), ms_read_wait=round(tot("ms_read_wait"), 2),
                           ms_cull=round(tot("ms_cull"), 2), tested_points=tot("tested_points"), returned_points=tot("returned_points"),
                           tested_points_per_s=tot("tested_points") / wall if wall > 0 else None, kernel_launches=tot("kernel_launches"), parity=ok)
                out["peak_within_budget"] = out["peak_device_bytes"] <= budget
                print(json.dumps(out), flush=True)
        h.close()
        if resident is not None:
            resident.free()
    finally:
        if tmp:
            shutil.rmtree(tmp, ignore_errors=True)
        ctx.close()


if __name__ == "__main__":
    main()
