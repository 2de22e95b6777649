"""python scripts/dir_query_batch_points_bench.py [--octree-points N] [--s2-points N] [--reps R] [--loop L] [--tmp PARENT]

Batched point queries that return their points straight from directories (OctreeDir / S2Dir.query_batch_points and their C
entries), on the setups of dir_query_bench.py and s2_dir_query_bench.py:
  octree  N (default 5e7) config-2 points (SYNTH_GAUSS_CLUSTERS, seed 1) written by build_octree_to_dir;
  s2      N (default 1e8) config-1 slab points (SYNTH_SLAB_ECEF, seed 1) with colour and intensity, written by build_s2_dir at
          level 20.
Location sets: 2000 bench.make_frusta frusta (octree: 1000 at far 10 and 1000 at far 102.4; S2: 2000 at far 10, since at far
102.4 the slab's survivors alone exceed device memory) and 1000 random OBBs (query_batch_points_bench.make_obbs).  Budgets: the default (most of the free device memory) and a quarter of the directory's
bytes.  One JSON line per (directory, location set, budget):
- c_call: the C entry alone into device arrays of the right size (every field the directory holds);
- python_call: query_batch_points (size query, allocation, fill; the size query is a second count pass);
- size_query: the C entry's size query alone;
- query_batch: the handle's counts-only call;
  each of these four: wall ms (median and every repetition, each ending in a device synchronise) and its pcv_dir_query_stats
  (bytes_read, chunks, peak from the last repetition; ms_cull, ms_read_wait, ms_select, ms_total as medians).  Each handle is
  first warmed up with the full batch in all four shapes; then the four calls alternate, in an order rotated every repetition,
  --reps times;
- resident: load_dir / load_s2_dir of the directory plus the resident query_batch_points, load included (once per directory and
  location set);
- query_points_loop: the handle's query_points to the host over the first --loop locations, per-location ms;
- parity: the offsets and every xyz / rgb / intensity element equal the resident call's on the timed inputs, and the offsets
  equal query_batch's counts.
The directories were just written, so their files were likely in the page cache: the reads measured are the page cache's, not
the disk's (nothing here drops the cache; that is a system-wide setting).  Every line carries the card and its power limit, read
in the same run.  Progress goes to stderr."""
import argparse
import ctypes as C
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

from bench import make_frusta  # noqa: E402
from query_batch_points_bench import make_obbs  # noqa: E402
from xray_dir_bench import SEED, card, dir_size  # noqa: E402

STATS = ("bytes_read", "bytes_uploaded", "node_files_read", "chunks", "ms_cull", "ms_read_wait", "ms_select", "ms_total", "peak_device_bytes",
         "max_device_bytes", "tested_points", "returned_points", "visited_pairs", "kernel_launches")


def log(*a):
    print("[dir_query_batch_points_bench]", *a, file=sys.stderr, flush=True)


def pick(st):
    return {k: st[k] for k in STATS}


def c_call(torch, fn, h, locs, total, bufs=None):
    """The C entry into device arrays of `total` points (bufs: the fields' tensors, allocated here when None); returns (offsets, bufs)."""
    from point_cloud_viewer_b200 import _native as N

    dev = torch.device("cuda", h.ctx.device)
    if bufs is None:
        has_rgb = getattr(h, "has_color", True)
        bufs = {"xyz": torch.empty((total, 3), dtype=torch.float64, device=dev), "src": torch.empty(total, dtype=torch.int64, device=dev)}
        if has_rgb:
            bufs["rgb"] = torch.empty((total, 3), dtype=torch.uint8, device=dev)
        if h.has_intensity:
            bufs["intensity"] = torch.empty(total, dtype=torch.float32, device=dev)
    arr = (N.Location * len(locs))(*locs)
    off = np.zeros(len(locs) + 1, np.uint64)
    p = lambda k: C.c_void_p(bufs[k].data_ptr()) if k in bufs else None  # noqa: E731
    N.check(fn(h.h, arr, len(locs), None, 0, off.ctypes.data, p("xyz"), p("rgb"), p("intensity"), p("src"), total))
    return off, bufs


def timed(torch, f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3, r


def run_dir(torch, pcv, ctx, kind, d, sets, reps, loop, common):
    L = pcv._native.lib()
    fn = L.pcv_octree_dir_query_batch_points_device if kind == "octree" else L.pcv_s2_dir_query_batch_points_device
    opener = pcv.OctreeDir if kind == "octree" else pcv.S2Dir
    _, size = dir_size(d)
    for set_name, locs in sets.items():
        # the resident baseline, load included; its outputs stay on the device for the parity check
        t = time.perf_counter()
        res = ctx.load_dir(d) if kind == "octree" else ctx.load_s2_dir(d)
        roff, rout = res.query_batch_points(locs, fields=[k for k in ("xyz", "rgb", "intensity") if k != "intensity" or res.has_intensity])
        torch.cuda.synchronize()
        resident_ms = (time.perf_counter() - t) * 1e3
        res.free()
        for budget in (0, size // 4):
            log(kind, set_name, "budget", budget)
            h = opener(ctx, d, budget)
            try:
                # warm-up with the full batch in every shape timed below: the S2 box scan, the pinned chunk buffers, the output
                # arrays and the first-call costs of each path
                h.query_batch(locs)
                off, _ = c_call(torch, fn, h, locs, 0, {})
                total = int(off[-1])
                off, bufs = c_call(torch, fn, h, locs, total)
                h.query_batch_points(locs)
                # the four calls alternate, their order rotated every repetition; medians of --reps
                runs = {k: [] for k in ("query_batch", "size_query", "c_call", "python_call")}
                calls = {
                    "query_batch": lambda: h.query_batch(locs),
                    "size_query": lambda: c_call(torch, fn, h, locs, 0, {}),
                    "c_call": lambda: c_call(torch, fn, h, locs, total, bufs),
                    "python_call": lambda: h.query_batch_points(locs),
                }
                names = list(calls)
                counts = None
                for r in range(reps):
                    for k in names[r % len(names):] + names[: r % len(names)]:
                        ms, res_k = timed(torch, calls[k])
                        runs[k].append((ms, pick(h.last_stats())))
                        if k == "query_batch":
                            counts = res_k[0]
                        elif k == "c_call":
                            off = res_k[0]
                        del res_k  # the Python call's tensors are freed before the next call

                def summary(k):
                    ms = [m for m, _ in runs[k]]
                    sts = [st for _, st in runs[k]]
                    out = dict(sts[-1], wall_ms=float(np.median(ms)), wall_ms_all=[round(m, 2) for m in ms])
                    for f in ("ms_cull", "ms_read_wait", "ms_select", "ms_total"):
                        out[f] = float(np.median([st[f] for st in sts]))
                    return out

                st = summary("c_call")
                parity = bool(np.array_equal(off, roff) and np.array_equal(np.diff(off.astype(np.int64)), counts.astype(np.int64)))
                for k, v in rout.items():
                    a, b = bufs[k], v
                    if k == "xyz":
                        a, b = a.view(torch.int64), b.view(torch.int64)
                    parity = parity and bool(torch.equal(a, b))
                del bufs
                t = time.perf_counter()
                looped = 0
                for loc in locs[:loop]:
                    looped += sum(len(b["src"]) for b in h.query_points(loc, batch_size=1 << 26))
                loop_s = time.perf_counter() - t
                out = dict(common, directory=kind, directory_bytes=size, locations_kind=set_name, locations=len(locs), reps=reps,
                           max_device_bytes=budget or st["max_device_bytes"], budget="default" if budget == 0 else "quarter of the directory",
                           written_points=total, c_call=st, python_call=summary("python_call"), size_query=summary("size_query"),
                           query_batch=summary("query_batch"), resident=dict(load_and_call_ms=resident_ms),
                           query_points_loop=dict(locations=min(loop, len(locs)), points=looped, s=loop_s, ms_per_location=loop_s * 1e3 / max(1, min(loop, len(locs)))),
                           peak_within_budget=st["peak_device_bytes"] <= st["max_device_bytes"], parity=parity)
                print(json.dumps(out), flush=True)
            finally:
                h.close()
        del rout


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--octree-points", type=float, default=5e7)
    ap.add_argument("--s2-points", type=float, default=1e8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop", type=int, default=20, help="locations of the query_points loop")
    ap.add_argument("--tmp", default=None)
    a = ap.parse_args()
    import torch

    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    name, power = card()
    ctx = pcv.Context(0)
    tmp = tempfile.mkdtemp(prefix="dir_query_batch_points_bench_", dir=a.tmp)
    common = dict(card=name, power_limit=power, page_cache="likely (just written)")
    try:
        if a.octree_points > 0:
            n = int(a.octree_points)
            kind = pcv.SYNTH_GAUSS_CLUSTERS
            bmin, bmax, res = pcv.synth_bbox(kind)
            log("octree directory: %d points" % n)
            x, y, z, rgb = pcv.synth_points_host(kind, SEED, 0, n)
            d = os.path.join(tmp, "octree")
            ctx.build_octree_to_dir(d, x, y, z, rgb, res, bmin, bmax)
            del x, y, z, rgb
            bmin, bmax = np.asarray(bmin, np.float64), np.asarray(bmax, np.float64)
            sets = {"frusta": make_frusta(G, bmin, bmax, 1000, 10.0) + make_frusta(G, bmin, bmax, 1000, 102.4), "obbs": make_obbs(G, bmin, bmax, 1000)}
            run_dir(torch, pcv, ctx, "octree", d, sets, a.reps, a.loop, dict(common, points=n))
            shutil.rmtree(d, ignore_errors=True)
        if a.s2_points > 0:
            n = int(a.s2_points)
            log("S2 directory: %d points" % n)
            x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED, 0, n)
            inten = (np.arange(n) % 1000).astype(np.float32)
            d = os.path.join(tmp, "s2")
            ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=20)
            del x, y, z, rgb, inten
            h = pcv.S2Dir(ctx, d)
            bmin, bmax = h.bbox_min, h.bbox_max
            h.close()
            sets = {"frusta": make_frusta(G, bmin, bmax, 2000, 10.0), "obbs": make_obbs(G, bmin, bmax, 1000)}
            run_dir(torch, pcv, ctx, "s2", d, sets, a.reps, a.loop, dict(common, points=n))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
        ctx.close()


if __name__ == "__main__":
    main()
