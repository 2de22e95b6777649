"""Batched point queries that return their points (Octree / S2Cloud.query_batch_points) on the GPU: 1e8 resident config-1 slab
points (SYNTH_SLAB_ECEF), as an octree and as an S2 cloud split at level 20.

One JSON line per (source, location set): bench.make_frusta (1000 frusta, far 10) and 1000 random OBBs.  Each line holds
- the call: wall time of query_batch_points (size query, allocation, call) and of the C call alone into buffers of the right size
  (medians of --reps, ending in a device synchronise), ms_select / ms_cull of pcv_last_query_stats, tested and
  written points, Gpoints/s tested and survivors written per second over ms_cull, algorithmic_bytes against 3.35 TB/s (HBM3 of
  the H100 SXM data sheet);
- the phase split of the C call from one torch.profiler run (kernel time by name: selection, sort, count, scan, place);
- the same locations through query_batch_device (counts only) and a loop of query_points to the host over the first --loop
  locations, with the per-location time;
- a parity verdict: the first locations' segments against their query_points streams, bit for bit.
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

from bench import make_frusta  # noqa: E402
from xray_dir_bench import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, HBM3
PHASES = (  # kernel name fragments of each phase (demangled names), first match wins
    ("select", ("k_loc_proj", "k_bfs_", "k_s2_select_cells")),
    ("count", ("k_qbp_count",)),
    ("place", ("k_qbp_place", "k_qbp_advance")),
    ("scan", ("ScanTileState<unsigned int", "policy_hub<unsigned int")),  # the u32 scan of the tile counts
    ("sort", ("k_qbp_keys", "k_qbp_pair_tiles", "k_qbp_tiles", "DeviceRadixSort", "DeviceScan")),  # sort, then the u64 scan of the pairs' tiles
)


def log(*a):
    print("[query_batch_points_bench]", *a, file=sys.stderr, flush=True)


def make_obbs(G, bmin, bmax, count, seed=11):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        c = bmin + rng.random(3) * (bmax - bmin)
        q = rng.random((4, 12)).sum(1) - 6.0
        out.append(G.obb(G.Isometry(c, q / np.linalg.norm(q)), tuple(2.0 + 18.0 * rng.random(3))))
    return out


def phase_split(torch, fn):
    """Kernel milliseconds per phase of one call of fn, from torch.profiler's CUDA activities."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ms = {p: 0.0 for p, _ in PHASES}
    other = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        t = e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        for p, frags in PHASES:
            if any(f in e.name for f in frags):
                ms[p] += t
                break
        else:
            other += t
    ms["other"] = other
    return ms


def raw_call(torch, fn, h, locs, total):
    """One call of the C entry into torch buffers of `total` points; returns the offsets."""
    import ctypes as C

    from point_cloud_viewer_b200 import _native as N

    arr = (N.Location * len(locs))(*locs)
    dev = torch.device("cuda", h.ctx.device)
    bufs = [torch.empty((total, 3), dtype=torch.float64, device=dev), torch.empty((total, 3), dtype=torch.uint8, device=dev),
            torch.empty(total, dtype=torch.float32, device=dev), torch.empty(total, dtype=torch.int64, device=dev)]
    off = np.zeros(len(locs) + 1, np.uint64)
    N.check(fn(h.h, arr, len(locs), None, 0, off.ctypes.data, *[C.c_void_p(b.data_ptr()) for b in bufs], total))
    return off


def run_set(torch, fn, h, locs, reps, loop):
    dev_counts, dev_tested = h.query_batch_device(locs)  # warm-up of the count-only form
    count_ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        h.query_batch_device(locs)
        count_ms.append((time.perf_counter() - t) * 1e3)
        cst = h.last_query_stats()
    off, out = h.query_batch_points(locs)  # warm-up
    del out
    walls, stats = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        off, out = h.query_batch_points(locs)
        torch.cuda.synchronize()
        walls.append((time.perf_counter() - t) * 1e3)
        stats.append(h.last_query_stats())
        if _ < reps - 1:
            del out
    st = stats[-1]
    med = {k: float(np.median([s[k] for s in stats])) for k in ("ms_device", "ms_select", "ms_cull")}
    total, tested = int(off[-1]), int(st["tested_points"])
    # parity: the first locations' segments against their streams
    host = {k: v[: int(off[min(4, len(locs))])].cpu().numpy() for k, v in out.items()}
    parity = True
    for i in range(min(4, len(locs))):
        bs = h.query_points(locs[i], batch_size=1 << 26)
        a, b = int(off[i]), int(off[i + 1])
        src = np.concatenate([x["src"] for x in bs]) if bs else np.zeros(0, np.uint64)
        xyz = np.concatenate([x["xyz"] for x in bs]) if bs else np.zeros((0, 3))
        parity &= bool(np.array_equal(host["src"][a:b].astype(np.uint64), src) and np.array_equal(host["xyz"][a:b].view(np.uint64), xyz.view(np.uint64)))
    parity &= bool(np.array_equal(np.diff(off.astype(np.int64)), dev_counts.astype(np.int64)))
    del out, host
    # the C call alone into buffers of the right size (Python's query_batch_points adds a size query: a second count pass)
    raw_call(torch, fn, h, locs, total)
    raw_ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        raw_call(torch, fn, h, locs, total)
        torch.cuda.synchronize()
        raw_ms.append((time.perf_counter() - t) * 1e3)
    rst = h.last_query_stats()
    split = phase_split(torch, lambda: raw_call(torch, fn, h, locs, total))
    # the per-location alternative: query_points to the host, one call per location
    torch.cuda.synchronize()
    t = time.perf_counter()
    looped = 0
    for loc in locs[:loop]:
        looped += sum(len(x["src"]) for x in h.query_points(loc, batch_size=1 << 26))
    loop_s = time.perf_counter() - t
    ms = med["ms_cull"]
    return dict(locations=len(locs), wall_ms=float(np.median(walls)), c_call_wall_ms=float(np.median(raw_ms)),
                c_call=dict(ms_device=rst["ms_device"], ms_select=rst["ms_select"], ms_cull=rst["ms_cull"]), **med, phase_ms=split, tested_points=tested, written_points=total,
                kernel_launches=int(st["kernel_launches"]), algorithmic_bytes=int(st["algorithmic_bytes"]),
                gpoints_per_s_tested=tested / (ms * 1e-3) / 1e9 if ms > 0 else None,
                gpoints_per_s_written=total / (ms * 1e-3) / 1e9 if ms > 0 else None,
                hbm_fraction=(st["algorithmic_bytes"] / (ms * 1e-3)) / HBM_BYTES_PER_S if ms > 0 else None,
                count_only=dict(wall_ms=float(np.median(count_ms)), ms_select=cst["ms_select"], ms_cull=cst["ms_cull"], ms_device=cst["ms_device"],
                                returned_points=int(dev_counts.sum())),
                query_points_loop=dict(locations=min(loop, len(locs)), points=looped, s=loop_s, ms_per_location=loop_s * 1e3 / max(1, min(loop, len(locs)))),
                parity=parity)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=float, default=1e8)
    ap.add_argument("--locations", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop", type=int, default=100, help="locations of the query_points loop")
    a = ap.parse_args()
    import torch

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
    inten = (np.arange(n) % 1000).astype(np.float32)
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    log("octree: %d nodes" % len(tree.meta))
    cloud = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=20)
    log("S2 cloud: %d cells" % cloud.num_cells)
    del x, y, z, rgb, inten
    common = dict(card=name, power_limit=power, points=n, hbm_peak_bytes_per_s=HBM_BYTES_PER_S)
    sets = {"frusta_far10": make_frusta(G, bmin, bmax, a.locations, 10.0), "obbs": make_obbs(G, bmin, bmax, a.locations)}
    L = pcv._native.lib()
    for src_name, h, fn in (("octree", tree, L.pcv_query_batch_points_device), ("s2", cloud, L.pcv_s2_query_batch_points_device)):
        for set_name, locs in sets.items():
            log(src_name, set_name)
            r = run_set(torch, fn, h, locs, a.reps, a.loop)
            print(json.dumps(dict(common, source=src_name, locations_kind=set_name, **r)), flush=True)
    cloud.free()
    tree.free()
    ctx.close()


if __name__ == "__main__":
    main()
