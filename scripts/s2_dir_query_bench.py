"""python scripts/s2_dir_query_bench.py [--points N]

Point queries straight from an S2 directory at scale: N config-1 slab points (the ECEF slab generator on the host, seed 1; default
1e8) with colour and intensity, written by Context.build_s2_dir at level 20 into a temporary directory, then queried through
Context.open_s2_dir at two budgets: the default (most of the free memory) and about an eighth of the directory's size.  Calls:
cell unions of 1, 64 and 4096 cells (the level-20 cell of a sampled point, distinct level-22 and level-24 cells), the box, OBB
and frustum of point_cloud_test/src/queries.rs at the slab pose (query_points, the survivors counted in the callback), and 1000
frusta through query_batch.  Every call runs twice on a fresh handle; both are reported, so the first polyhedral call shows the
box scan (its bytes_read and ms_select include it).  For comparison: load_s2_dir, then the same calls on the resident cloud;
parity = equal survivors and tested points.  The directory was just written, so its files were likely in the page cache: the
reads are the page cache's, not the disk's (dropping caches is a system-wide setting and is not done here).  Not run: a
directory larger than device memory or than 2^32 points.  Prints one JSON line per (budget, call) and one for the resident
path; the card's name and power limit are read in the same run.  Progress goes to stderr."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

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
    print("[s2_dir_query_bench]", *a, file=sys.stderr, flush=True)


def frusta(G, bmin, bmax, count, far, seed=7):  # bench.make_frusta
    rng = np.random.default_rng(seed)
    persp = G.Perspective.new_fov(1.0, 1.2, 0.1, far)
    out = []
    for _ in range(count):
        eye = bmin + rng.random(3) * (bmax - bmin)
        q = rng.random((4, 12)).sum(1) - 6.0
        out.append(G.frustum(G.Isometry(eye, q / np.linalg.norm(q)), persp))
    return out


def run(q, what, loc):
    """One call on a handle or a resident cloud: (wall ms, survivors, tested)."""
    t = time.perf_counter()
    if what == "batch":
        counts, tested = (q.query_batch if hasattr(q, "query_batch") else q.query_batch_device)(loc)
        wall = (time.perf_counter() - t) * 1e3
        return wall, int(counts.sum()), int(tested.sum())
    got = [0]

    def cb(b):
        got[0] += len(b["src"])
        return False

    q.query_points(loc, callback=cb, batch_size=1 << 22)
    wall = (time.perf_counter() - t) * 1e3
    counts, tested = q.query_batch(loc if isinstance(loc, list) else [loc]) if hasattr(q, "query_batch") else q.query_batch_device([loc])
    return wall, got[0], int(tested[0])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=float, default=1e8)
    a = ap.parse_args()
    import point_cloud_viewer_b200 as pcv

    G = pcv.geometry
    name, power = card()
    n = int(a.points)
    ctx = pcv.Context(0)
    log("generating %d points on the host" % n)
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, SEED, 0, n)
    inten = (np.arange(n) % 1000).astype(np.float32)
    rng = np.random.default_rng(11)
    unions = {}
    for k, level in ((1, 20), (64, 22), (4096, 24)):
        pick = rng.integers(0, n, 8 * k)
        ids = np.unique(ctx.s2_cell_ids(x[pick], y[pick], z[pick], level))
        unions["union_%d" % k] = G.cell_union(rng.choice(ids, min(k, len(ids)), replace=False))
    tmp = tempfile.mkdtemp(prefix="s2_dir_query_bench_")
    try:
        d = os.path.join(tmp, "l20")
        t = time.perf_counter()
        ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=20)
        write_s = time.perf_counter() - t
        del x, y, z, rgb, inten
        dir_bytes = sum(os.path.getsize(os.path.join(d, f)) for f in os.listdir(d))
        log("directory: %.2f GB written in %.1f s" % (dir_bytes / 1e9, write_s))
        h = ctx.open_s2_dir(d)
        bmin, bmax = h.bbox_min, h.bbox_max
        h.close()
        dd = bmax - bmin
        q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
        e = G.Isometry((4157222.543, 664789.307, 4774952.099), q)
        calls = dict(unions)
        calls.update({  # point_cloud_test/src/queries.rs at the slab pose
            "aabb": G.aabb(bmin + 0.2 * dd, bmin + 0.8 * dd),
            "obb": G.obb(e, (50.0, 50.0, 5.0)),
            "frustum": G.frustum(e, G.Perspective.new_fov(1.0, 1.2, 0.1, 10.0)),
        })
        batch = frusta(G, bmin, bmax, 1000, 10.0)
        common = dict(card=name, power_limit=power, points=n, directory_bytes=dir_bytes, page_cache="likely (just written)")
        # the resident path: load, then every call twice
        t = time.perf_counter()
        cloud = ctx.load_s2_dir(d)
        load_ms = (time.perf_counter() - t) * 1e3
        resident = {}
        for label, loc in list(calls.items()) + [("frusta_1000", batch)]:
            what = "batch" if label == "frusta_1000" else "stream"
            resident[label] = [run(cloud, what, loc) for _ in range(2)]
        print(json.dumps(dict(common, path="load_s2_dir + resident", load_ms=load_ms,
                              calls={k: [dict(wall_ms=w, returned=r, tested=t_) for w, r, t_ in v] for k, v in resident.items()})), flush=True)
        cloud.free()
        ctx.release_cached_memory()
        for budget in (0, dir_bytes // 8):
            for label, loc in list(calls.items()) + [("frusta_1000", batch)]:
                what = "batch" if label == "frusta_1000" else "stream"
                try:
                    hh = ctx.open_s2_dir(d, budget)
                except pcv.PcvError as err:
                    print(json.dumps(dict(common, budget=budget, query=label, error=str(err))), flush=True)
                    continue
                reps = []
                for _ in range(2):
                    if what == "batch":
                        w, r, t_ = run(hh, what, loc)
                        st = hh.last_stats()
                    else:
                        t = time.perf_counter()
                        got = [0]
                        hh.query_points(loc, callback=lambda b: got.__setitem__(0, got[0] + len(b["src"])) or False, batch_size=1 << 22)
                        w = (time.perf_counter() - t) * 1e3
                        st = hh.last_stats()
                        r, t_ = got[0], int(st["tested_points"])
                    reps.append(dict(wall_ms=w, returned=r, tested=t_, **{k: st[k] for k in ("bytes_read", "ms_select", "ms_read_wait", "ms_cull", "peak_device_bytes",
                                                                                            "max_device_bytes", "chunks")}))
                hh.close()
                want = resident[label][0]
                parity = all(x_["returned"] == want[1] and x_["tested"] == want[2] for x_ in reps)
                print(json.dumps(dict(common, budget=budget, query=label, first=reps[0], repeat=reps[1], resident_wall_ms=[v[0] for v in resident[label]],
                                      parity=parity)), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
