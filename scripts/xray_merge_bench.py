"""Merging partial X-ray quadtrees (Context.merge_xray_quadtrees): the sub-root-then-merge workflow on one GPU.

A config-2 octree of --points points is built resident; for every tile size and root level given, every sub-root at that level
is written with xray_quadtree_write_dir(root=(L, i)) into one shared directory, and the pieces are merged into a fresh
directory.  The pixel size is chosen per tile size so that the deepest level is --deepest-256 (256 px) or --deepest-big (the
other sizes), which keeps the leaves' PNG volume affordable at 4096 px.  For every case one JSON line gives the card and its
power limit (read in the same run), the sub-root build time, the merge's copy, decode, parent-kernel and encode/write times,
its peak device bytes, and the CPU time of the oracle's build_parent + Lanczos3 for the same parents (tests/oracle_api.py)."""
import argparse
import io
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


def log(*a):
    print("[xray_merge_bench]", *a, file=sys.stderr, flush=True)


def oracle_parents_s(inputs, background):
    """CPU seconds of the oracle's parents over the same sub-roots (their PNG decoding not counted)."""
    import numpy as np
    from PIL import Image

    import oracle_api as O
    import xray_merge_ref as R

    metas, pngs = [], {}
    for d in inputs:
        for name in sorted(os.listdir(d)):
            if name.startswith("meta") and name.endswith(".pb"):
                metas.append(R.read_meta(open(os.path.join(d, name), "rb").read()))
            elif name.endswith(".png"):
                pngs[name] = os.path.join(d, name)
    _, (L, _, T, _, roots, parents, _) = R.plan(metas)
    tiles = {r: np.asarray(Image.open(io.BytesIO(open(pngs[R.node_name(*r) + ".png"], "rb").read())).convert("RGBA")) for r in roots}
    t = time.perf_counter()
    for level in range(L - 1, -1, -1):
        for (l, i) in sorted(q for q in parents if q[0] == level):
            tiles[(l, i)] = O.build_parent_tile([tiles.get((l + 1, 4 * i + k)) for k in range(4)], background, T)
    return time.perf_counter() - t, len(parents)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=float, default=1e8)
    ap.add_argument("--tiles", default="256,4096")
    ap.add_argument("--levels", default="2,3")
    ap.add_argument("--deepest-256", type=int, default=6)
    ap.add_argument("--deepest-big", type=int, default=3)
    ap.add_argument("--no-oracle", action="store_true")
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
    tmp = tempfile.mkdtemp(prefix="xray_merge_bench_", dir=a.tmp)
    try:
        for T in [int(v) for v in a.tiles.split(",")]:
            deepest = a.deepest_256 if T <= 256 else a.deepest_big
            px = ext / T / 2 ** deepest * 0.999  # the deepest level is `deepest`
            for L in [int(v) for v in a.levels.split(",")]:
                inp, out = os.path.join(tmp, "in_%d_%d" % (T, L)), os.path.join(tmp, "out_%d_%d" % (T, L))
                t = time.perf_counter()
                for i in range(4 ** L):
                    tree.xray_quadtree_write_dir(inp, T, px, root=(L, i))
                build_s = time.perf_counter() - t
                t = time.perf_counter()
                info = ctx.merge_xray_quadtrees(inp, out)
                merge_s = time.perf_counter() - t
                row = dict(card=name, power_limit=power, points=n, tile_px=T, root_level=L, deepest_level=info["deepest_level"], sub_roots=4 ** L,
                           metas_empty=info["metas_empty"], sub_root_builds_s=round(build_s, 2), merge_s=round(merge_s, 3), files_copied=info["files_copied"],
                           bytes_copied=info["bytes_copied"], roots_decoded=info["roots_decoded"], parents_built=info["parents_built"],
                           ms_copy=round(info["ms_copy"], 1), ms_decode_summed=round(info["ms_decode"], 1), ms_parents=round(info["ms_parents"], 2),
                           ms_write_summed=round(info["ms_write"], 1), ms_total=round(info["ms_total"], 1), peak_device_bytes=info["peak_device_bytes"],
                           device_bytes_needed=info["device_bytes_needed"])
                if not a.no_oracle and info["parents_built"]:
                    s, k = oracle_parents_s([inp], (255, 255, 255, 255))
                    row.update(oracle_parents_s=round(s, 2), oracle_parents=k)
                print(json.dumps(row), flush=True)
                shutil.rmtree(inp, ignore_errors=True)
                shutil.rmtree(out, ignore_errors=True)
    finally:
        tree.free()
        ctx.close()
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
