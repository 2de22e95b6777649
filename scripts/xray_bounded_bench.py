"""python scripts/xray_bounded_bench.py [--points N] [--tile-px T] [--over F] [--dir PARENT] [--write-root-level L]

The bounded X-ray quadtree at scale: N config-2 points (the benchmark's generator, seed 1) are built into a device-resident
octree, then build_xray_quadtree runs with T-px tiles (default 256) at the largest power-of-two fraction of the map's extent
per tile that makes the created leaves' images F times the card's memory (default 1.2), under max_device_bytes = those bytes
/ 8.  Prints one JSON line: leaves, parents and nodes; device ms of the leaves and of the parents; wall seconds of the call
delivering every tile to a callback and of the bounded write_dir (PNG files under PARENT, removed afterwards; with
--write-root-level L only the first non-empty subtree at level L is written, which the line says); tiles per second; the
peak of the driver's device memory and the leaf positions it evaluated; the card and its power limit; and a verdict: 256
sampled created leaves equal pcv_xray_tile + assign_background, sampled parents equal pcv_xray_build_parent of their delivered
children, every tile comes after its children and once, and the created leaves' bytes exceed the card's memory.  Progress
goes to stderr."""
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
WHITE = (255, 255, 255, 255)


def card():
    """(name, power limit) of GPU 0, read in the same run as the measurement."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, power = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:
        return None, "unknown (%s)" % str(e)[:80]


def log(*a):
    print("[xray_bounded_bench]", *a, file=sys.stderr, flush=True)


def mix(level, index):
    return ((index * 0x9E3779B97F4A7C15 + level * 0xBF58476D1CE4E5B9) >> 17) & 0xFFFFFFFF


def leaf_rect(info, i, deepest):
    mnx, mny, e = info["rect_min_x"], info["rect_min_y"], info["rect_edge"]
    for lv in range(deepest - 1, -1, -1):  # quad_rect_of: child bit 0 -> +y, bit 1 -> +x
        k = (i >> (2 * lv)) & 3
        e = e / 2.0
        mny += e if k & 1 else 0.0
        mnx += e if k & 2 else 0.0
    return mnx, mny, e


def run(n, T, over, base_dir, write_root_level):
    import numpy as np
    import torch

    import point_cloud_viewer_b200 as pcv

    kind = pcv.SYNTH_GAUSS_CLUSTERS
    bmin, bmax, res = pcv.synth_bbox(kind)
    ctx = pcv.Context(0)
    x, y, z = (torch.empty(n, dtype=torch.float64, device="cuda") for _ in range(3))
    rgb = torch.empty(3 * n, dtype=torch.uint8, device="cuda")
    ctx.synth_points_device(kind, SEED, 0, n, x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr())
    total_mem = torch.cuda.get_device_properties(0).total_memory
    tbytes = T * T * 4
    # the pixel size: leaves of edge T * px on the grid from the box's minimum, as find_quadtree_bounding_rect_and_levels lays them
    extent = max(bmax[0] - bmin[0], bmax[1] - bmin[1])
    px, leaves_est = extent / T, 1
    while leaves_est * tbytes < over * total_mem:
        px /= 2.0
        e = T * px
        key = torch.floor((x - bmin[0]) / e).to(torch.int64) * (1 << 31) + torch.floor((y - bmin[1]) / e).to(torch.int64)
        leaves_est = int(torch.unique(key).numel())
        del key
        log("pixel size %.6g m: %d occupied leaves (%.1f GB of images)" % (px, leaves_est, leaves_est * tbytes / 1e9))
    budget = leaves_est * tbytes // 8
    tree = ctx.build_octree(x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr(), res, bmin, bmax, n=n, device=True)
    del x, y, z, rgb
    torch.cuda.empty_cache()
    log("octree of %d points: %d nodes; quadtree at %d px, %.6g m per pixel, max_device_bytes %d" % (n, len(tree.nodes), T, px, budget))
    name, power = card()
    # sampled leaves and parents (by a hash of the id); a parent's children are kept when they arrive, before it
    k_leaf = max(1, leaves_est // 256)
    k_par = max(1, leaves_est // 4 // 64)
    order, kept = [], {}
    deepest_box = [None]

    def sampled_parent(level, index):
        return level >= 0 and mix(level, index) % k_par == 0

    def on_tile(level, index, img):
        order.append((level, index))
        if deepest_box[0] is None:
            deepest_box[0] = level  # the first tile delivered is a leaf
        if (level == deepest_box[0] and mix(level, index) % k_leaf == 0) or sampled_parent(level - 1, index >> 2) or (
                level < deepest_box[0] and sampled_parent(level, index)):
            kept[(level, index)] = img.copy()
        return False

    w0 = time.perf_counter()
    info, _ = tree.xray_quadtree(T, px, on_tile=on_tile, keep_tiles=False, max_device_bytes=budget)
    wall = time.perf_counter() - w0
    deepest = info["deepest_level"]
    log("quadtree in %.1f s: %s" % (wall, info))
    # verdict
    pos = {k: i for i, k in enumerate(order)}
    post_order = len(pos) == len(order) and all(pos[(l + 1, (i << 2) + c)] < p for (l, i), p in pos.items() for c in range(4) if (l + 1, (i << 2) + c) in pos)
    leaves_ok, nleaf_checked = True, 0
    for (l, i), img in kept.items():
        if l != deepest or mix(l, i) % k_leaf:
            continue
        mnx, mny, e = leaf_rect(info, i, deepest)
        _, want, _ = tree.xray_tile((mnx, mny, bmin[2]), (mnx + e, mny + e, bmax[2]), T, T)
        leaves_ok = leaves_ok and bool(np.array_equal(img, pcv.xray_assign_background(ctx, want, WHITE)))
        nleaf_checked += 1
    parents_ok, npar_checked = True, 0
    for (l, i), img in kept.items():
        if l < deepest and sampled_parent(l, i):
            ch = [kept.get((l + 1, (i << 2) + c)) for c in range(4)]
            parents_ok = parents_ok and bool(np.array_equal(img, pcv.xray_build_parent(ctx, ch, WHITE, T)))
            npar_checked += 1
    leaf_bytes = info["num_leaves"] * tbytes
    # write_dir
    d = tempfile.mkdtemp(prefix="pcv_xray_", dir=base_dir)
    root = (0, 0)
    if write_root_level:
        root = (write_root_level, min(i >> (2 * (deepest - write_root_level)) for (l, i) in order if l == deepest))
    try:
        w0 = time.perf_counter()
        winfo = tree.xray_quadtree_write_dir(d, T, px, root=root, max_device_bytes=budget)
        wall_dir = time.perf_counter() - w0
        files = len(os.listdir(d))
    finally:
        shutil.rmtree(d, ignore_errors=True)
    log("write_dir of %s in %.1f s: %d files" % (root, wall_dir, files))
    out = {"n": n, "tile_px": T, "pixel_size_m": px, "deepest_level": deepest, "leaves": info["num_leaves"], "parents": info["num_nodes"] - info["num_leaves"],
           "nodes": info["num_nodes"], "ms_leaves": info["ms_leaves"], "ms_parents": info["ms_parents"], "wall_s": wall,
           "tiles_per_s": info["num_nodes"] / wall, "write_dir": {"root": list(root), "nodes": winfo["num_nodes"], "files": files, "wall_s": wall_dir,
                                                                  "tiles_per_s": winfo["num_nodes"] / wall_dir},
           "max_device_bytes": info["max_device_bytes"], "peak_device_bytes": info["peak_device_bytes"], "block_level": info["block_level"],
           "blocks_processed": info["blocks_processed"], "positions_evaluated": info["positions_evaluated"], "key_batches": info["key_batches"],
           "created_leaf_bytes": leaf_bytes, "card_memory_bytes": total_mem, "gpu": name, "power_limit": power,
           "verdict": {"ok": leaves_ok and parents_ok and post_order and leaf_bytes > total_mem and nleaf_checked > 0 and npar_checked > 0,
                       "sampled_leaves_equal_xray_tile": leaves_ok, "leaves_checked": nleaf_checked, "sampled_parents_equal_build_parent": parents_ok,
                       "parents_checked": npar_checked, "post_order": post_order, "created_leaf_bytes_exceed_card_memory": leaf_bytes > total_mem,
                       "peak_within_budget": info["peak_device_bytes"] <= info["max_device_bytes"]}}
    tree.free()
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=float, default=2e8)
    ap.add_argument("--tile-px", type=int, default=256)
    ap.add_argument("--over", type=float, default=1.2, help="created leaves' images over the card's memory")
    ap.add_argument("--dir", default=None, help="parent of the temporary write_dir output (default: the system temporary directory)")
    ap.add_argument("--write-root-level", type=int, default=0, help="write only the first non-empty subtree at this level (0: the whole quadtree)")
    args = ap.parse_args()
    print(json.dumps({"xray_bounded": run(int(args.points), args.tile_px, args.over, args.dir, args.write_root_level)}))


if __name__ == "__main__":
    main()
