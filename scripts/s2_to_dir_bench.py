"""S2 directories straight from host memory (pcv_s2_build_to_dir) against the in-core build + write_dir, on synthetic slab points
at split level 20.  Prints one JSON line per row: points/s end to end, the split's device time, the device's wait for input,
the wait for the writers, the peak device bytes, the batches, and the card's name and power limit read in the same run.

    python scripts/s2_to_dir_bench.py --n 100000000 --big 1200000000 --out /tmp/s2bench
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import point_cloud_viewer_b200 as pcv  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def points(n, chunk=50_000_000):
    x, y, z = np.empty(n), np.empty(n), np.empty(n)
    rgb = np.empty(3 * n, np.uint8)
    for f in range(0, n, chunk):
        m = min(chunk, n - f)
        a, b, c, r = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, f, m)
        x[f:f + m], y[f:f + m], z[f:f + m], rgb[3 * f:3 * (f + m)] = a, b, c, r
    inten = (np.arange(n, dtype=np.uint64) % 511).astype(np.float32)
    return x, y, z, rgb, inten


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--big", type=int, default=0, help="points of the row above one in-core build (0: skip)")
    ap.add_argument("--out", default="/tmp/s2_to_dir_bench")
    ap.add_argument("--level", type=int, default=20)
    a = ap.parse_args()
    ctx = pcv.Context(0)
    gpu = card()
    rows = []

    def emit(r):
        r["card"] = gpu
        print(json.dumps(r), flush=True)
        rows.append(r)

    x, y, z, rgb, inten = points(a.n)
    d = os.path.join(a.out, "stream")
    shutil.rmtree(a.out, ignore_errors=True)
    os.makedirs(a.out)
    ctx.build_s2_dir(os.path.join(a.out, "warm"), x[:1_000_000], y[:1_000_000], z[:1_000_000], rgb[:3_000_000], inten[:1_000_000], split_level=a.level)
    info = ctx.build_s2_dir(d, x, y, z, rgb, inten, split_level=a.level)
    emit({"row": "stream", "n": a.n, "points_per_s": a.n / info["ms_total"] * 1e3, **{k: info[k] for k in ("ms_total", "ms_split", "ms_input_wait", "ms_write_wait",
                                                                                                              "peak_device_bytes", "batches", "num_cells")}})
    shutil.rmtree(d)
    t0 = time.perf_counter()
    c = ctx.build_s2_cloud(x, y, z, rgb, inten, split_level=a.level)
    t1 = time.perf_counter()
    c.write_dir(os.path.join(a.out, "incore"))
    t2 = time.perf_counter()
    c.free()
    emit({"row": "in_core+write_dir", "n": a.n, "points_per_s": a.n / (t2 - t0), "ms_total": (t2 - t0) * 1e3, "ms_build": (t1 - t0) * 1e3, "ms_write": (t2 - t1) * 1e3})
    shutil.rmtree(os.path.join(a.out, "incore"))
    del x, y, z, rgb, inten
    if a.big:
        x, y, z, rgb, inten = points(a.big)
        info = ctx.build_s2_dir(os.path.join(a.out, "big"), x, y, z, rgb, inten, split_level=a.level)
        emit({"row": "stream_big", "n": a.big, "points_per_s": a.big / info["ms_total"] * 1e3, **{k: info[k] for k in ("ms_total", "ms_split", "ms_input_wait",
                                                                                                                          "ms_write_wait", "peak_device_bytes",
                                                                                                                          "batches", "num_cells")}})
    shutil.rmtree(a.out, ignore_errors=True)
    ctx.close()


if __name__ == "__main__":
    main()
