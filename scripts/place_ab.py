"""A/B of two builds of the library on the benchmark's build (config 2: Gaussian clusters, device-resident inputs, default
N = 5e8), e.g. a build of the parent commit against the tree's own.  Each round runs every library in its own process (the
order alternates between rounds): W warm-up builds, S timed builds with CUDA events around each call as bench.py takes them,
then one profiled build for the per-kernel times and a fingerprint of everything the last build wrote (position codes,
colours, source indices), so that the two libraries can be seen to compute the same octree.

    python scripts/place_ab.py --lib-a /path/to/parent/libpcv_b200.so [--lib-b in-tree] [--rounds 5] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 1  # bench.py's generator seed


def fingerprint(torch, tree, dev):
    """Position-weighted sums of the octree's device arrays, read as 32-bit words in 64 MB chunks (wrapping int64 arithmetic)."""
    import ctypes as C

    from point_cloud_viewer_b200 import _native as N
    from point_cloud_viewer_b200.distributed import _RawCuda

    p = [C.c_void_p() for _ in range(4)]
    N.check(N.lib().pcv_octree_device_arrays(tree.h, *[C.byref(v) for v in p]))
    arrays = {"xyz": (p[0].value, int(tree.xyz_bytes)), "rgb": (p[1].value, 3 * int(tree.num_points)), "src": (p[3].value, 4 * int(tree.num_points))}
    out = {}
    for name, (ptr, nbytes) in arrays.items():
        raw = torch.as_tensor(_RawCuda(ptr, (nbytes,), "|u1"), device=dev)
        acc, chunk = 0, 64 << 20
        for o in range(0, nbytes, chunk):
            b = raw[o:o + chunk]
            if b.numel() % 4:
                b = torch.cat([b, torch.zeros(4 - b.numel() % 4, dtype=torch.uint8, device=dev)])
            w = b.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
            k = torch.arange(o // 4, o // 4 + w.numel(), device=dev, dtype=torch.int64)
            acc = (acc + int((w * (k % 1000003 + 1)).sum().item())) & 0xFFFFFFFFFFFFFFFF
        out[name] = "%016x" % acc
    return out


def child(args):
    import torch

    sys.path.insert(0, ROOT)
    import point_cloud_viewer_b200 as pcv

    dev = torch.device("cuda", 0)
    n = int(args.points)
    kind = pcv.SYNTH_GAUSS_CLUSTERS
    bmin, bmax, res = pcv.synth_bbox(kind)
    ctx = pcv.Context(0)
    xs = [torch.empty(n, dtype=torch.float64, device=dev) for _ in range(3)]
    rgb = torch.empty(n * 3, dtype=torch.uint8, device=dev)
    ctx.synth_points_device(kind, SEED, 0, n, xs[0].data_ptr(), xs[1].data_ptr(), xs[2].data_ptr(), rgb.data_ptr())

    def step():
        return ctx.build_octree(xs[0].data_ptr(), xs[1].data_ptr(), xs[2].data_ptr(), rgb.data_ptr(), res, bmin, bmax, n=n, device=True)

    for _ in range(args.warmup):
        step().free()
    step_ms, place_ms, last = [], [], None
    for _ in range(args.steps):
        if last is not None:
            last.free()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        last = step()
        torch.cuda.synchronize()
        e1.record()
        torch.cuda.synchronize()
        step_ms.append(e0.elapsed_time(e1))
        place_ms.append(ctx.last_build_stats()["ms_place"])
    fp = fingerprint(torch, last, dev)
    nodes = int(last.num_nodes)
    last.free()
    ctx.set_profiling(True)
    step().free()
    ks = {k: {"ms": v["ms"], "launches": v["launches"], "algorithmic_bytes": v["algorithmic_bytes"]} for k, v in ctx.kernel_stats().items()}
    ctx.set_profiling(False)
    print(json.dumps({"step_ms": step_ms, "ms_place": place_ms, "kernels": ks, "fingerprint": fp, "nodes": nodes}), flush=True)
    ctx.close()


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers stay usable without it
        return "unknown (%s)" % e


def spread(v):
    return max(v) - min(v) if v else 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib-a", help="library A (e.g. a build of the parent commit); required")
    ap.add_argument("--lib-b", default=os.path.join(ROOT, "point_cloud_viewer_b200", "libpcv_b200.so"), help="library B (default: the tree's own)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--points", type=float, default=5e8)
    ap.add_argument("--out", help="write the per-round results and the summary as JSON")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    if not args.lib_a:
        ap.error("--lib-a is required")

    libs = {"A": os.path.abspath(args.lib_a), "B": os.path.abspath(args.lib_b)}
    card = gpu_info()
    print("card: %s | A = %s | B = %s | N = %.3g, %d rounds of %d warm-up + %d timed builds" % (card, libs["A"], libs["B"], args.points, args.rounds, args.warmup, args.steps), flush=True)
    rounds = []
    for r in range(args.rounds):
        row = {}
        for name in ("AB" if r % 2 == 0 else "BA"):
            env = dict(os.environ, PCV_B200_LIB=libs[name])
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--points", str(args.points), "--warmup", str(args.warmup), "--steps", str(args.steps)]
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
            if p.returncode != 0 or not lines:
                sys.exit("round %d, library %s failed (rc %d):\n%s" % (r, name, p.returncode, (p.stderr or p.stdout)[-2000:]))
            row[name] = json.loads(lines[-1])
        rounds.append(row)
        print("round %d: " % r + " | ".join("%s step %.2f ms, ms_place %.2f, k_place %.2f ms" % (
            k, statistics.median(row[k]["step_ms"]), statistics.median(row[k]["ms_place"]), row[k]["kernels"]["k_place"]["ms"]) for k in "AB"), flush=True)

    summary = {"card": card, "points": args.points, "rounds": args.rounds, "libs": libs}
    for k in "AB":
        step = [statistics.median(rw[k]["step_ms"]) for rw in rounds]
        place = [statistics.median(rw[k]["ms_place"]) for rw in rounds]
        kern = {kn: [rw[k]["kernels"][kn]["ms"] for rw in rounds] for kn in rounds[0][k]["kernels"]}
        summary[k] = {"step_ms": {"median": statistics.median(step), "spread": spread(step)},
                      "ms_place": {"median": statistics.median(place), "spread": spread(place)},
                      "kernels": {kn: {"median": statistics.median(v), "spread": spread(v)} for kn, v in kern.items() if max(v) > 0}}
    kp = rounds[0]["B"]["kernels"]["k_place"]
    peak = 3.35e12  # H100 SXM data-sheet HBM3 bandwidth
    for k in "AB":
        ms = summary[k]["kernels"]["k_place"]["median"]
        summary[k]["k_place_hbm_share"] = kp["algorithmic_bytes"] / (ms * 1e-3) / peak if ms > 0 else None
    fps = {k: {json.dumps(rw[k]["fingerprint"], sort_keys=True) for rw in rounds} for k in "AB"}
    summary["same_outputs"] = len(fps["A"]) == 1 and fps["A"] == fps["B"]
    summary["fingerprint"] = {k: sorted(v) for k, v in fps.items()}

    print("\n%-14s %22s %22s %10s" % ("median (spread)", "A", "B", "B - A"))
    for label, key in (("step ms", "step_ms"), ("ms_place", "ms_place")):
        a, b = summary["A"][key], summary["B"][key]
        print("%-14s %14.2f (%5.2f) %14.2f (%5.2f) %+10.2f" % (label, a["median"], a["spread"], b["median"], b["spread"], b["median"] - a["median"]))
    for kn in sorted(summary["A"]["kernels"], key=lambda s: -summary["A"]["kernels"][s]["median"]):
        a, b = summary["A"]["kernels"][kn], summary["B"]["kernels"].get(kn, {"median": 0.0, "spread": 0.0})
        print("%-14s %14.2f (%5.2f) %14.2f (%5.2f) %+10.2f" % (kn, a["median"], a["spread"], b["median"], b["spread"], b["median"] - a["median"]))
    print("k_place share of data-sheet HBM (%.1f GB): A %.2f, B %.2f" % (kp["algorithmic_bytes"] / 1e9, summary["A"]["k_place_hbm_share"], summary["B"]["k_place_hbm_share"]))
    print("outputs identical across libraries and rounds: %s" % summary["same_outputs"])
    print("card: %s" % card)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"summary": summary, "rounds": rounds}, f, indent=1)


if __name__ == "__main__":
    main()
