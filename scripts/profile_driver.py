"""One build of 1e8 benchmark points + one 200-frusta query batch + one 4096^2 X-ray tile: the kernels of the three measured
workloads, once each, for `ncu --set full`."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import point_cloud_viewer_b200 as pcv
import bench

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
dev = torch.device("cuda", 0)
kind = pcv.SYNTH_GAUSS_CLUSTERS
bmin, bmax, res = pcv.synth_bbox(kind)
ctx = pcv.Context(0)
x, y, z = [torch.empty(n, dtype=torch.float64, device=dev) for _ in range(3)]
rgb = torch.empty(n * 3, dtype=torch.uint8, device=dev)
ctx.synth_points_device(kind, 1, 0, n, x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr())
tree = ctx.build_octree(x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr(), res, bmin, bmax, n=n, device=True)
locs = bench.make_frusta(pcv.geometry, bmin, bmax, 200, 102.4)
counts, tested = tree.query_batch_device(locs)
ts = 256.0
tree.xray_tile((bmin[0] + ts, bmin[1] + 2 * ts, bmin[2]), (bmin[0] + 2 * ts, bmin[1] + 3 * ts, bmax[2]), 4096, 4096)
print("driver done: %d nodes, %d tested, %d returned" % (tree.num_nodes, int(tested.sum()), int(counts.sum())))
