"""bench.py --dump-outputs: the sampled slots map to the right nodes (CPU), and the dumped arrays equal what the octree's host
API returns for the same build (GPU)."""
import os

import numpy as np
import pytest

import bench


def _meta(counts, encs):
    import point_cloud_viewer_b200 as pcv

    m = np.zeros(len(counts), pcv.NODE_DTYPE)
    m["num_points"], m["enc"] = counts, encs
    m["point_offset"] = np.concatenate([[0], np.cumsum(counts)[:-1]])
    m["xyz_byte_offset"] = np.concatenate([[0], np.cumsum(np.asarray(counts) * 3 * np.array([0, 1, 2, 4, 8])[encs])[:-1]])
    return m


def test_sample_index_maps_slots_to_their_nodes():
    counts, encs = [0, 5, 0, 0, 7, 1, 0, 3], [1, 2, 1, 3, 4, 1, 2, 3]  # empty nodes share the offset of the next one
    m = _meta(counts, encs)
    slots, node, bpc, byte0 = bench.dump_sample_index(m, sum(counts), sample=1000)
    want = np.repeat(np.arange(len(counts)), counts)
    assert np.array_equal(slots, np.arange(sum(counts))) and np.array_equal(node, want)
    assert np.array_equal(bpc, np.array([0, 1, 2, 4, 8])[np.asarray(encs)[want]])
    assert np.array_equal(byte0, m["xyz_byte_offset"][want].astype(np.int64) + (slots - m["point_offset"][want].astype(np.int64)) * 3 * bpc)
    a = bench.dump_sample_index(m, sum(counts), sample=6)[0]
    assert len(a) == 6 and np.array_equal(a, np.unique(a)) and np.array_equal(a, bench.dump_sample_index(m, sum(counts), sample=6)[0])


@pytest.mark.gpu
def test_dump_outputs_equal_the_host_api(ctx, tmp_path):
    import torch

    import point_cloud_viewer_b200 as pcv

    kind = pcv.SYNTH_GAUSS_CLUSTERS
    n = 2_000_000
    x, y, z, rgb = pcv.synth_points_host(kind, bench.SEED, 0, n)
    bmin, bmax, res = pcv.synth_bbox(kind)
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax)
    bench.dump_outputs(tree, str(tmp_path), torch, torch.device("cuda", 0))
    d = {f[:-4]: np.load(os.path.join(tmp_path, f)) for f in os.listdir(tmp_path)}
    assert all(a.dtype in (np.float32, np.float64) for a in d.values()) and sum(a.nbytes for a in d.values()) <= bench.DUMP_LIMIT
    meta = tree.meta
    ids = d["node_id_words"].astype(np.uint64)
    assert np.array_equal((ids[:, 0] << np.uint64(32)) | ids[:, 1], meta["id_high"]) and np.array_equal((ids[:, 2] << np.uint64(32)) | ids[:, 3], meta["id_low"])
    for k in ("num_points", "level", "point_offset"):
        assert np.array_equal(d["node_" + k], meta[k].astype(np.float64)), k
    assert np.array_equal(d["node_encoding"], meta["enc"]) and np.array_equal(d["node_cube"], meta["cube"])
    slots = d["sample_slot"].astype(np.int64)
    assert len(slots) == bench.DUMP_SAMPLE and np.array_equal(slots, np.unique(slots))
    xyz, crgb, _, src = tree.download()
    assert np.array_equal(d["sample_src_index"], src[slots].astype(np.float64))
    assert np.array_equal(d["sample_rgb"], crgb.reshape(-1, 3)[slots].astype(np.float32))
    for m in meta:
        cnt = int(m["num_points"])
        lo, hi = np.searchsorted(slots, [int(m["point_offset"]), int(m["point_offset"]) + cnt])
        if hi == lo:
            continue
        dt = {1: "u1", 2: "<u2", 3: "<f4", 4: "<f8"}[int(m["enc"])]
        codes = xyz[int(m["xyz_byte_offset"]): int(m["xyz_byte_offset"]) + cnt * 3 * np.dtype(dt).itemsize].view(dt).reshape(cnt, 3)
        assert np.array_equal(d["sample_xyz_code"][lo:hi], codes[slots[lo:hi] - int(m["point_offset"])].astype(np.float64))
    tree.free()
