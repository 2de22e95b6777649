"""build_octree in every division mode (build_modes.py) on the GPU, bit for bit against the oracle: every case in-core, the
narrow ones again through the generic partition kernel, three clouds of more than 4 194 304 points (those builds queue every
pass without reading the state back in between), and the degenerate and wild clouds through the one-rank sharded build and
the out-of-core build, whose prefix histograms run without the root cube and so in another mode than the builds they feed."""
import os

import numpy as np
import pytest

import build_modes as B
import oracle_api as O
from parity import compare_trees
from test_out_of_core_gpu import assert_same_dir
from test_sharded_native_gpu import SoloComm

pytestmark = pytest.mark.gpu


def _env(case, monkeypatch, generic=False):
    for k in ("PCV_CHECKED_FAST", "PCV_NO_POW2", "PCV_PASS_GENERIC", "PCV_NO_FUSED_PASS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)
    if generic:
        monkeypatch.setenv("PCV_PASS_GENERIC", "1")


def _oracle(case):
    return O.build(*case.columns(), case.rgb.reshape(-1, 3), case.res, case.bmin, case.bmax, intensity=case.inten, max_points_per_node=case.maxpts)


def _build_and_compare(case, monkeypatch, generic=False):
    import point_cloud_viewer_b200 as pcv

    _env(case, monkeypatch, generic)
    ctx = pcv.Context(0, max_points_per_node=case.maxpts)
    try:
        x, y, z, stride = case.xyz()
        tree = ctx.build_octree(x, y, z, case.rgb, case.res, case.bmin, case.bmax, intensity=case.inten, stride=stride, n=case.n)
        compare_trees(B.Bits(_oracle(case), oracle=True), B.Bits(tree))
        assert sum(m["num_points"] for m in tree.nodes.values()) == case.n
        tree.free()
    finally:
        ctx.close()


@pytest.mark.parametrize("case", B.CASES, ids=str)
def test_in_core_build_equals_oracle(case, monkeypatch):
    _build_and_compare(case, monkeypatch)


@pytest.mark.parametrize("case", [c for c in B.CASES if not c.wide], ids=str)
def test_generic_pass_kernel_equals_oracle(case, monkeypatch):
    """PCV_PASS_GENERIC=1: the mixed-encoding k_pass for every pass, in every mode."""
    _build_and_compare(case, monkeypatch, generic=True)


LARGE = [("zero", "wide", "degenerate"), ("ones", "narrow", "clean"), ("offset", "wide", "wild")]


@pytest.mark.parametrize("box_name,profile,cloud", LARGE, ids=["-".join(c) for c in LARGE])
def test_large_queued_build_equals_oracle(box_name, profile, cloud, monkeypatch):
    case = B.Case("large-%s-%s-%s" % (box_name, profile, cloud), box_name, profile, cloud, maxpts=5000, n=4_300_000, intensity=True, seed=101)
    assert case.n >= 4_194_304 and case.mode == B.BOX_MODE[box_name]
    _build_and_compare(case, monkeypatch)


SPLIT = [(b, c) for b in ("ones", "zero", "offset") for c in ("degenerate", "wild")]


def _split_case(box_name, cloud):
    return B.Case("split-%s-%s" % (box_name, cloud), box_name, "narrow", cloud, maxpts=2000, n=300_000, intensity=cloud == "wild", seed=7)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("box_name,cloud", SPLIT, ids=["-".join(c) for c in SPLIT])
def test_one_rank_sharded_build_equals_plain_build(box_name, cloud, fused, monkeypatch):
    import torch

    import point_cloud_viewer_b200 as pcv
    from point_cloud_viewer_b200 import distributed as D

    case = _split_case(box_name, cloud)
    _env(case, monkeypatch)
    if not fused:
        monkeypatch.setenv("PCV_NO_FUSED_PASS", "1")
    dev = torch.device("cuda", 0)
    ctx = pcv.Context(0, max_points_per_node=case.maxpts)
    x, y, z = [torch.from_numpy(c).to(dev) for c in case.columns()]
    rgb = torch.from_numpy(case.rgb).to(dev)
    inten = torch.from_numpy(case.inten).to(dev) if case.inten is not None else None
    single = ctx.build_octree(x.data_ptr(), y.data_ptr(), z.data_ptr(), rgb.data_ptr(), case.res, case.bmin, case.bmax,
                              intensity=inten.data_ptr() if inten is not None else None, n=case.n, device=True)
    comm = SoloComm(dev)
    tree = D.build_octree_sharded_native(ctx, x, y, z, rgb, inten, 0, case.res, case.bmin, case.bmax, prefix_levels=2, comm=comm)
    assert (ctx.shard_send_cells(tree.send_handle[1]) is not None) == (fused and tree.k == 2)
    merged = tree.gather_all(comm)
    assert set(single.nodes) == set(merged)
    for name, m in single.nodes.items():
        g = merged[name]
        assert (g["num_points"], g["enc"], tuple(g["cube"])) == (m["num_points"], m["enc"], tuple(m["cube"])), name
        if m["num_points"]:
            sx, sc, si, ss = single.node_data(name)
            assert np.array_equal(sx, g["xyz"]) and np.array_equal(sc, g["rgb"]) and np.array_equal(ss, g["src"]), name
            if inten is not None:
                assert np.array_equal(si.view(np.uint32), np.asarray(g["intensity"]).view(np.uint32)), name
    cs = tree.c_comm
    tree.free()
    ctx.sharded_release(cs)
    single.free()
    ctx.close()


@pytest.mark.parametrize("box_name,cloud", SPLIT, ids=["-".join(c) for c in SPLIT])
def test_out_of_core_build_equals_in_core_dir(box_name, cloud, monkeypatch, tmp_path):
    import point_cloud_viewer_b200 as pcv

    case = _split_case(box_name, cloud)
    _env(case, monkeypatch)
    ctx = pcv.Context(0, max_points_per_node=case.maxpts)
    try:
        x, y, z, stride = case.xyz()
        tree = ctx.build_octree(x, y, z, case.rgb, case.res, case.bmin, case.bmax, intensity=case.inten, stride=stride, n=case.n)
        tree.write_dir(tmp_path / "in_core")
        tree.free()
        info = ctx.build_octree_to_dir(tmp_path / "ooc", x, y, z, case.rgb, case.res, case.bmin, case.bmax, intensity=case.inten, stride=stride, n=case.n,
                                       max_points_in_core=case.n // 3)
        assert info["groups"] > 1 and info["num_points"] == case.n, info
        assert_same_dir(tmp_path / "ooc", tmp_path / "in_core")
    finally:
        ctx.close()
