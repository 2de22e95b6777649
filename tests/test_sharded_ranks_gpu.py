"""The sharded build with 2, 3, 4 and 8 ranks on one GPU: every rank is its own process on device 0, the collectives go over gloo
through host memory, and the library's kernels store into the peer slabs of the other processes through CUDA IPC, as they do
across GPUs.  Every case of sharded_cases.py runs each of its paths; the merged tree must equal the single build of the whole
cloud bit for bit, provenance included, and each path must report that it actually ran."""
import os
import pickle
import sys
import time

import numpy as np
import pytest

import sharded_cases as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT_S = 120


def _comm_class():
    import torch

    from point_cloud_viewer_b200 import distributed as D

    class HostStagedComm(D.TorchComm):
        """TorchComm on the CPU device for gloo: device tensors cross the all-to-all through host memory, and every barrier waits
        for this process's device work first (the peers read what its kernels stored)."""

        def __init__(self):
            super().__init__(torch.device("cpu"))

        def all_to_all(self, tensor, send_counts, recv_counts, alloc=None):
            out = super().all_to_all(tensor.cpu(), send_counts, recv_counts)
            return out.to(tensor.device)

        def barrier(self):
            torch.cuda.synchronize()
            self.dist.barrier()

        def done_with(self, *tensors):
            torch.cuda.synchronize()
            for t in tensors:
                owner = getattr(t, "_pcv_owner", None) if t is not None else None
                if owner is not None:
                    owner.free()

    return HostStagedComm


def _set_env(env):
    for k in S.ENV_KEYS:
        os.environ.pop(k, None)
    os.environ.update(env)


def _ran(ctx, tree, path):
    """Which exchange the build reports it ran."""
    if path in ("fused", "records"):
        fused = ctx.sharded_phases()["fused_exchange_pass"]
        assert fused == (ctx.shard_send_cells(tree.send_handle[1]) is not None), "phases and send handle disagree"
        return "fused" if fused else "records"
    ph = tree.phases_ms
    return "py" if "ingest + histogram" in ph else "pyx" if "pack+exchange" in ph else "staged" if "all_to_all" in ph else "?"


def _worker(rank, world, store_path, out_dir):
    for p in (ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(S.WORLD_ENV.get(world, {}))
    import datetime

    import torch
    import torch.distributed as dist

    dist.init_process_group("gloo", store=dist.FileStore(store_path, world), rank=rank, world_size=world, timeout=datetime.timedelta(seconds=TIMEOUT_S))
    import point_cloud_viewer_b200 as pcv
    from point_cloud_viewer_b200 import distributed as D

    comm = _comm_class()()
    dev = torch.device("cuda", 0)
    ctxs, c_comms = {}, {}  # the maximum node size is a property of the context: one context per size, kept for the whole world
    for case in S.CASES[world]:
        ctx = ctxs.get(case.maxpts) or ctxs.setdefault(case.maxpts, pcv.Context(0, max_points_per_node=case.maxpts))
        P, rgb, inten, res, bmin, bmax = case.data()
        lo, hi = case.ranges()[rank]
        x, y, z = [torch.from_numpy(np.ascontiguousarray(P[lo:hi, a])).to(dev) for a in range(3)]
        c = torch.from_numpy(rgb[3 * lo:3 * hi].copy()).to(dev)
        it = torch.from_numpy(inten[lo:hi].copy()).to(dev) if inten is not None else None
        if case.release_before:
            ctx.sharded_release(c_comms[case.maxpts])
        for path in case.paths:
            _set_env(case.path_env(path))
            if path in ("fused", "records"):
                tree = D.build_octree_sharded_native(ctx, x, y, z, c, it, lo, res, bmin, bmax, prefix_levels=case.k, comm=comm)
                c_comms[case.maxpts] = tree.c_comm
            else:
                ops = D.CudaOps(ctx, x, y, z, c, it, res, bmin, bmax)
                tree = D.build_sharded(ops, comm, lo, prefix_levels=case.k, max_points_per_node=case.maxpts)
            ran = _ran(ctx, tree, path)
            nodes = tree.gather_all(comm)
            info = comm.all_gather_objects(dict(k=tree.k, c2r=np.asarray(tree.cell_to_rank).tolist(), recv=int(tree.recv_points), ran=ran))
            tree.free()
            if rank == 0:
                with open(os.path.join(out_dir, "%s.%s.pkl" % (case.name, path)), "wb") as f:
                    pickle.dump(dict(nodes=nodes, ranks=info), f)
    for maxpts, ctx in ctxs.items():
        if maxpts in c_comms:
            ctx.sharded_release(c_comms[maxpts])
        _close_python_slabs(ctx, comm)
        ctx.close()
    dist.barrier()
    dist.destroy_process_group()


def _close_python_slabs(ctx, comm):
    from point_cloud_viewer_b200 import distributed as D

    for cls in (D.RecordSlab, D.PeerSlab):
        slab = cls._cache.get(id(ctx))
        if slab is not None:
            slab.close(comm)


def _spawn(world, tmp_path):
    """Runs the world's ranks; returns (output directory, most device memory in use while they ran)."""
    import threading

    import torch
    import torch.multiprocessing as mp

    out = tmp_path / ("r%d" % world)
    out.mkdir()
    peak, stop = [0], threading.Event()

    def sample():
        while not stop.wait(0.2):
            free, total = torch.cuda.mem_get_info(0)
            peak[0] = max(peak[0], total - free)

    sampler = threading.Thread(target=sample, daemon=True)
    sampler.start()
    pc = mp.start_processes(_worker, args=(world, str(tmp_path / ("store%d" % world)), str(out)), nprocs=world, join=False, start_method="spawn")
    deadline = time.monotonic() + 60 * 15
    try:
        while not pc.join(timeout=5):
            assert time.monotonic() < deadline, "world %d timed out" % world
    finally:
        stop.set()
        sampler.join()
        for p in pc.processes:
            if p.is_alive():
                p.terminate()
        for p in pc.processes:
            p.join(30)
            if p.is_alive():
                p.kill()
                p.join()
    return out, peak[0]


def _compare(case, got, single, ref, plan):
    P = case.data()[0]
    nodes, ranks = got["nodes"], got["ranks"]
    for r, info in enumerate(ranks):
        assert info["k"] == plan["k"], (r, info["k"], plan["k"])
        assert np.array_equal(np.asarray(info["c2r"]), plan["c2r"]), (r, "cell_to_rank")
    assert [info["recv"] for info in ranks] == [int(v) for v in plan["M"].sum(0)]
    assert sum(info["recv"] for info in ranks) == len(P)
    for tree in [single] + ([ref] if ref is not None else []):
        assert set(tree.nodes) == set(nodes), sorted(set(tree.nodes) ^ set(nodes))[:10]
        for name, m in tree.nodes.items():
            g = nodes[name]
            assert (g["num_points"], g["enc"], tuple(g["cube"])) == (m["num_points"], m["enc"], tuple(m["cube"])), name
            if m["num_points"]:
                sx, sc, si, ss = tree.node_data(name, case.intensity) if tree is ref else tree.node_data(name)
                assert np.array_equal(ss, g["src"]), (name, "provenance")
                assert np.array_equal(sx, g["xyz"]) and np.array_equal(sc, g["rgb"]), name
                if si is not None or g.get("intensity") is not None:
                    assert np.array_equal(np.asarray(si).view(np.uint32), np.asarray(g["intensity"]).view(np.uint32)), name


@pytest.mark.parametrize("world", sorted(S.CASES))
def test_ranks_on_one_gpu_equal_single_build(world, tmp_path):
    import oracle_api as O
    import point_cloud_viewer_b200 as pcv

    t0 = time.monotonic()
    out, peak = _spawn(world, tmp_path)
    t_spawn = time.monotonic() - t0
    ran = set()
    for case in S.CASES[world]:
        P, rgb, inten, res, bmin, bmax = case.data()
        plan = S.plan(case)
        for k, v in case.env.items():
            os.environ[k] = v
        try:
            ctx = pcv.Context(0, max_points_per_node=case.maxpts)
            cols = [np.ascontiguousarray(P[:, a]) for a in range(3)]
            single = ctx.build_octree(*cols, rgb, res, bmin, bmax, intensity=inten)
            ref = O.build(*cols, rgb.reshape(-1, 3), res, bmin, bmax, intensity=inten, max_points_per_node=case.maxpts) if len(P) <= 300_000 else None
            for path in case.paths:
                got = pickle.load(open(out / ("%s.%s.pkl" % (case.name, path)), "rb"))
                want = "records" if (path == "fused" and plan["k"] != 2) else path
                assert all(info["ran"] == want for info in got["ranks"]), (case, path, [info["ran"] for info in got["ranks"]])
                ran.add(want)
                try:
                    _compare(case, got, single, ref, plan)
                except AssertionError as e:
                    raise AssertionError("%s, path %s: %s" % (case, path, e)) from None
            single.free()
            ctx.close()
        finally:
            for k in case.env:
                os.environ.pop(k, None)
    print("\nworld %d: %d cases, paths %s; ranks %.1f s, device memory in use at the peak %.2f GiB (all processes on the device)" % (
        world, len(S.CASES[world]), sorted(ran), t_spawn, peak / 2 ** 30))
