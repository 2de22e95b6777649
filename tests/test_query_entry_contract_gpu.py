"""The argument contract the point queries of all three sources share - the resident octree, the octree directory and the S2
cloud, each through its nodes / cells, stream and batch entry points: an unknown location kind and a null filter array are
PCV_ERR_INVALID, so are filters over points without intensity; a consumer callback that stops the stream gives
PCV_ERR_CANCELLED after exactly the batches it saw; every streamed batch holds batch_size points except the last."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SOURCES = ("octree", "dir", "s2")
N_POINTS = 60_000


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    """The seeded ECEF slab with intensity as each source, and the octree, directory and S2 cloud of it without intensity."""
    import point_cloud_viewer_b200 as pcv

    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, N_POINTS)
    inten = (np.arange(N_POINTS) % 1000).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    ctx = pcv.Context(0, max_points_per_node=2000)
    with_i, without_i = {}, {}
    for intensity, out in ((inten, with_i), (None, without_i)):
        tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=intensity)
        d = str(tmp_path_factory.mktemp("contract"))
        tree.write_dir(d)
        out.update(octree=tree, dir=ctx.open_dir(d), s2=ctx.build_s2_cloud(x, y, z, rgb, intensity))
    yield dict(pcv=pcv, with_i=with_i, without_i=without_i, bmin=np.asarray(bmin), bmax=np.asarray(bmax))
    for h in list(with_i.values()) + list(without_i.values()):
        h.close() if isinstance(h, pcv.OctreeDir) else h.free()
    ctx.close()


def _fns(source):
    """(nodes or cells in location, stream, stream of a cell union, batch, batch of cell unions) of one source's C ABI."""
    from point_cloud_viewer_b200 import _native as N

    L = N.lib()
    return {
        "octree": (L.pcv_nodes_in_location, L.pcv_query_points, L.pcv_query_cell_union, L.pcv_query_batch_device, L.pcv_query_cell_unions_batch_device),
        "dir": (L.pcv_octree_dir_nodes_in_location, L.pcv_octree_dir_query_points, L.pcv_octree_dir_query_cell_union, L.pcv_octree_dir_query_batch,
                L.pcv_octree_dir_query_cell_unions_batch),
        "s2": (L.pcv_s2_cells_in_location, L.pcv_s2_query_points, L.pcv_s2_query_cell_union, L.pcv_s2_query_batch_device,
               L.pcv_s2_query_cell_unions_batch_device),
    }[source]


def _calls(h, source, loc, filters, nfilt):
    """The return codes of the nodes, stream and batch calls over one location; the callback accepts every batch."""
    from point_cloud_viewer_b200 import _native as N

    nodes, stream, _, batch, _ = _fns(source)
    h = h.h
    cap = 1 << 16
    ids, n = np.zeros(2 * cap, np.uint64), C.c_uint64()
    counts, tested = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    cb = N.BATCH_CB(lambda _u, _b: 0)
    return (nodes(h, C.byref(loc), ids.ctypes.data, cap, C.byref(n)),
            stream(h, C.byref(loc), filters, nfilt, 4096, cb, None),
            batch(h, (N.Location * 1)(loc), 1, filters, nfilt, counts.ctypes.data, tested.ctypes.data))


@pytest.mark.parametrize("source", SOURCES)
def test_unknown_location_kind_is_invalid(scene, source):
    G = scene["pcv"].geometry
    h = scene["with_i"][source]
    assert _calls(h, source, G.all_points(), None, 0) == (0, 0, 0)
    bad = G.all_points()
    bad.kind = 7
    assert _calls(h, source, bad, None, 0) == (-1, -1, -1)


@pytest.mark.parametrize("source", SOURCES)
def test_null_filters_are_invalid(scene, source):
    from point_cloud_viewer_b200 import _native as N

    G = scene["pcv"].geometry
    h = scene["with_i"][source].h
    _, stream, stream_cu, batch, batch_cu = _fns(source)
    loc, cu = G.all_points(), N.CellUnion(None, 0, 0)
    cb = N.BATCH_CB(lambda _u, _b: 0)
    counts, tested = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    f = (N.Interval * 1)(N.Interval(0.0, 500.0))
    for filters, want in ((f, 0), (None, -1)):
        assert stream(h, C.byref(loc), filters, 1, 4096, cb, None) == want
        assert stream_cu(h, C.byref(cu), filters, 1, 4096, cb, None) == want
        assert batch(h, (N.Location * 1)(loc), 1, filters, 1, counts.ctypes.data, tested.ctypes.data) == want
        assert batch_cu(h, (N.CellUnion * 1)(cu), 1, filters, 1, counts.ctypes.data, tested.ctypes.data) == want


@pytest.mark.parametrize("source", SOURCES)
def test_filters_need_intensity(scene, source):
    pcv = scene["pcv"]
    G = pcv.geometry
    h = scene["without_i"][source]
    assert len(h.query_points(G.all_points(), batch_size=1 << 20)) == 1
    for call in (lambda: h.query_points(G.all_points(), filters=[(0.0, 500.0)]),
                 lambda: (h.query_batch if source == "dir" else h.query_batch_device)([G.all_points()], filters=[(0.0, 500.0)])):
        with pytest.raises(pcv.PcvError) as e:
            call()
        assert e.value.code == -1 and "Filter attribute needs to be specified as query attribute." in str(e.value)


def _same_batch(a, b):
    return all((a[k] is None and b[k] is None) or np.array_equal(a[k], b[k]) for k in ("xyz", "rgb", "intensity", "src"))


@pytest.mark.parametrize("source", SOURCES)
def test_cancel_delivers_a_prefix(scene, source):
    pcv = scene["pcv"]
    h = scene["with_i"][source]
    box = pcv.geometry.aabb(scene["bmin"], scene["bmin"] + 0.8 * (scene["bmax"] - scene["bmin"]))
    full = h.query_points(box, filters=[(0.0, 700.0)], batch_size=1001)
    assert len(full) > 4
    for k in (1, 3):
        got = []

        def stop_after_k(b):
            got.append(b)
            return len(got) == k

        with pytest.raises(pcv.PcvError) as e:
            h.query_points(box, callback=stop_after_k, filters=[(0.0, 700.0)], batch_size=1001)
        assert e.value.code == -5
        assert len(got) == k and all(_same_batch(a, b) for a, b in zip(got, full[:k]))


@pytest.mark.parametrize("source", SOURCES)
def test_batches_hold_batch_size_points(scene, source):
    pcv = scene["pcv"]
    h = scene["with_i"][source]
    everything = np.concatenate([b["src"] for b in h.query_points(pcv.geometry.all_points(), batch_size=1 << 30)])
    assert len(everything) == N_POINTS
    for bs in (1000, 2048, 4097, N_POINTS, N_POINTS + 1):
        sizes = [len(b["src"]) for b in h.query_points(pcv.geometry.all_points(), batch_size=bs)]
        assert all(s == bs for s in sizes[:-1]) and 0 < sizes[-1] <= bs, (bs, sizes)
        assert sum(sizes) == N_POINTS
