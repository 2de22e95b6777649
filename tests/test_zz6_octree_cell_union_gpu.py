"""Octree point queries by S2 cell union (pcv_*cell_union*): the points returned equal every point of the octree whose leaf cell
the union contains (the oracle's from_point and CellUnion::contains), in the order the AllPoints stream delivers them; the node
list holds every node with such a point, in BFS order, and equals the CPU restatement of the node test (csrc/s2.h
s2_cube_relation + BFS over the node table).  The same over an octree directory read in several chunks."""
import ctypes as C

import numpy as np
import pytest

import s2_api as S
from test_octree_dir_query_gpu import _cat, _smallest_budget
from test_s2_cube_relation import IN, OUT, face_ij_level, parent, relation

pytestmark = pytest.mark.gpu

CENTRE = np.array([4157222.543, 664789.307, 4774952.099])  # the slab's origin (ecef_from_local.translation, csrc/synth.cuh)


def _tree_info(pcv, tree):
    """AllPoints stream (batches concatenated), the BFS node table and each stream position's node."""
    G = pcv.geometry
    allp = _cat(tree.query_points(G.all_points(), batch_size=1 << 30))
    order = tree.nodes_in_location(G.all_points())  # every node, in BFS (table) order
    counts = np.array([tree.nodes[nm]["num_points"] for nm in order], np.int64)
    node_of = np.repeat(np.arange(len(order)), counts)
    leaves = S.oracle_cell_ids(allp["xyz"], 30)
    return dict(all=allp, order=order, counts=counts, node_of=node_of, leaves=leaves)


@pytest.fixture(scope="module")
def slab(tmp_path_factory):
    """The reference's 1e6-point config-1 slab (point_cloud_test/tests/main.rs), with an intensity channel, and its directory."""
    import point_cloud_viewer_b200 as pcv

    n = 1_000_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    inten = (np.arange(n) % 997).astype(np.float32)
    c = pcv.Context(0)
    tree = c.build_octree(x, y, z, rgb, res, bmin, bmax, intensity=inten)
    d = str(tmp_path_factory.mktemp("slab_cu"))
    tree.write_dir(d)
    info = _tree_info(pcv, tree)
    yield dict(pcv=pcv, ctx=c, tree=tree, dir=d, **info)
    tree.free()
    c.close()


def _want(s, cu):
    """The oracle's predicate over the AllPoints stream: the mask of the points whose leaf cell the normalised union contains."""
    cu = S.normalize(np.asarray(cu, np.uint64))
    return S.union_test(cu, s["leaves"])[0] if len(cu) else np.zeros(len(s["leaves"]), bool)


def _assert_stream_equal(got, allp, mask):
    assert len(got["src"]) == int(mask.sum())
    assert np.array_equal(got["xyz"].view(np.uint64), allp["xyz"][mask].view(np.uint64))  # bit-equal positions
    assert np.array_equal(got["rgb"], allp["rgb"][mask])
    assert np.array_equal(got["src"], allp["src"][mask])  # and the AllPoints order
    if allp["intensity"] is not None:
        assert np.array_equal(got["intensity"], allp["intensity"][mask])


def _stream(s, cu, bs=1 << 30, filters=()):
    return s["tree"].query_points(s["pcv"].geometry.cell_union(cu), filters=filters, batch_size=bs)


def _reference_union():
    cell = int(S.oracle_cell_ids(CENTRE[None, :], 20)[0])
    return np.array([cell, S.orc().orc_s2_next(cell)], np.uint64)  # queries.rs:49-53


def _cpu_nodes(s, tree_nodes, cu):
    """The node list restated on the CPU: s2_cube_relation of every node cube, a node listed iff it and all its ancestors are not Out."""
    cu = S.normalize(np.asarray(cu, np.uint64))
    order = s["order"]
    m = np.array([tree_nodes[nm]["cube"][:3] for nm in order], np.float64)
    e = np.array([tree_nodes[nm]["cube"][3] for nm in order], np.float64)
    rel = relation(cu, m, e)
    ok = {}
    out = []
    for nm, r in zip(order, rel):
        p = ok.get(nm[:-1], True) if len(nm) > 1 else True
        ok[nm] = p and r != OUT
        if ok[nm]:
            out.append(nm)
    return out, dict(zip(order, rel))


def test_reference_union_streams(slab):
    s = slab
    cu = _reference_union()
    mask = _want(s, cu)
    assert 0 < mask.sum() < len(mask)
    for bs in (5000, 500000):
        batches = _stream(s, cu, bs)
        assert all(len(b["src"]) == bs for b in batches[:-1]) and 0 < len(batches[-1]["src"]) <= bs
        _assert_stream_equal(_cat(batches), s["all"], mask)
    with pytest.raises(s["pcv"].PcvError) as ei:
        s["tree"].query_points(s["pcv"].geometry.cell_union(cu), callback=lambda b: True, batch_size=5000)
    assert ei.value.code == -5  # PCV_ERR_CANCELLED


def test_more_unions(slab):
    s = slab
    rng = np.random.default_rng(7)
    leaves = s["leaves"]
    pick = rng.choice(len(leaves), 64, replace=False)
    cu = leaves[pick]
    got = _cat(_stream(s, cu))
    _assert_stream_equal(got, s["all"], _want(s, cu))
    assert set(s["all"]["src"][pick].tolist()) <= set(got["src"].tolist())  # every sampled point comes back
    mixed = np.array([parent(int(leaves[k]), int(rng.integers(12, 19))) for k in rng.choice(len(leaves), 40)], np.uint64)
    _assert_stream_equal(_cat(_stream(s, mixed, 100000)), s["all"], _want(s, mixed))
    f, _, _ = S.face_ij(int(leaves[0]))
    face = np.array([(f << 61) | (1 << 60)], np.uint64)
    got = _cat(_stream(s, face))
    _assert_stream_equal(got, s["all"], np.ones(len(leaves), bool))  # the whole face: AllPoints
    assert _stream(s, np.zeros(0, np.uint64)) == []
    assert s["tree"].nodes_in_location(s["pcv"].geometry.cell_union([])) == []
    # un-normalised: duplicates, nested cells and a cell with all four children; the same points as the normalised form
    raw = np.concatenate([mixed, mixed[:5], [parent(int(mixed[0]), 10)], [parent(int(leaves[1]), 20)], [parent(int(leaves[1]), 24)]]).astype(np.uint64)
    f14, i14, j14, _ = face_ij_level(parent(int(leaves[2]), 14))
    kids = [parent(int(S.orc().orc_s2_from_face_ij(f14, i14 + di, j14 + dj)), 15) for di in (0, 1 << 15) for dj in (0, 1 << 15)]
    raw = np.concatenate([raw, np.array(kids, np.uint64)])
    norm = S.normalize(raw)
    a, b = _cat(_stream(s, raw)), _cat(_stream(s, norm))
    _assert_stream_equal(a, s["all"], _want(s, norm))
    assert np.array_equal(a["src"], b["src"])
    # intensity filter intervals
    flt = [(100.0, 400.0), (150.0, 900.0)]
    inten = s["all"]["intensity"].astype(np.float64)
    m = _want(s, mixed) & (inten >= 150.0) & (inten <= 400.0)
    _assert_stream_equal(_cat(_stream(s, mixed, 7777, flt)), s["all"], m)


def test_face_corner_and_origin_clouds():
    import point_cloud_viewer_b200 as pcv

    rng = np.random.default_rng(3)
    c = pcv.Context(0, max_points_per_node=2000)
    corner = np.ones(3) / np.sqrt(3.0) * 6371000.0  # the (1, 1, 1) corner of faces 0, 1 and 2
    P = corner + rng.uniform(-40.0, 40.0, (200_000, 3))
    cloud = dict(x=P[:, 0].copy(), y=P[:, 1].copy(), z=P[:, 2].copy())
    bmin, bmax = P.min(0), P.max(0)
    rgb = rng.integers(0, 256, (len(P), 3), dtype=np.uint8).reshape(-1)
    trees = [c.build_octree(cloud["x"], cloud["y"], cloud["z"], rgb, 0.001, bmin, bmax)]
    Q = rng.normal(0.0, 30.0, (200_000, 3))  # a cloud around the origin: every face, and nodes that touch the origin
    Q[:8] = 0.0
    t2 = c.build_octree(Q[:, 0].copy(), Q[:, 1].copy(), Q[:, 2].copy(), rgb, 0.001, Q.min(0), Q.max(0))
    root = t2.nodes["r"]["cube"]
    assert all(root[k] <= 0.0 <= root[k] + root[3] for k in range(3))  # the root cube holds the origin
    trees.append(t2)
    for t in trees:
        s = dict(pcv=pcv, tree=t, **_tree_info(pcv, t))
        leaves = s["leaves"]
        for cu in (leaves[rng.choice(len(leaves), 32, replace=False)],
                   np.array([parent(int(leaves[k]), int(rng.integers(3, 16))) for k in rng.choice(len(leaves), 12)], np.uint64)):
            _assert_stream_equal(_cat(_stream(s, cu, 50000)), s["all"], _want(s, cu))
            names = t.nodes_in_location(pcv.geometry.cell_union(cu))
            assert names == _cpu_nodes(s, t.nodes, cu)[0]
        t.free()
    c.close()


def test_node_lists(slab):
    s = slab
    G = s["pcv"].geometry
    rng = np.random.default_rng(11)
    leaves = s["leaves"]
    unions = [_reference_union(), leaves[rng.choice(len(leaves), 16)],
              np.array([parent(int(leaves[k]), int(rng.integers(12, 19))) for k in rng.choice(len(leaves), 8)], np.uint64)]
    pos = {nm: i for i, nm in enumerate(s["order"])}
    starts = np.concatenate([[0], np.cumsum(s["counts"])])
    for cu in unions:
        names = s["tree"].nodes_in_location(G.cell_union(cu))
        mask = _want(s, cu)
        holding = {s["order"][k] for k in np.unique(s["node_of"][mask])}
        assert holding <= set(names)  # every node with a passing point
        idx = [pos[nm] for nm in names]
        assert idx == sorted(idx)  # a subsequence of the AllPoints (BFS) list
        want, rel = _cpu_nodes(s, s["tree"].nodes, cu)
        assert names == want
        for nm in names:  # a node classified In is returned whole
            if rel[nm] == IN:
                k = pos[nm]
                assert mask[starts[k]:starts[k + 1]].all()
    assert len(s["tree"].nodes_in_location(G.cell_union(_reference_union()))) < len(s["order"])
    assert any(r == IN for r in _cpu_nodes(s, s["tree"].nodes, unions[2])[1].values())


def _union_counts(leaves_sorted, cu):
    """Points per normalised union from sorted leaf ids: the cells are disjoint ranges of leaf ids."""
    cu = S.normalize(np.asarray(cu, np.uint64)).astype(np.uint64)
    if len(cu) == 0:
        return 0
    lsb = cu & (~cu + np.uint64(1))
    lo, hi = cu - (lsb - np.uint64(1)), cu + (lsb - np.uint64(1))
    return int((np.searchsorted(leaves_sorted, hi, side="right") - np.searchsorted(leaves_sorted, lo, side="left")).sum())


def _batch_unions(s, k=1200):
    rng = np.random.default_rng(21)
    leaves = s["leaves"]
    out = []
    for i in range(k):
        m = int(rng.integers(0, 6))
        out.append(np.array([parent(int(leaves[j]), int(rng.integers(10, 31))) if rng.random() < 0.9 else int(leaves[j])
                             for j in rng.choice(len(leaves), m)], np.uint64))
    out[0] = _reference_union()
    return out


def test_batch(slab):
    s = slab
    G = s["pcv"].geometry
    unions = _batch_unions(s)
    counts, tested = s["tree"].query_batch_device([G.cell_union(u) for u in unions])
    st = s["tree"].last_query_stats()
    ls = np.sort(s["leaves"])
    assert [int(v) for v in counts] == [_union_counts(ls, u) for u in unions]
    assert st["returned_points"] == int(counts.sum()) and st["tested_points"] == int(tested.sum())
    for i in range(0, len(unions), 60):  # streaming totals and the points of the selected nodes
        names = s["tree"].nodes_in_location(G.cell_union(unions[i]))
        assert int(tested[i]) == sum(s["tree"].nodes[nm]["num_points"] for nm in names)
        assert int(counts[i]) == len(_cat(_stream(s, unions[i]))["src"])
    with pytest.raises(ValueError):
        s["tree"].query_batch_device([G.cell_union(unions[0]), G.all_points()])


def test_directory(slab):
    s = slab
    pcv, G = s["pcv"], s["pcv"].geometry
    _, _, _, src_all = s["tree"].download()
    lo, _ = _smallest_budget(s["ctx"], s["dir"])
    h = pcv.OctreeDir(s["ctx"], s["dir"], lo + (6 << 20))
    # a directory slot (point_offset + j in the directory's node table) -> the resident octree's slot of the same point
    dm = h.nodes()
    order = np.argsort(dm["point_offset"], kind="stable")
    d_off = dm["point_offset"][order].astype(np.int64)
    r_off = np.array([s["tree"].nodes[pcv.node_name(m["id_high"], m["id_low"])]["point_offset"] for m in dm[order]], np.int64)

    def res_slot(slots):
        slots = slots.astype(np.int64)
        k = np.searchsorted(d_off, slots, side="right") - 1
        return r_off[k] + (slots - d_off[k])

    unions =[_reference_union(), _batch_unions(s, 40)[7], np.array([(int(S.face_ij(int(s["leaves"][0]))[0]) << 61) | (1 << 60)], np.uint64)]
    for cu in unions:
        got = _cat(h.query_points(G.cell_union(cu), filters=[(0.0, 900.0)], batch_size=30000))
        chunks = h.last_stats()["chunks"]
        want = _cat(_stream(s, cu, 30000, [(0.0, 900.0)]))
        assert np.array_equal(src_all[res_slot(got["src"])], want["src"])
        assert np.array_equal(got["xyz"].view(np.uint64), want["xyz"].view(np.uint64)) and np.array_equal(got["rgb"], want["rgb"])
        assert got["sizes"] == want["sizes"]
        assert h.nodes_in_location(G.cell_union(cu)) == s["tree"].nodes_in_location(G.cell_union(cu))
    assert chunks > 1  # the whole face (the last union) did not fit one chunk
    h.close()
    h = pcv.OctreeDir(s["ctx"], s["dir"], lo + (64 << 20))
    bu = _batch_unions(s, 1000)
    c1, t1 = h.query_batch([G.cell_union(u) for u in bu])
    c2, t2 = s["tree"].query_batch_device([G.cell_union(u) for u in bu])
    assert np.array_equal(c1, c2) and np.array_equal(t1, t2)
    h.close()


def test_errors(slab):
    s = slab
    pcv, G = s["pcv"], s["pcv"].geometry
    N = pcv._native
    for bad in ([0], [7 << 61 | 1], [int(_reference_union()[0]) + 2]):
        with pytest.raises(pcv.PcvError) as ei:
            s["tree"].query_points(G.cell_union(bad))
        assert ei.value.code == -1
        with pytest.raises(pcv.PcvError) as ei:
            s["tree"].nodes_in_location(G.cell_union(bad))
        assert ei.value.code == -1
    cu = N.CellUnion(None, 3, 0)
    n = C.c_uint64()
    out = np.zeros(2 * (len(s["order"]) + 1), np.uint64)
    assert N.lib().pcv_nodes_in_cell_union(s["tree"].h, C.byref(cu), out.ctypes.data, len(s["order"]) + 1, C.byref(n)) == -1
    assert N.lib().pcv_query_cell_unions_batch_device(s["tree"].h, C.byref(cu), 1, None, 0, None, None) == -1
    # filters over an octree without intensity: the existing error
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 5, 0, 20_000)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    t = s["ctx"].build_octree(x, y, z, rgb, res, bmin, bmax)
    with pytest.raises(pcv.PcvError) as ei:
        t.query_points(G.cell_union(_reference_union()), filters=[(0.0, 1.0)])
    assert ei.value.code == -1 and "Filter attribute" in str(ei.value)
    t.free()
