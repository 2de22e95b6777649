"""The CUDA culls at the edges of the point test, on octrees that hold all four position encodings (test_cull_ref.TREES).

Every boundary location of cull_ref (points exactly on Aabb faces and octree cube planes, Obb half extents equal to |q| or one ulp
less, frustum planes with r == +-w, the band T < |r| < |w|, w < 0, w == 0, tiny and huge w), with and without interval filters
on the special intensities (interval ends, -0.0, NaN, +-inf, an f32 subnormal, f32 0.1), goes through each kernel that culls:

  k_sat_nodes        nodes_in_location (resident and OctreeDir) equals the oracle's
  k_cull             Octree.query_points streams exactly the oracle's points; the survivors are the float64 reference's
  k_bfs_level +      query_batch_device: every count is the reference's, every `tested` the oracle's
    k_cull_fused<true>
  k_cull_chunk       OctreeDir.query_points equals the resident stream, at the smallest accepted budget and the default one
  k_cull_fused<false> OctreeDir.query_batch counts are the reference's
  k_lod_shuffle      shuffle_nodes equals the oracle's reshuffle for every encoding's bytes per coordinate
"""
import numpy as np
import pytest

import cull_ref as R
import oracle_api as O
from parity import compare_trees
from test_cull_ref import RESOLUTION, TREES, oracle_scene
from test_octree_dir_query_gpu import _smallest_budget

pytestmark = pytest.mark.gpu


class _IntensityBits:
    """A tree whose node_data returns the intensities as their f32 bit patterns (NaN == NaN, -0.0 != 0.0) for compare_trees."""

    def __init__(self, t, oracle):
        self.t, self.oracle = t, oracle
        self.nodes = t.nodes
        self.has_intensity = True

    def node_data(self, name, with_i=True):
        x, c, i, s = self.t.node_data(name, True) if self.oracle else self.t.node_data(name)
        return x, c, i.view(np.uint32), s


def _product_loc(pcv, loc):
    o = pcv._native.Location()
    for f, _ in O.Location._fields_:
        setattr(o, f, getattr(loc, f))
    return o


def _cat(batches):
    if not batches:
        return dict(xyz=np.zeros((0, 3)), rgb=np.zeros((0, 3), np.uint8), intensity=np.zeros(0, np.float32), src=np.zeros(0, np.uint64))
    return {k: np.concatenate([b[k] for b in batches]) for k in ("xyz", "rgb", "intensity", "src")}


def _build(s, ctx):
    return ctx.build_octree(s["x"], s["y"], s["z"], np.ascontiguousarray(s["rgb"]).reshape(-1), RESOLUTION, s["bmin"], s["bmax"], intensity=s["intensity"])


@pytest.fixture(scope="module", params=sorted(TREES))
def scene(request, tmp_path_factory):
    import point_cloud_viewer_b200 as pcv

    s = oracle_scene(request.param)
    ctx = pcv.Context(0, max_points_per_node=s["mppn"])
    tree = _build(s, ctx)
    compare_trees(_IntensityBits(s["ref"], True), _IntensityBits(tree, False))
    d = str(tmp_path_factory.mktemp("edges_" + request.param))
    tree.write_dir(d)
    # per location: the points of the nodes the oracle visits (positions into P, in visit order) and the reference's test of them
    pos = {}
    first = 0
    for nm in s["order"]:
        cnt = s["ref"].nodes[nm]["num_points"]
        pos[nm] = np.arange(first, first + cnt)
        first += cnt
    cases = []
    for k, (name, loc, labels) in enumerate(s["locs"]):
        visited = s["ref"].nodes_in_location(loc)
        idx = np.concatenate([pos[nm] for nm in visited] or [np.zeros(0, np.int64)]).astype(np.int64)
        cases.append(dict(name=name, loc=loc, ploc=_product_loc(pcv, loc), labels=labels, visited=visited, idx=idx,
                          inside=R.contains(loc, s["P"][idx]), filters=R.FILTERS[k % len(R.FILTERS)]))
    where = np.empty(len(s["P"]), np.int64)
    where[s["src"].astype(np.int64)] = np.arange(len(s["P"]))  # original point index -> position in P
    s.update(pcv=pcv, ctx=ctx, tree=tree, dir=d, cases=cases, where=where)
    yield s
    tree.free()
    ctx.close()


def _want(s, c, filters):
    """The reference's survivors of a case: positions into P, in visit order."""
    return c["idx"][c["inside"] & R.keep_filters(s["pint"][c["idx"]], filters)]


def test_nodes_in_location(scene):
    h = scene["ctx"].open_dir(scene["dir"])
    for c in scene["cases"]:
        assert scene["tree"].nodes_in_location(c["ploc"]) == c["visited"], c["name"]
        assert h.nodes_in_location(c["ploc"]) == c["visited"], c["name"]
    h.close()


def test_query_points_at_the_edges(scene):
    s = scene
    seen = set()
    for c in s["cases"]:
        for filters in ((), c["filters"]):
            got = _cat(s["tree"].query_points(c["ploc"], filters=filters, batch_size=4099))
            want = s["ref"].query(c["loc"], filters=filters, with_intensity=True)
            assert np.array_equal(got["src"], want["src"]), (c["name"], filters)
            assert np.array_equal(got["xyz"], want["xyz"]) and np.array_equal(got["rgb"], want["rgb"]), (c["name"], filters)
            assert np.array_equal(got["intensity"].view(np.uint32), want["intensity"].view(np.uint32)), (c["name"], filters)
            keep = _want(s, c, filters)
            assert np.array_equal(got["src"], s["src"][keep]), (c["name"], filters, len(got["src"]), len(keep))
            if not filters:  # every designed edge point has its designed outcome
                kept = np.zeros(len(s["P"]), bool)
                kept[s["where"][got["src"].astype(np.int64)]] = True
                visited = np.zeros(len(s["P"]), bool)
                visited[c["idx"]] = True
                for cls, idx in c["labels"].items():
                    idx = idx[visited[idx]]  # points of nodes the location does not visit are never tested
                    assert np.all(kept[idx] == R.EXPECT[cls]), (c["name"], cls)
                    if len(idx):
                        seen.add(cls)
    assert seen == set(R.EXPECT) - {"frustum_w0_edge"}, set(R.EXPECT) - seen  # see test_cull_ref


def test_query_batch_device_at_the_edges(scene):
    s = scene
    plocs = [c["ploc"] for c in s["cases"]]
    for filters in [()] + R.FILTERS:
        counts, tested = s["tree"].query_batch_device(plocs, filters=filters)
        st = s["tree"].last_query_stats()
        for i, c in enumerate(s["cases"]):
            assert counts[i] == len(_want(s, c, filters)), (c["name"], filters, int(counts[i]), len(_want(s, c, filters)))
            assert tested[i] == len(c["idx"]) == s["ref"].query(c["loc"])["tested"], (c["name"], filters)
        assert st["returned_points"] == int(counts.sum()) == st["stored_points"]
        assert st["tested_points"] == int(tested.sum())
    assert counts.sum() > 0


def test_octree_dir_at_the_edges(scene):
    s = scene
    pcv, ctx, tree = s["pcv"], s["ctx"], s["tree"]
    # slot of the directory handle -> original point index, through the node tables of both
    _, _, _, tsrc = tree.download()
    tmeta = {(int(m["id_high"]), int(m["id_low"])): int(m["point_offset"]) for m in tree.meta}
    small = _smallest_budget(ctx, s["dir"])[0]
    plocs = [c["ploc"] for c in s["cases"]]
    for budget in (small, 0):
        h = pcv.OctreeDir(ctx, s["dir"], budget)
        orig = np.zeros(h.num_points, np.uint64)
        for m in h.meta:
            n, dpo = int(m["num_points"]), int(m["point_offset"])
            tpo = tmeta[(int(m["id_high"]), int(m["id_low"]))]
            orig[dpo:dpo + n] = tsrc[tpo:tpo + n]
        # the smallest budget (one cull tile per chunk) streams every fourth case with one of the filters, in turn; the default
        # budget streams every case, with and without its filters
        runs = [(c, (R.FILTERS[j % len(R.FILTERS)],)) for j, c in enumerate(s["cases"][::4])] if budget == small else \
            [(c, ((), c["filters"])) for c in s["cases"]]
        split_seen = False
        for c, filter_sets in runs:
            for filters in filter_sets:
                got = _cat(h.query_points(c["ploc"], filters=filters, batch_size=1 << 20))
                st = h.last_stats()
                want = _cat(tree.query_points(c["ploc"], filters=filters, batch_size=1 << 20))
                assert np.array_equal(orig[got["src"].astype(np.int64)], want["src"]), (budget, c["name"], filters)
                assert np.array_equal(want["src"], s["src"][_want(s, c, filters)]), (budget, c["name"], filters)  # the reference's
                assert np.array_equal(got["xyz"], want["xyz"]) and np.array_equal(got["rgb"], want["rgb"]), (budget, c["name"])
                assert np.array_equal(got["intensity"].view(np.uint32), want["intensity"].view(np.uint32)), (budget, c["name"])
                if budget == small:  # a node of more than 2048 points spans several chunks
                    split = sum(1 for nm in c["visited"] if s["ref"].nodes[nm]["num_points"] > 2048)
                    assert st["max_device_bytes"] == small and (split == 0 or st["chunks"] > split), (c["name"], split, st["chunks"])
                    split_seen |= split > 0
        assert split_seen or budget != small
        # A batch needs room for its selection frontier (24 bytes per (location, node) pair of a level) besides what the handle
        # holds, and the smallest budget has none: the product refuses it ("split the batch").  So at that leg the batches hold 8
        # locations and the budget adds room for the largest frontier 8 locations can have; the culls of the visited
        # nodes then still run in many chunks.
        nb = 8 if budget == small else len(plocs)
        hb = pcv.OctreeDir(ctx, s["dir"], small + nb * (4096 + 24 * h.num_nodes) + (64 << 10)) if budget == small else h
        # k_cull_fused<false>'s interval filter: every filter edge at the default budget, f32 0.1 in many chunks
        for filters in [()] + (R.FILTERS if budget != small else [R.FILTERS[3]]):
            parts, chunks = [], 0
            for i in range(0, len(plocs), nb):
                parts.append(hb.query_batch(plocs[i:i + nb], filters=filters))
                chunks = max(chunks, hb.last_stats()["chunks"])
            counts, tested = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
            assert chunks > 1 or budget != small, chunks
            for i, c in enumerate(s["cases"]):
                assert counts[i] == len(_want(s, c, filters)) and tested[i] == len(c["idx"]), (budget, c["name"], filters)
        if hb is not h:
            hb.close()
        h.close()


def test_shuffle_nodes_every_encoding(scene):
    """k_lod_shuffle moves 1, 2, 4 and 8 bytes per coordinate; a boundary query afterwards keeps the same survivors."""
    s = scene
    pcv = s["pcv"]
    tree = _build(s, s["ctx"])
    before = {nm: tree.node_data(nm) for nm, m in tree.nodes.items() if m["num_points"]}
    seed = 77031
    tree.shuffle_nodes(seed)
    encs = set()
    for nm, m in tree.nodes.items():
        cnt = m["num_points"]
        if not cnt:
            continue
        order = pcv.lod_order(seed, nm, cnt)
        bx, bc, bi, bs = before[nm]
        gx, gc, gi, gs = tree.node_data(nm)
        assert np.array_equal(gx, O.reshuffle(order, bx, 3 * pcv.ENC_BYTES[m["enc"]])), (nm, m["enc"])
        assert np.array_equal(gc.reshape(-1), O.reshuffle(order, bc, 3)), nm
        o = order.astype(np.int64)
        assert np.array_equal(gs, bs[o]) and np.array_equal(gi.view(np.uint32), bi.view(np.uint32)[o]), nm
        encs.add(m["enc"])
    assert encs == {1, 2, 3, 4}
    for c in s["cases"][:: max(1, len(s["cases"]) // 24)]:
        got = np.sort(_cat(tree.query_points(c["ploc"], filters=c["filters"]))["src"])
        assert np.array_equal(got, np.sort(s["src"][_want(s, c, c["filters"])])), c["name"]
    tree.free()
