"""The float64 culling reference (cull_ref.py) against the oracle, on octrees that hold all four position encodings: the
reference's point test equals the oracle's for every point and every boundary location, every edge class the locations were
built for is reached and has its designed outcome, and the oracle's filtered query equals the reference applied to the points
of the nodes it visits.  The GPU tests (test_query_edges_gpu.py) hold the CUDA culls to the same reference."""
import collections

import numpy as np
import pytest

import cull_ref as R
import oracle_api as O

# (cloud, max_points_per_node): the four-encoding tree, and one whose nodes of every encoding span several cull tiles
TREES = {"deep": (False, 200), "wide": (True, 6000)}
RESOLUTION = 1e-7


def _copy_loc(loc, Loc):
    o = Loc()
    for f, _ in Loc._fields_:
        setattr(o, f, getattr(loc, f))
    return o


def oracle_scene(name):
    """The cloud, its oracle octree, the decoded points P of every node in visit order (the oracle's query of all points,
    pinned bit for bit against the product's), their intensities and provenance, and the boundary locations."""
    big, mppn = TREES[name]
    x, y, z, rgb, inten = R.edge_cloud(big)
    P0 = np.stack([x, y, z], 1)
    bmin, bmax = P0.min(0), P0.max(0)
    ref = O.build(x, y, z, rgb, RESOLUTION, bmin, bmax, intensity=inten, max_points_per_node=mppn)
    every = ref.query(O.Location(), with_intensity=True)  # kind 0: all points
    order = ref.nodes_in_location(O.Location())
    P = every["xyz"]
    from point_cloud_viewer_b200 import geometry as G

    locs = R.edge_locations(O.Location, ref.nodes, order, P, G)
    return dict(x=x, y=y, z=z, rgb=rgb, intensity=inten, bmin=bmin, bmax=bmax, mppn=mppn, ref=ref, order=order, P=P,
                src=every["src"], pint=every["intensity"], locs=locs)


@pytest.fixture(scope="module", params=sorted(TREES))
def scene(request):
    return oracle_scene(request.param)


def _node_slices(s):
    out, first = {}, 0
    for nm in s["order"]:
        cnt = s["ref"].nodes[nm]["num_points"]
        out[nm] = slice(first, first + cnt)
        first += cnt
    return out


def test_trees_cover_every_encoding(scene):
    nodes = scene["ref"].nodes
    enc = collections.Counter(m["enc"] for m in nodes.values() if m["num_points"])
    assert set(enc) == {1, 2, 3, 4}, enc
    if scene["mppn"] > 2048:  # every encoding has a node of two cull tiles or more, and nodes that end inside a 256-point round
        for e in (1, 2, 3, 4):
            sizes = [m["num_points"] for m in nodes.values() if m["enc"] == e]
            assert max(sizes) > 2048 and any(n % 256 for n in sizes), (e, max(sizes))
    vals = scene["pint"]
    for v in R.SPECIAL_INTENSITY:
        assert np.any(np.isnan(vals)) if np.isnan(v) else np.any((vals == v) & (np.signbit(vals) == np.signbit(v))), v


def test_contains_equals_oracle(scene):
    P = scene["P"]
    for name, loc, _ in scene["locs"]:
        assert np.array_equal(R.contains(loc, P), O.location_contains(loc, P)), name


def test_every_edge_class_is_reached_with_its_outcome(scene):
    """Every class has points in nodes the location visits, so the per-point culls of a query test them."""
    P = scene["P"]
    sl = _node_slices(scene)
    seen, reached = collections.Counter(), collections.Counter()
    for name, loc, labels in scene["locs"]:
        got = R.contains(loc, P)
        visited = np.zeros(len(P), bool)
        for nm in scene["ref"].nodes_in_location(loc):
            visited[sl[nm]] = True
        for cls, idx in labels.items():
            assert np.all(got[idx] == R.EXPECT[cls]), (name, cls, int(np.sum(got[idx] != R.EXPECT[cls])))
            seen[cls] += int(visited[idx].sum())
            reached[cls] += len(idx)
    reached = +reached
    assert set(reached) == set(R.EXPECT), set(R.EXPECT) - set(reached)
    # r == +-1 at w == 0 lies outside every node the frustum visits, so only the point test itself sees that class.  The strict
    # `min(c) > -1` it pins is reached on the GPU through the tiny- and huge-w edges instead: there r == -w divides to exactly -1.
    missing = [c for c in R.EXPECT if seen[c] == 0]
    assert missing == ["frustum_w0_edge"], (missing, dict(seen))
    assert seen["frustum_tiny_w_edge"] and seen["frustum_huge_w_edge"]


def test_filters_equal_oracle(scene):
    ref, pint = scene["ref"], scene["pint"]
    for f in R.FILTERS:
        keep = R.keep_filters(pint, f)
        want = ref.query(O.Location(), filters=f, with_intensity=True)
        assert np.array_equal(want["src"], scene["src"][keep]), f
    v = pint.astype(np.float64)
    # the edges FILTERS were written for
    assert not R.keep_filters(np.float32([0.1]), [(0.0, 0.1)])[0] and R.keep_filters(np.float32([-0.0]), [(0.0, 1.0)])[0]
    assert not R.keep_filters(np.float32([np.nan]), [(-np.inf, np.inf)])[0] and R.keep_filters(np.float32([-np.inf]), [(-np.inf, 0.0)])[0]
    assert R.keep_filters(np.float32([R.SUBNORMAL_F32]), [(R.SUBNORMAL_F32, 1.0)])[0] and not R.keep_filters(np.float32([0.0]), [(R.SUBNORMAL_F32, 1.0)])[0]
    assert np.sum(v == 0.25) and np.sum(v == 0.75)


def test_oracle_query_is_reference_over_visited_nodes(scene):
    ref, P = scene["ref"], scene["P"]
    sl = _node_slices(scene)
    for k, (name, loc, _) in enumerate(scene["locs"]):
        f = R.FILTERS[k % len(R.FILTERS)]
        visited = ref.nodes_in_location(loc)
        idx = np.concatenate([np.arange(sl[nm].start, sl[nm].stop) for nm in visited] or [np.zeros(0, np.int64)]).astype(np.int64)
        for filters in ((), f):
            want = ref.query(loc, filters=filters, with_intensity=True)
            keep = R.contains(loc, P[idx]) & R.keep_filters(scene["pint"][idx], filters)
            assert np.array_equal(want["src"], scene["src"][idx[keep]]), (name, filters)
            assert np.array_equal(want["xyz"], P[idx[keep]]), name
            assert want["tested"] == len(idx), name
