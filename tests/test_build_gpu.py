"""GPU parity of build_octree: CUDA path (through the C ABI) vs the oracle, bit-exact."""
import numpy as np
import pytest

import oracle_api as O
from parity import compare_trees, decode_node

pytestmark = pytest.mark.gpu


def _clustered(rng, n, nclusters=20, offset=(4.1e6, 6.6e5, 4.7e6)):
    cen = rng.random((nclusters, 3)) * [200, 200, 20]
    k = rng.integers(0, nclusters, n)
    P = cen[k] + rng.normal(0, 1, (n, 3)) * rng.random((nclusters, 1))[k] * 3
    P[: n // 10] = P[0]
    P += offset
    return P


def test_reference_scenario_100001(ctx):
    """src/octree/tests.rs:18-46: 100 000 points at the origin + 1 outlier, resolution 1.0."""
    n = 100001
    x, y, z = np.zeros(n), np.zeros(n), np.zeros(n)
    x[-1], y[-1], z[-1] = -200.0, -40.0, 30.0
    rgb = np.tile(np.array([255, 0, 0], np.uint8), n)
    tree = ctx.build_octree(x, y, z, rgb, 1.0, (0, 0, 0), (-200, -40, 30))
    assert {k: v["num_points"] for k, v in tree.nodes.items()} == {"r": 12501, "r0": 0, "r4": 87500}
    ref = O.build(x, y, z, rgb.reshape(-1, 3), 1.0, (-200, -40, 0), (0, 0, 30))
    compare_trees(ref, tree)
    tree.free()


@pytest.mark.parametrize("n,maxpts,G,res", [(200000, 500, 3, 0.001), (200000, 500, 2, 0.001), (150000, 500, 1, 0.001),
                                             (50000, 50, 3, 1e-6), (300000, 1000, 3, 1e-9), (1000, 100000, 3, 0.001), (1, 100000, 3, 0.001)])
def test_small_deep_trees(n, maxpts, G, res):
    """G only seeds the cloud: levels_per_pass no longer changes the build (every pass resolves two levels, one when a single
    level is left), so the G parametrisations are different clouds, not different pass schedules."""
    import point_cloud_viewer_b200 as pcv

    rng = np.random.default_rng(n + G)
    P = _clustered(rng, n)
    x, y, z = [np.ascontiguousarray(P[:, i]) for i in range(3)]
    rgb = rng.integers(0, 255, n * 3, dtype=np.uint8)
    inten = rng.random(n).astype(np.float32)
    c = pcv.Context(0, max_points_per_node=maxpts, levels_per_pass=G)
    tree = c.build_octree(x, y, z, rgb, res, P.min(0), P.max(0), intensity=inten)
    ref = O.build(x, y, z, rgb.reshape(-1, 3), res, P.min(0), P.max(0), intensity=inten, max_points_per_node=maxpts)
    compare_trees(ref, tree)
    assert sum(v["num_points"] for v in tree.nodes.values()) == n
    tree.free()
    c.close()


def test_aos_input_and_empty(ctx):
    rng = np.random.default_rng(3)
    P = np.ascontiguousarray(_clustered(rng, 30000))
    rgb = rng.integers(0, 255, 30000 * 3, dtype=np.uint8)
    flat = P.reshape(-1)
    t1 = ctx.build_octree(flat[0:], flat[1:], flat[2:], rgb, 0.001, P.min(0), P.max(0), stride=3, n=30000)
    x, y, z = [np.ascontiguousarray(P[:, i]) for i in range(3)]
    ref = O.build(x, y, z, rgb.reshape(-1, 3), 0.001, P.min(0), P.max(0))
    compare_trees(ref, t1)
    t1.free()
    e = ctx.build_octree(np.zeros(0), np.zeros(0), np.zeros(0), np.zeros(0, np.uint8), 0.001, (0, 0, 0), (1, 1, 1), n=0)
    assert len(e.nodes) == 0
    e.free()


def test_bbox(ctx):
    rng = np.random.default_rng(9)
    P = _clustered(rng, 1234567)
    x, y, z = [np.ascontiguousarray(P[:, i]) for i in range(3)]
    mn, mx = ctx.bbox(x, y, z)
    assert np.array_equal(mn, P.min(0)) and np.array_equal(mx, P.max(0))
    assert O.bbox(x, y, z) == tuple(mn) + tuple(mx)


def test_config1_slab_1e6(ctx):
    """BASELINE config 1 shape (point_cloud_test defaults): sum(num_points) == N (tests/main.rs:10-23) and decoded
    positions within 2*sqrt(3)*resolution of the originals (tests/main.rs:167)."""
    import point_cloud_viewer_b200 as pcv

    n = 1_000_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    tree = ctx.build_octree(x, y, z, rgb, res, bmin, bmax)
    assert sum(v["num_points"] for v in tree.nodes.values()) == n
    ref = O.build(x, y, z, rgb.reshape(-1, 3), res, bmin, bmax)
    compare_trees(ref, tree)
    # The reference's threshold (2*sqrt(3)*resolution) holds for its own slab pose, where no point passes through
    # more than two fix-point stages.  Every re-quantisation truncates (codec.rs:110-112), so a point that is stored
    # in a Uint16 node after k fix-point writes can sit up to k code steps low per axis; with this pose some nodes
    # reach k = 4.  Pin the reference's bound for >= 99 % of the points and twice that for all of them.
    P = np.stack([x, y, z], 1)
    dist = []
    for name, m in tree.nodes.items():
        if m["num_points"] == 0:
            continue
        xyzb, _, _, src = tree.node_data(name)
        dist.append(np.linalg.norm(decode_node(m, xyzb.tobytes()) - P[src.astype(np.int64)], axis=1))
    dist = np.concatenate(dist)
    thr = 2 * np.sqrt(3) * res
    assert len(dist) == n and (dist <= thr).mean() >= 0.99 and dist.max() <= 2 * thr, ((dist <= thr).mean(), dist.max())
    tree.free()


def test_synth_host_device_identical(ctx):
    import torch

    import point_cloud_viewer_b200 as pcv

    n = 100000
    for kind in (pcv.SYNTH_SLAB_ECEF, pcv.SYNTH_GAUSS_CLUSTERS):
        hx, hy, hz, hrgb = pcv.synth_points_host(kind, 7, (1 << 20) - 50000, n)
        dx, dy, dz = [torch.empty(n, dtype=torch.float64, device="cuda") for _ in range(3)]
        drgb = torch.empty(n * 3, dtype=torch.uint8, device="cuda")
        ctx.synth_points_device(kind, 7, (1 << 20) - 50000, n, dx.data_ptr(), dy.data_ptr(), dz.data_ptr(), drgb.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(dx.cpu().numpy(), hx) and np.array_equal(dy.cpu().numpy(), hy) and np.array_equal(dz.cpu().numpy(), hz)
        assert np.array_equal(drgb.cpu().numpy(), hrgb)


def test_degenerate_numerators_take_the_ieee_path(ctx):
    """Zero, negative-zero, tiny (< 2^-500), subnormal and boundary coordinates in two boxes at the origin.  The unit box has
    power-of-two edges (division mode 3): every quotient is an exact scaling and nothing is flagged.  The 0.75 box touches zero
    with edges that are not powers of two (mode 1): the reciprocal division flags these numerators and the block repeats its
    tile with the IEEE operator.  Both stay bit-identical to the oracle."""
    import point_cloud_viewer_b200 as pcv
    from tb_api import level_table

    rng = np.random.default_rng(17)
    n = 60000
    for hi, mode in ((1.0, 3), (0.75, 1)):
        P = rng.random((n, 3)) * hi
        P[:5000] = 0.0
        P[5000:6000, 0] = -0.0
        P[6000:7000, 1] = 1e-200
        P[7000:8000, 2] = 5e-324
        P[8000:9000] = hi  # on the max corner
        P[9000:10000] = hi / 2  # exactly on the centre planes (strict > decides)
        x, y, z = [np.ascontiguousarray(P[:, i]) for i in range(3)]
        rgb = rng.integers(0, 255, n * 3, dtype=np.uint8)
        for maxpts, res in ((300, 1e-4), (2000, 1e-9)):
            assert level_table(hi, res, (0.0, 0.0, 0.0))["fast"] == mode
            c = pcv.Context(0, max_points_per_node=maxpts)
            tree = c.build_octree(x, y, z, rgb, res, (0, 0, 0), (hi, hi, hi))
            ref = O.build(x, y, z, rgb.reshape(-1, 3), res, (0, 0, 0), (hi, hi, hi), max_points_per_node=maxpts)
            compare_trees(ref, tree)
            tree.free()
            c.close()


def test_wild_inputs_with_unchecked_fast_path(ctx):
    """Root cube far from zero -> the kernels skip the per-numerator range checks (LevelTable::fast == 2) and only look at
    the raw inputs once: huge, infinite and NaN coordinates (outside the bounding box) must send their tiles through the
    IEEE operator and still match the oracle bit for bit."""
    import point_cloud_viewer_b200 as pcv

    rng = np.random.default_rng(23)
    n = 80000
    P = rng.random((n, 3)) * 100.0 + [4.1e6, 6.6e5, 4.7e6]
    bmin, bmax = P.min(0).copy(), P.max(0).copy()
    P[100] = [1e200, 6.6e5, 4.7e6]
    P[5000, 1] = -1e300
    P[9000, 2] = np.inf
    P[12000, 0] = -np.inf
    P[20000] = [np.nan, 6.6e5 + 1, 4.7e6 + 1]
    P[20001, 2] = 2.0 ** 399  # just inside the admissible input range
    P[30000] = 0.0  # far outside the box, towards zero
    x, y, z = [np.ascontiguousarray(P[:, i]) for i in range(3)]
    rgb = rng.integers(0, 255, n * 3, dtype=np.uint8)
    for maxpts, res, G in ((400, 1e-4, 2), (3000, 1e-9, 3), (400, 1e-3, 1)):
        c = pcv.Context(0, max_points_per_node=maxpts, levels_per_pass=G)
        tree = c.build_octree(x, y, z, rgb, res, bmin, bmax)
        ref = O.build(x, y, z, rgb.reshape(-1, 3), res, bmin, bmax, max_points_per_node=maxpts)
        compare_trees(ref, tree)
        tree.free()
        c.close()
