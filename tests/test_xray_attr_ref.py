"""The exact per-pixel reference of the X-ray attribute strategies (tests/xray_attr_ref.py), validated on the CPU against
the oracle: its pixel assignment reproduces the XRay strategy's bucket sets bit for bit, its ranges are single values
equal to the oracle's bytes where every sum is exact, the oracle lies inside every range on general clouds, and the
oracle's Welford stddev meets the height-stddev tolerance (which pins the oracle's OnlineStats restatement)."""
import numpy as np
import pytest

import oracle_api as O
import xray_attr_ref as R

MPP = 1000


def _points(ref, tmin, tmax, qfg=None):
    q = ref.query(R.location(O.Location, tmin, tmax, qfg), with_intensity=True)
    return q["xyz"], q["rgb"], q["intensity"]


def _build(x, y, z, rgb, inten, res, mpp=MPP):
    bmin = np.array([x.min(), y.min(), z.min()])
    bmax = np.array([x.max(), y.max(), z.max()])
    return O.build(x, y, z, rgb.reshape(-1, 3), res, bmin, bmax, intensity=inten, max_points_per_node=mpp)


@pytest.fixture(scope="module")
def slab():
    import point_cloud_viewer_b200 as pcv

    n = 60_000
    x, y, z, rgb = pcv.synth_points_host(pcv.SYNTH_SLAB_ECEF, 80293751232, 0, n)
    rng = np.random.default_rng(3)
    inten = (rng.random(n) * 1000.0).astype(np.float32)
    bmin, bmax, res = pcv.synth_bbox(pcv.SYNTH_SLAB_ECEF)
    ref = O.build(x, y, z, rgb.reshape(-1, 3), res, bmin, bmax, intensity=inten, max_points_per_node=2000)
    G = pcv.geometry
    q = G.quat_mul(G.quat_from_axis_angle([0, 0, 1], 0.7), G.quat_from_axis_angle([0, 1, 0], -0.9))
    qfg = G.Isometry((4157222.543, 664789.307, 4774952.099), q).inverse().as7()
    d = np.asarray(bmax) - np.asarray(bmin)
    tiles = [(np.asarray(bmin) + [0.2, 0.2, 0.0] * d, np.asarray(bmin) + [0.7, 0.7, 1.0] * d, 96, 64, None),
             (np.array([-40.0, -30.0, -10.0]), np.array([24.0, 34.0, 10.0]), 128, 128, np.asarray(qfg))]
    return ref, tiles


@pytest.fixture(scope="module", params=[0.05, 1e-6], ids=["coarse", "fine"])
def exact(request):
    x, y, z, rgb, inten, cols = R.exact_cloud()
    ref = _build(x, y, z, rgb, inten, request.param)
    allq = ref.query(R.location(O.Location, (-1, -1, -1), (200, 200, 100)), with_intensity=True)
    return ref, R.exact_tiles(allq["xyz"], allq["intensity"], cols), cols


def test_pixel_assignment_reproduces_the_oracle_zbits(slab, exact):
    for ref, tiles in (slab, exact[:2]):
        for tmin, tmax, w, h, qfg in [t if len(t) == 5 else t[1:] for t in tiles]:
            if w * h > 1 << 20:
                continue
            xyz, _, _ = _points(ref, tmin, tmax, qfg)
            bits, over = R.zbits(xyz, tmin, tmax, w, h, qfg)
            _, _, zb_o, zover_o = ref.xray_tile(tmin, tmax, w, h, query_from_global=qfg)
            assert np.array_equal(bits, zb_o) and np.array_equal(over, zover_o)
            assert bits.any()


def test_exact_cloud_reaches_every_face(exact):
    """x == 0 and y == 0 are kept, y == h is dropped (Aabb: the max faces lie outside the half-open box), and x == w is
    dropped under the query frame (Obb: closed faces)."""
    ref, tiles, _ = exact
    seen = set()
    for name, tmin, tmax, w, h, qfg in tiles:
        if w * h > 1 << 20:
            continue
        xyz, _, _ = _points(ref, tmin, tmax, qfg)
        x, y, _, _ = R.discretise(xyz, tmin, tmax, w, h, qfg)
        seen |= {k for k, hit in (("x==0", (x == 0).any()), ("y==0", (y == 0).any()), ("x==w", (x == w).any()), ("y==h", (y == h).any())) if hit}
    assert seen == {"x==0", "y==0", "x==w", "y==h"}, seen


def test_exact_cloud_decodes_every_encoding():
    x, y, z, rgb, inten, _ = R.exact_cloud()
    encs = set()
    for res in (0.05, 1e-6):
        encs |= {m["enc"] for m in _build(x, y, z, rgb, inten, res).nodes.values() if m["num_points"]}
    assert encs == {1, 2, 3, 4}, encs  # Uint8, Uint16, Float32, Float64


INTENSITY_PARAMS = [(0.0, 1000.0), (2.0, 3.0), (1.0, 1.5), (3.0, 60.0)]  # p1 - p0 > 1, == 1, < 1


def test_exact_cloud_single_values_equal_the_oracle(exact):
    ref, tiles, cols = exact
    for name, tmin, tmax, w, h, qfg in tiles:
        if w * h > 1 << 20:
            continue
        xyz, rgb, inten = _points(ref, tmin, tmax, qfg)
        runs = [(R.COLORED, 0.0, 0.0, b) for b in (0.0, 1e9, 1.0)] + [(R.INTENSITY, p0, p1, b) for p0, p1 in INTENSITY_PARAMS for b in (0.0, 1e9, 1.0)]
        for mode, p0, p1, b in runs:
            lo, hi, cov = R.tile_ranges(xyz, rgb, inten, tmin, tmax, w, h, mode, p0, p1, qfg=qfg, bin_size=b, logf_ulps=0)
            if b:
                _, want = ref.xray_tile_attr_binned(tmin, tmax, w, h, mode, b, p0, p1, query_from_global=qfg)
            else:
                _, want = ref.xray_tile_attr(tmin, tmax, w, h, mode, p0, p1, query_from_global=qfg)
            assert np.array_equal(lo, hi), (name, mode, p0, p1, b, int((lo != hi).sum()))
            assert np.array_equal(lo, want), (name, mode, p0, p1, b, np.argwhere(lo != want)[:4])
            assert cov.sum() > 0


def test_general_clouds_oracle_inside_every_range(slab):
    ref, tiles = slab
    for tmin, tmax, w, h, qfg in tiles:
        xyz, rgb, inten = _points(ref, tmin, tmax, qfg)
        for mode, p0, p1, b in [(R.COLORED, 0, 0, 0.0), (R.INTENSITY, 0.0, 1000.0, 0.0), (R.INTENSITY, 100.0, 800.0, 0.0), (R.INTENSITY, 400.0, 401.0, 0.0),
                                (R.COLORED, 0, 0, 7.5), (R.COLORED, 0, 0, 1e-30), (R.INTENSITY, 0.0, 1000.0, 7.5), (R.INTENSITY, 0.0, 1000.0, 1.0)]:
            lo, hi, cov = R.tile_ranges(xyz, rgb, inten, tmin, tmax, w, h, mode, p0, p1, qfg=qfg, bin_size=b)
            if b:
                _, want = ref.xray_tile_attr_binned(tmin, tmax, w, h, mode, b, p0, p1, query_from_global=qfg)
            else:
                _, want = ref.xray_tile_attr(tmin, tmax, w, h, mode, p0, p1, query_from_global=qfg)
            R.check_tile(want, lo, hi, cov, (mode, p0, p1, b))
            assert cov.sum() > 200


def test_oracle_welford_meets_the_stddev_tolerance(slab, exact):
    """Welford in f64 (the oracle's OnlineStats) stays within SD_REL_TOL * max(p0, sd) of the exact stddev, also on a
    column 1e6 m away from the tile's mid height."""
    x, y, z, rgb, inten, (tmin, tmax, w, h) = R.far_cloud()
    far = _build(x, y, z, rgb, inten, 1e-4, mpp=50)
    cases = [(slab[0], t) for t in slab[1]] + [(exact[0], t[1:]) for t in exact[1] if t[3] * t[4] <= 1 << 20] + [(far, (tmin, tmax, w, h, None))]
    for ref, (tmin, tmax, w, h, qfg) in cases:
        xyz, rgb, inten = _points(ref, tmin, tmax, qfg)
        for p0, cm in ((0.05, 0), (0.05, 1), (0.8, 0), (2.5, 1)):
            lo, hi, cov = R.tile_ranges(xyz, rgb, inten, tmin, tmax, w, h, R.HEIGHT_STDDEV, p0, colormap=cm, qfg=qfg)
            _, want = ref.xray_tile_attr(tmin, tmax, w, h, R.HEIGHT_STDDEV, p0, 0.0, cm, query_from_global=qfg)
            R.check_tile(want, lo, hi, cov, (p0, cm))

