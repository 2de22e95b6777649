"""Pins of the inpainting restatement (tests/xray_inpaint_ref.py) that the GPU tests compare against: the close against scipy's
binary morphology, the fill's distances against scipy's exact Euclidean distance transform, its tie order against brute force,
the blend against hand-computed f32 values, the stitch and the spatial ids.  No GPU."""
import numpy as np
import pytest
from scipy import ndimage

import xray_inpaint_ref as R


@pytest.mark.parametrize("k", [1, 2, 3, 8, 40])
def test_close_equals_scipy_dilation_then_erosion(k):
    rng = np.random.default_rng(k)
    for shape, p in (((64, 64), 0.9), ((37, 53), 0.7), ((64, 64), 0.02), ((20, 90), 0.5)):
        m = rng.random(shape) > p
        st = np.ones((2 * k + 1, 2 * k + 1), bool)
        want = ndimage.binary_erosion(ndimage.binary_dilation(m, st, border_value=0), st, border_value=1)
        assert np.array_equal(R.close(m, k), want), (k, shape, p)
    # empty and full masks
    assert not R.close(np.zeros((16, 16), bool), k).any()
    assert R.close(np.ones((16, 16), bool), k).all()


@pytest.mark.parametrize("seed", range(4))
def test_fill_distances_equal_the_exact_distance_transform(seed):
    rng = np.random.default_rng(seed)
    sample = rng.random((64, 48)) > 0.97
    sample[5, 7] = True
    holes = ~sample
    hr, hc, sr, sc = R.nearest_sample(sample, holes)
    assert sample[sr, sc].all()
    d2 = (hr - sr) ** 2 + (hc - sc) ** 2
    edt = ndimage.distance_transform_edt(~sample)
    assert np.array_equal(d2, np.round(edt[hr, hc] ** 2).astype(np.int64))


def _brute(sample, holes):
    sr, sc = np.nonzero(sample)
    out = {}
    for r, c in zip(*np.nonzero(holes)):
        d = (sr - r) ** 2 + (sc - c) ** 2
        best = min(zip(d, sc, sr))  # distance, then the smaller column, then the smaller row
        out[(r, c)] = (best[2], best[1])
    return out


@pytest.mark.parametrize("seed", range(6))
def test_fill_tie_order_equals_brute_force(seed):
    rng = np.random.default_rng(100 + seed)
    # lattices and symmetric patterns: most hole pixels have several nearest samples
    h, w = 17, 19
    sample = np.zeros((h, w), bool)
    step = 2 + seed % 3
    sample[::step, ::step] = True
    sample[rng.integers(0, h, 3), rng.integers(0, w, 3)] = True
    if seed % 2:
        sample = sample | sample[::-1, ::-1]
    holes = ~sample
    hr, hc, sr, sc = R.nearest_sample(sample, holes)
    want = _brute(sample, holes)
    for r, c, a, b in zip(hr, hc, sr, sc):
        assert (a, b) == want[(r, c)], (r, c)


def test_fill_ties_by_hand():
    s = np.zeros((5, 5), bool)
    s[0, 2] = s[4, 2] = s[2, 0] = s[2, 4] = True  # (2, 2) is at distance 2 from all four
    hr, hc, sr, sc = R.nearest_sample(s, np.eye(5, dtype=bool) & ~s)
    got = {(r, c): (a, b) for r, c, a, b in zip(hr, hc, sr, sc)}
    assert got[(2, 2)] == (2, 0)  # the smallest column
    s = np.zeros((5, 5), bool)
    s[0, 2] = s[4, 2] = True
    hr, hc, sr, sc = R.nearest_sample(s, np.eye(5, dtype=bool))
    got = {(r, c): (a, b) for r, c, a, b in zip(hr, hc, sr, sc)}
    assert got[(2, 2)] == (0, 2)  # same column: the smaller row


def test_inpaint_fills_small_holes_only():
    img = np.zeros((32, 32, 4), np.uint8)
    img[:, :16] = (10, 20, 30, 255)
    img[5, 5] = (0, 0, 0, 0)      # a one-pixel hole: filled from its left neighbour (smallest column among four at distance 1)
    img[4, 4] = (99, 98, 97, 255)
    out, holes = R.inpaint(img, 1)
    assert holes == 1 and tuple(out[5, 5]) == (10, 20, 30, 255)
    out, holes = R.inpaint(img, 3)  # the right half stays empty: only the 3 columns next to the border close
    assert holes == 1 and (out[:, 17:, 3] == 0).all()


def test_blend_by_hand():
    T = 4
    nb = np.zeros((1, T, 4), np.uint8)
    cur = np.full((1, T, 4), 255, np.uint8)
    nb[0, :, 0] = 200
    cur[0, :, 0] = 101
    v = R.blend(nb, cur, T, 1)
    # wt = i / 3 in f32; 200 * wt + 101 * (1 - wt), each step rounded to f32, then rounded half away from zero
    f = np.float32
    want0 = []
    for i in range(T):
        wt = f(i) / f(3)
        want0.append(int(np.floor(float(f(f(200) * wt) + f(f(101) * f(f(1) - wt))) + 0.5)))
    assert list(v[0, :, 0]) == want0 == [101, 134, 167, 200]
    assert list(v[0, :, 3]) == [255, 170, 85, 0]
    # a value at exactly .5 rounds away from zero: 1 * 0.5 + 0 * 0.5 with T - 1 = 2 at i = 1
    nb = np.array([[[1, 3, 5, 7]] * 3], np.uint8)
    cur = np.zeros((1, 3, 4), np.uint8)
    assert list(R.blend(nb, cur, 3, 1)[0, 1]) == [1, 2, 3, 4]
    assert R.blend(nb.transpose(1, 0, 2), cur.transpose(1, 0, 2), 3, 0)[1, 0].tolist() == [1, 2, 3, 4]


def test_stitch_takes_the_facing_halves_and_quarters():
    T = 4
    tiles = {}
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            t = np.zeros((T, T, 4), np.uint8)
            t[..., 0] = 10 * (dx + 1) + (dy + 1)
            t[..., 1] = np.arange(T)[:, None] * T + np.arange(T)[None, :]
            t[..., 3] = 255
            tiles[(5 + dx, 5 + dy)] = t
    s = R.stitch(5, 5, tiles, T)
    w = T // 2
    assert (s[w:w + T, w:w + T] == tiles[(5, 5)]).all()
    assert (s[:w, :w] == tiles[(4, 6)][w:, w:]).all()       # TopLeft: its bottom-right quarter
    assert (s[:w, w:3 * w] == tiles[(5, 6)][w:, :]).all()   # Top: its bottom half
    assert (s[w:3 * w, 3 * w:] == tiles[(6, 5)][:, :w]).all()  # Right: its left half
    assert (s[3 * w:, 3 * w:] == tiles[(6, 4)][:w, :w]).all()  # BottomRight: its top-left quarter
    s = R.stitch(5, 5, {(5, 5): tiles[(5, 5)]}, T)
    assert (s[:w] == R.TRANSPARENT).all() and (s[:, 3 * w:] == R.TRANSPARENT).all()


def test_spatial_ids_and_neighbours():
    for level in range(5):
        for i in range(4 ** level):
            x, y = R.xy(level, i)
            assert R.index_of(level, x, y) == i
    assert R.xy(1, 1) == (0, 1) and R.xy(1, 2) == (1, 0)  # bit 0 of a digit: +y, bit 1: +x
    assert R.neighbor(1, 0, 0, 1) == 1 and R.neighbor(1, 0, -1, 0) is None and R.neighbor(2, 10, 1, 0) is None and R.neighbor(2, 5, 1, 0) == 7
