"""A plain, high-precision reference of one X-ray attribute tile (colour mean, intensity mean, height stddev; binned or not).

Input: the decoded points of the tile's location (positions, colours, intensities, e.g. from `query_points` over
`location(...)`).  Output: for every pixel and channel the range [lo, hi] of admissible RGBA bytes.

- Pixel assignment restates, in numpy float64 and in the same order of operations, the per-point arithmetic of the X-ray
  kernels: `iso_apply` under a query frame, `(p - tmin) / tdiag * w`, `(1 - ...) * h`, Rust's saturating `as u32` (NaN -> 0)
  and `x < w && y < h`.  `zbits` adds the z bucket; it must reproduce the XRay strategy's bucket sets bit for bit, which
  is what makes the assignment trustworthy.
- A sum of n f32 terms in any order (what f32 atomics produce) lies within gamma_{n-1} * sum |v_i| of the exact sum,
  gamma_k = k u / (1 - k u), u = 2^-24.  Where every partial sum in any order is exactly representable (all terms are
  multiples of the smallest term's lowest set bit g, and sum |v_i| < 2^24 g), the sum is exact and the range is one value.
  Both ends of the envelope go through the monotone f32 steps after the sum (`/ (float)n`, the clamp to [p0, p1],
  `logf(m - p0) / logf(p1 - p0)`, `(v * 255) as u8`) in np.float32 arithmetic; `logf` is glibc's, and each of its finite,
  non-zero results is widened by one ulp on either side (the device `logf` is specified to 1 ulp).
- The binned forms nest two such sums: per (pixel, bin) the bin's mean, then the pixel's sum over its bins' means.
- Height stddev: the exact population stddev of the column's z, to within `SD_REL_TOL * max(p0, sd)`, mapped through the
  clamp and Jet (evaluated at the interval's ends and at every breakpoint inside it) or Purplish in f32.
"""
import ctypes
import math

import numpy as np

F32 = np.float32
U24 = 2.0 ** -24
U53 = 2.0 ** -53
FLT_MAX = float(np.finfo(np.float32).max)
SD_REL_TOL = 1e-6  # what Welford in f64 meets on every cloud of tests/test_xray_attr_ref.py
TRANSPARENT = np.array([255, 255, 255, 0], np.uint8)
LOC_AABB, LOC_OBB = 1, 3
COLORED, INTENSITY, HEIGHT_STDDEV = 1, 2, 3


# ---- location and pixel assignment ------------------------------------------------------------------------
def quat_rot(iso7, p):
    """geometry_host.hpp quat_rot on an (n, 3) array: t = 2 (qv x p); qv x t; t w + c + p, in that order."""
    qv = np.asarray(iso7[3:6], np.float64)
    t = np.cross(qv, p) * 2.0
    c = np.cross(qv, t)
    return t * float(iso7[6]) + c + p


def iso_apply(iso7, p):
    return quat_rot(iso7, p) + np.asarray(iso7[:3], np.float64)


def location(cls, tmin, tmax, qfg=None):
    """The tile's location as the X-ray entry points build it (geometry_host.hpp xray_location): Aabb(box), or
    Obb::from(box).transformed(query_from_global.inverse()).  `cls` is a ctypes Location (the product's or the oracle's)."""
    tmin, tmax = np.asarray(tmin, np.float64), np.asarray(tmax, np.float64)
    bmin, bmax = np.fmin(tmin, tmax), np.fmax(tmin, tmax)
    loc = cls()
    if qfg is None:
        loc.kind = LOC_AABB
        loc.aabb_min = (ctypes.c_double * 3)(*bmin)
        loc.aabb_max = (ctypes.c_double * 3)(*bmax)
        return loc
    q = np.asarray(qfg, np.float64)
    ginv = np.array([0, 0, 0, -q[3], -q[4], -q[5], q[6]], np.float64)
    ginv[:3] = quat_rot(ginv, -q[None, :3])[0]
    centre = np.array([(bmin[k] + bmax[k]) * 0.5 for k in range(3)])
    qfo = ginv.copy()
    qfo[:3] = ginv[:3] + quat_rot(ginv, centre[None])[0]
    ofq = np.array([0, 0, 0, -qfo[3], -qfo[4], -qfo[5], qfo[6]], np.float64)
    ofq[:3] = quat_rot(ofq, -qfo[None, :3])[0]
    loc.kind = LOC_OBB
    loc.query_from_obb = (ctypes.c_double * 7)(*qfo)
    loc.obb_from_query = (ctypes.c_double * 7)(*ofq)
    loc.half_extent = (ctypes.c_double * 3)(*[(bmax[k] - bmin[k]) * 0.5 for k in range(3)])
    return loc


def as_u32(v):
    """Rust `f64 as u32`: truncating, saturating, NaN -> 0."""
    v = np.asarray(v, np.float64)
    out = np.zeros(v.shape, np.int64)
    ok = v > 0
    out[ok] = np.floor(np.minimum(v[ok], 4294967295.0)).astype(np.int64)
    return out


def as_i64(v):
    """Rust `f64 as i64`: truncating, saturating, NaN -> 0."""
    v = np.asarray(v, np.float64)
    out = np.zeros(v.shape, np.int64)
    big, small = v >= 9223372036854775808.0, v <= -9223372036854775808.0
    mid = ~(big | small) & (v == v)
    out[mid] = np.trunc(v[mid]).astype(np.int64)
    out[big] = np.iinfo(np.int64).max
    out[small] = np.iinfo(np.int64).min
    return out


def transformed(xyz, qfg=None):
    p = np.asarray(xyz, np.float64).reshape(-1, 3)
    return iso_apply(qfg, p) if qfg is not None else p.copy()


def discretise(xyz, tmin, tmax, w, h, qfg=None):
    """(x, y, z bucket, transformed points) of every point, before the `x < w && y < h` test."""
    p = transformed(xyz, qfg)
    lo = np.fmin(np.asarray(tmin, np.float64), np.asarray(tmax, np.float64))
    d = np.fmax(np.asarray(tmin, np.float64), np.asarray(tmax, np.float64)) - lo
    x = as_u32((p[:, 0] - lo[0]) / d[0] * float(w))
    y = as_u32((1.0 - (p[:, 1] - lo[1]) / d[1]) * float(h))
    z = as_u32((p[:, 2] - lo[2]) / d[2] * 1024.0)
    return x, y, z, p


def zbits(xyz, tmin, tmax, w, h, qfg=None):
    """The XRay strategy's per-pixel bucket sets: (h, w, 32) uint32 (bucket < 1024) and the (h, w) 'bucket >= 1024' flags."""
    x, y, z, _ = discretise(xyz, tmin, tmax, w, h, qfg)
    m = (x < w) & (y < h)
    px, zz = y[m] * w + x[m], z[m]
    bits = np.zeros((h * w, 32), np.uint32)
    lo = zz < 1024
    np.bitwise_or.at(bits, (px[lo], zz[lo] >> 5), (np.uint32(1) << (zz[lo] & 31).astype(np.uint32)))
    over = np.zeros(h * w, np.uint8)
    over[px[~lo]] = 1
    return bits.reshape(h, w, 32), over.reshape(h, w)


# ---- sums of f32 terms in any order -------------------------------------------------------------------------
def _gamma(k, u):
    k = np.asarray(k, np.float64)
    return k * u / (1.0 - k * u)


def grain(v):
    """The weight of the lowest set bit of each f32 value (inf for zeros and non-finite values)."""
    b = np.asarray(v, np.float32).view(np.uint32).astype(np.int64)
    e, m = (b >> 23) & 0xFF, b & 0x7FFFFF
    m = np.where(e > 0, m | 0x800000, m)
    ex = np.where(e > 0, e - 150, -149)
    g = (m & -m).astype(np.float64) * np.exp2(ex.astype(np.float64))
    g[(m == 0) | (e == 255)] = np.inf
    return g


def _f32_down(v):
    c = v.astype(np.float32)
    c = np.where(c.astype(np.float64) > v, np.nextafter(c, F32(-np.inf)), c)
    return c.astype(np.float32)


def _f32_up(v):
    c = v.astype(np.float32)
    c = np.where(c.astype(np.float64) < v, np.nextafter(c, F32(np.inf)), c)
    return c.astype(np.float32)


class Groups:
    """Points grouped by an int64 key (pixel, or pixel and bin): sorted order and segment starts."""

    def __init__(self, key):
        self.order = np.argsort(key, kind="stable")
        k = key[self.order]
        self.start = np.flatnonzero(np.r_[True, k[1:] != k[:-1]]) if len(k) else np.zeros(0, np.int64)
        self.keys = k[self.start]
        self.count = np.diff(np.r_[self.start, len(k)])

    def reduce(self, ufunc, v):
        v = np.asarray(v)[self.order]
        return ufunc.reduceat(v, self.start) if len(v) else np.zeros(0, v.dtype)


def _quiet(f):  # overflow, inf - inf and 0 / 0 are part of the arithmetic being restated
    def g(*a, **k):
        with np.errstate(all="ignore"):
            return f(*a, **k)

    g.__doc__ = f.__doc__
    return g


@_quiet
def sum_range(g, lo_terms, hi_terms=None):
    """[lo, hi] (f32) of the f32 sum of every group's terms in any order; term i lies in [lo_terms[i], hi_terms[i]]
    (f32 values, one value when hi_terms is None).  Returns (lo, hi, exact)."""
    lo_t = np.asarray(lo_terms, np.float32)
    hi_t = lo_t if hi_terms is None else np.asarray(hi_terms, np.float32)
    same = g.reduce(np.logical_and, lo_t.view(np.uint32) == hi_t.view(np.uint32))
    ends, exact_ends = [], []
    for t, down in ((lo_t, True), (hi_t, False)):  # the f32 sum is monotone in every term: bound each end on its own
        fin = np.isfinite(t)
        t64 = np.where(fin, t, 0).astype(np.float64)
        S = g.reduce(np.add, t64)
        A = g.reduce(np.add, np.abs(t64))
        exact = A < 2.0 ** 24 * g.reduce(np.minimum, grain(t))
        hw = np.where(exact, 0.0, (_gamma(g.count - 1, U24) + _gamma(g.count - 1, U53)) * A * (1 + 2.0 ** -40))
        if down:
            e = np.where(exact, S.astype(np.float32), _f32_down(np.nextafter(S - hw, -np.inf)))
            e = np.where(A * (1 + _gamma(g.count, U24)) >= FLT_MAX, np.minimum(e, F32(FLT_MAX)), e)
        else:
            e = np.where(exact, S.astype(np.float32), _f32_up(np.nextafter(S + hw, np.inf)))
            e = np.where(A * (1 + _gamma(g.count, U24)) >= FLT_MAX, F32(np.inf), e)  # a partial sum may overflow
        # non-finite terms decide the sum on their own: NaN, or +-inf, or NaN when both infinities meet
        nan = g.reduce(np.logical_or, np.isnan(t))
        pinf = g.reduce(np.logical_or, t == np.inf)
        ninf = g.reduce(np.logical_or, t == -np.inf)
        e = e.astype(np.float32)
        e[pinf] = np.inf
        e[ninf] = -np.inf
        e[nan | (pinf & ninf)] = np.nan
        ends.append(e)
        exact_ends.append(exact | nan | pinf | ninf)
    return ends[0], ends[1], same & exact_ends[0] & exact_ends[1]


# ---- the f32 steps after the sum ------------------------------------------------------------------------------
def to_u8(v):
    """Color<f32>::to_u8: (v * 255.) as u8, saturating, NaN -> 0."""
    s = np.asarray(v, np.float32) * F32(255.0)
    out = np.zeros(s.shape, np.int64)
    ok = s > 0
    out[ok] = np.floor(np.minimum(s[ok], F32(255.0))).astype(np.int64)
    return out


_libm = None
_logf_cache = {}


def glibc_logf(a):
    """glibc logf of every element of an f32 array."""
    global _libm
    if _libm is None:
        _libm = ctypes.CDLL("libm.so.6")
        _libm.logf.restype = ctypes.c_float
        _libm.logf.argtypes = [ctypes.c_float]
    a = np.asarray(a, np.float32)
    u, inv = np.unique(a, return_inverse=True)
    r = np.empty(len(u), np.float32)
    for i, v in enumerate(u):
        k = float(v)
        if k != k:
            r[i] = np.nan
            continue
        if k not in _logf_cache:
            _logf_cache[k] = _libm.logf(k)
        r[i] = _logf_cache[k]
    return r[inv].reshape(a.shape)


def _ulp_widen(v, ulps):
    v = np.asarray(v, np.float32)
    if not ulps:
        return v, v
    lo, hi = v.copy(), v.copy()
    w = np.isfinite(v) & (v != 0)
    for _ in range(ulps):
        lo[w] = np.nextafter(lo[w], F32(-np.inf))
        hi[w] = np.nextafter(hi[w], F32(np.inf))
    return lo, hi


def brighten_u8(m_lo, m_hi, p0, p1, logf_ulps=1):
    """[lo, hi] of to_u8(logf(clamp(m) - p0) / logf(p1 - p0)) for m in [m_lo, m_hi] (f32; fmaxf / fminf ignore NaN)."""
    p0, p1 = F32(p0), F32(p1)
    den = glibc_logf(np.array([p1 - p0], np.float32))
    d_lo, d_hi = _ulp_widen(den, logf_ulps)
    outs = []
    for m in (m_lo, m_hi):
        m = np.fmin(np.fmax(np.asarray(m, np.float32), p0), p1)
        n_lo, n_hi = _ulp_widen(glibc_logf(m - p0), logf_ulps)
        for num in (n_lo, n_hi):
            for d in (d_lo, d_hi):
                outs.append(to_u8(num / d[0]))
    o = np.stack(outs)
    return o.min(0), o.max(0)


def jet_base(val):  # xray/src/colormap.rs, as k_xray_resolve_attr evaluates it in f32
    val = np.asarray(val, np.float32)
    f = lambda v, y0, x0, y1, x1: (v - F32(x0)) * (F32(y1) - F32(y0)) / (F32(x1) - F32(x0)) + F32(y0)
    return np.where(val <= F32(-0.75), F32(0.0), np.where(val <= F32(-0.25), f(val, 0.0, -0.75, 1.0, -0.25), np.where(
        val <= F32(0.25), F32(1.0), np.where(val <= F32(0.75), f(val, 1.0, 0.25, 0.0, 0.75), F32(0.0))))).astype(np.float32)


def colormap_u8(colormap, val):
    val = np.asarray(val, np.float32)
    if colormap == 0:
        return np.stack([to_u8(jet_base(val - F32(0.5))), to_u8(jet_base(val)), to_u8(jet_base(val + F32(0.5)))], -1)
    a = F32(1.0) - val
    return np.stack([to_u8(a * F32(0.8)), to_u8(a * F32(0.8)), to_u8(a * F32(1.0))], -1)


_JET_BREAKS = [F32(b) - F32(o) for b in (-0.75, -0.25, 0.25, 0.75) for o in (-0.5, 0.0, 0.5)]


def stddev_u8(sd_lo, sd_hi, p0, colormap):
    """[lo, hi] (n, 3) of the colormap of clamp((float)sd, 0, p0) / p0 for sd in [sd_lo, sd_hi] (float64)."""
    p0 = F32(p0)

    def val(sd):
        s = np.minimum(np.maximum(sd, F32(0.0)), p0)
        return (s / p0).astype(np.float32)

    v_lo, v_hi = val(_f32_down(np.asarray(sd_lo, np.float64))), val(_f32_up(np.asarray(sd_hi, np.float64)))
    cands = [v_lo, v_hi]
    for b in _JET_BREAKS:  # Jet is monotone between its breakpoints
        for c in (np.nextafter(b, F32(-np.inf)), b, np.nextafter(b, F32(np.inf))):
            cands.append(np.where((v_lo < c) & (c < v_hi), c, v_lo).astype(np.float32))
    o = np.stack([colormap_u8(colormap, c) for c in cands])
    return o.min(0), o.max(0)


# ---- one tile ---------------------------------------------------------------------------------------------------
def exact_moments(g, z):
    """Per group: mean and population variance of z in float64, by the corrected two-pass algorithm (relative error of
    the variance of order n 2^-53, far below SD_REL_TOL for the clouds here)."""
    n = g.count.astype(np.float64)
    m1 = g.reduce(np.add, z) / n
    inv = np.repeat(np.arange(len(g.count)), g.count)
    zs = np.asarray(z, np.float64)[g.order]
    d = zs - m1[inv]
    c = np.add.reduceat(d, g.start) if len(d) else np.zeros(0)
    m = m1 + c / n
    d = zs - m[inv]
    s1 = np.add.reduceat(d, g.start) if len(d) else np.zeros(0)
    var = (np.add.reduceat(d * d, g.start) if len(d) else np.zeros(0)) / n - (s1 / n) ** 2
    return m, np.maximum(var, 0.0)


@_quiet
def tile_ranges(xyz, rgb, intensity, tmin, tmax, w, h, mode, p0=0.0, p1=0.0, colormap=0, qfg=None, bin_size=0.0, logf_ulps=1,
                sd_rel_tol=SD_REL_TOL):
    """(lo, hi): (h, w, 4) int arrays of admissible bytes per pixel and channel, and `covered`: (h, w) bool, the pixels
    with at least one counted point.  Points with a negative intensity do not count in the intensity strategy (the
    reference abandons the whole batch at the first one, generation.rs:245-247; the restatement skips the point)."""
    x, y, _, p = discretise(xyz, tmin, tmax, w, h, qfg)
    keep = (x < w) & (y < h)
    rgb = np.asarray(rgb, np.uint8).reshape(-1, 3)
    inten = None if intensity is None else np.asarray(intensity, np.float32).reshape(-1)
    if mode == INTENSITY:
        keep &= ~(inten < 0)
    px = (y * w + x)[keep]
    lo = np.tile(TRANSPARENT, (h * w, 1))
    hi = lo.copy()
    covered = np.zeros(h * w, bool)
    if len(px) == 0:
        return lo.reshape(h, w, 4), hi.reshape(h, w, 4), covered.reshape(h, w)
    if mode == COLORED:
        vals = [(rgb[keep, k].astype(np.float32) / F32(255.0)).astype(np.float32) for k in range(3)]
    elif mode == INTENSITY:
        vals = [inten[keep]]
    if bin_size != 0.0:
        assert mode in (COLORED, INTENSITY)
        bins = as_i64(inten[keep].astype(np.float64) / float(bin_size))
        order = np.lexsort((bins, px))
        key = np.empty(len(px), np.int64)
        ps, bs = px[order], bins[order]
        newg = np.r_[True, (ps[1:] != ps[:-1]) | (bs[1:] != bs[:-1])]
        key[order] = np.cumsum(newg) - 1
        gb = Groups(key)
        bin_px = px[gb.order][gb.start]
        gp = Groups(bin_px)
        out_lo, out_hi = [], []
        for v in vals:
            s_lo, s_hi, _ = sum_range(gb, v)
            cnt = gb.count.astype(np.float32)
            b_lo, b_hi = (s_lo / cnt).astype(np.float32), (s_hi / cnt).astype(np.float32)
            t_lo, t_hi, _ = sum_range(gp, b_lo, b_hi)
            nb = gp.count.astype(np.float32)
            out_lo.append((t_lo / nb).astype(np.float32))
            out_hi.append((t_hi / nb).astype(np.float32))
        keys = gp.keys
    elif mode in (COLORED, INTENSITY):
        gp = Groups(px)
        out_lo, out_hi = [], []
        for v in vals:
            s_lo, s_hi, _ = sum_range(gp, v)
            n = gp.count.astype(np.float32)
            out_lo.append((s_lo / n).astype(np.float32))
            out_hi.append((s_hi / n).astype(np.float32))
        keys = gp.keys
    else:
        gp = Groups(px)
        keys = gp.keys
        _, var = exact_moments(gp, p[keep, 2])
        sd = np.sqrt(var)
        tol = sd_rel_tol * np.maximum(float(p0), sd)
        c_lo, c_hi = stddev_u8(np.maximum(sd - tol, 0.0), sd + tol, p0, colormap)
    covered[keys] = True
    if mode == COLORED:
        for k in range(3):
            lo[keys, k], hi[keys, k] = to_u8(out_lo[k]), to_u8(out_hi[k])
    elif mode == INTENSITY:
        g_lo, g_hi = brighten_u8(out_lo[0], out_hi[0], p0, p1, logf_ulps)
        for k in range(3):
            lo[keys, k], hi[keys, k] = g_lo, g_hi
    else:
        lo[keys, :3], hi[keys, :3] = c_lo, c_hi
    lo[keys, 3] = hi[keys, 3] = 255
    return lo.reshape(h, w, 4), hi.reshape(h, w, 4), covered.reshape(h, w)


def check_tile(got, lo, hi, covered, what=""):
    """Asserts coverage (alpha) and that every byte lies in its range; returns the number of single-valued channels."""
    got = np.asarray(got, np.uint8)
    assert np.array_equal(got[..., 3] == 255, covered), (what, "covered pixels", int((got[..., 3] == 255).sum()), int(covered.sum()))
    bad = (got < lo) | (got > hi)
    if bad.any():
        i = np.argwhere(bad)[:5]
        raise AssertionError("%s: %d bytes outside their range, e.g. %s" % (
            what, int(bad.sum()), [(tuple(int(v) for v in t), int(got[tuple(t)]), int(lo[tuple(t)]), int(hi[tuple(t)])) for t in i]))
    return int((lo == hi)[covered].sum())


# ---- scenes ------------------------------------------------------------------------------------------------------
EXACT_COUNTS = (1, 2, 3, 7, 255, 256, 4097, 150_000)
EDGE_INTENSITIES = (  # columns of 2 or 4 points; what each checks is in its name
    ("negative_skipped", [5.0, -1.0, 7.0, -1.0]),
    ("only_negative", [-1.0, -2.0]),
    ("minus_zero_counts", [-0.0, 4.0]),
    ("nan", [np.nan, 3.0]),
    ("plus_inf", [np.inf, 2.0]),
    ("sum_overflows", [3e38, 3e38]),
)
FACES = ("x_min", "x_max", "y_min", "y_max")
FACE_TAG = {f: 1001.0 + i for i, f in enumerate(FACES)}
EXACT_BOX = (96, 64, 16.0)  # the main tile: 96 x 64 pixels of 1 m, z in [0, 16)


def _rgb_of(inten):
    """Colours in {0, 255}, a function of the intensity: a bin of width <= 1 over integer intensities has one colour."""
    i = np.where(np.isfinite(inten), np.minimum(np.abs(inten), 1e9), 0).astype(np.int64)
    return (np.stack([(i >> k) & 1 for k in range(3)], 1) * 255).astype(np.uint8)


def exact_cloud(seed=5):
    """Columns at pixel centres of the main tile whose sums are exact in f32 in any order (colours in {0, 1}, integer
    intensities with sums < 2^24, z on a 0.25 m grid), one column per count of EXACT_COUNTS and per edge of
    EDGE_INTENSITIES, and one point on each face of the main tile (intensity FACE_TAG[face]).
    Returns (x, y, z, rgb (n, 3), intensity, columns {name: (cx, cy)})."""
    rng = np.random.default_rng(seed)
    xs, ys, zs, its, cols = [], [], [], [], {}
    specs = [("count_%d" % n, rng.integers(0, 101, n).astype(np.float32)) for n in EXACT_COUNTS] + [(nm, np.array(v, np.float32)) for nm, v in EDGE_INTENSITIES]
    for k, (name, inten) in enumerate(specs):
        cx, cy = 4 + 6 * k, 10 + 3 * k
        cols[name] = (cx, cy)
        n = len(inten)
        xs.append(np.full(n, cx + 0.5))
        ys.append(np.full(n, cy + 0.5))
        zs.append(6.0 + (np.arange(n) % 16) * 0.25)
        its.append(inten)
    W, H, _ = EXACT_BOX
    for f, (fx, fy) in zip(FACES, ((0.0, 20.5), (float(W), 20.5), (30.5, 0.0), (30.5, float(H)))):
        xs.append(np.array([fx]))
        ys.append(np.array([fy]))
        zs.append(np.array([8.0]))
        its.append(np.array([FACE_TAG[f]], np.float32))
    x, y, z, inten = np.concatenate(xs), np.concatenate(ys), np.concatenate(zs), np.concatenate(its).astype(np.float32)
    return x, y, z, _rgb_of(inten), inten, cols


def exact_tiles(xyz, inten, cols):
    """The tiles of the exact cloud, from its decoded points: the main tile's x / y faces are the decoded coordinates of
    the face points, so those points land exactly on the faces.  Returns [(name, tmin, tmax, w, h, qfg)]."""
    face = {f: np.asarray(xyz)[np.asarray(inten) == FACE_TAG[f]][0] for f in FACES}
    x0, x1, y0, y1 = face["x_min"][0], face["x_max"][0], face["y_min"][1], face["y_max"][1]
    cx, cy = cols["count_4097"]
    shift = np.array([-16.0, -8.0, 0.0])
    frame = np.array([-16.0, -8.0, 0.0, 0.0, 0.0, 0.0, 1.0])  # a translation: the query-frame path with exact arithmetic
    return [
        ("96x64", (x0, y0, 0.0), (x1, y1, 16.0), 96, 64, None),
        ("96x64_frame", tuple(np.array([x0, y0, 0.0]) + shift), tuple(np.array([x1, y1, 16.0]) + shift), 96, 64, frame),
        ("31x33", (x0, y0, 0.0), (x0 + 31.0, y0 + 33.0, 16.0), 31, 33, None),
        ("1x1", (cx, cy, 0.0), (cx + 1.0, cy + 1.0, 16.0), 1, 1, None),
        ("4096x4096", (x0, y0, 0.0), (x1, y1, 16.0), 4096, 4096, None),
    ]


def far_cloud():
    """Height stddev far from the tile's mid height: two columns of 1 cm spread at +-1e6 m from the mid height of a 4e6 m
    tall tile, one near it, and two points that stretch the octree's box.  Tile: [0, 0, -2e6] .. [4, 4, 2e6], 4 x 4."""
    k = np.arange(64)
    spread = (k % 5) * 0.0025
    x = np.concatenate([np.full(64, 0.5), np.full(64, 2.5), np.full(64, 1.5), [-1.0, 5.0]])
    y = np.concatenate([np.full(64, 0.5), np.full(64, 1.5), np.full(64, 2.5), [-1.0, 5.0]])
    z = np.concatenate([1e6 + spread, -1e6 + spread, 3.0 + spread, [-2.1e6, 2.1e6]])
    inten = (k % 7).astype(np.float32)
    inten = np.concatenate([inten, inten, inten, [0, 0]]).astype(np.float32)
    return x, y, z, _rgb_of(inten), inten, ((0.0, 0.0, -2e6), (4.0, 4.0, 2e6), 4, 4)
