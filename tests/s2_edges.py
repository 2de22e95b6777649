"""Deterministic ECEF point sets at the places where S2 cell arithmetic goes wrong (host numpy, no GPU): the eight cube corners,
the twelve cube edges, the whole globe, points on cell and face boundaries at several levels with their one-ulp neighbours, exact
face ties and signed zeros, and one heavily repeated position among single-point cells.  Every point lies within the S2 split's
valid radius band [6352800, 6384400] m (csrc/s2.h kEarthRadiusMinM / kEarthRadiusMaxM)."""
import itertools

import numpy as np

R_MIN, R_MAX = 6352800.0, 6384400.0
R = 6371000.0
BOUNDARY_LEVELS = (1, 5, 10, 20, 25, 30)


def _tangent_patch(rng, direction, n, half_width, half_height):
    """n points in a box of the local tangent frame at R * direction: +-half_width across, +-half_height along the normal."""
    d = np.asarray(direction, np.float64)
    d = d / np.linalg.norm(d)
    ref = np.array([0.0, 0.0, 1.0]) if abs(d[2]) < 0.9 else np.array([1.0, 0.0, 0.0])
    e1 = np.cross(ref, d)
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(d, e1)
    a = rng.uniform(-half_width, half_width, (n, 1))
    b = rng.uniform(-half_width, half_width, (n, 1))
    h = rng.uniform(-half_height, half_height, (n, 1))
    return R * d + a * e1 + b * e2 + h * d


def corner_directions():
    """The eight cube corners (+-1, +-1, +-1) / sqrt(3); each touches three faces."""
    return [np.array(s, np.float64) / np.sqrt(3.0) for s in itertools.product((1.0, -1.0), repeat=3)]


def edge_directions():
    """The midpoints of the twelve cube edges, e.g. (1, 1, 0) / sqrt(2); each touches two faces."""
    out = []
    for zero in range(3):
        for s in itertools.product((1.0, -1.0), repeat=2):
            v = np.zeros(3)
            v[[k for k in range(3) if k != zero]] = s
            out.append(v / np.sqrt(2.0))
    return out


def corners(per_patch=40_000, seed=11):
    """8 patches about 600 m wide and 100 m tall, one centred on each cube corner, patch after patch."""
    rng = np.random.default_rng(seed)
    return np.concatenate([_tangent_patch(rng, d, per_patch, 300.0, 50.0) for d in corner_directions()])


def edges(per_patch=20_000, seed=12):
    """12 patches of the same size, one on the midpoint of each cube edge."""
    rng = np.random.default_rng(seed)
    return np.concatenate([_tangent_patch(rng, d, per_patch, 300.0, 50.0) for d in edge_directions()])


def globe(n=1_000_000, seed=13):
    """Uniform directions on the sphere, radius uniform in the valid band: all six faces and every sign combination."""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1)[:, None]
    return v * rng.uniform(R_MIN, R_MAX, (n, 1))


def st_to_uv(s):
    """The inverse of the quadratic projection (the published S2 STtoUV)."""
    s = np.asarray(s, np.float64)
    return np.where(s >= 0.5, (4.0 * s * s - 1.0) / 3.0, (1.0 - 4.0 * (1.0 - s) * (1.0 - s)) / 3.0)


def face_uv_to_xyz(face, u, v):
    """The published S2 faceUVtoXYZ: an (unnormalised) direction on `face` at (u, v)."""
    one = np.ones_like(u)
    table = [(one, u, v), (-u, one, v), (-u, -v, one), (-one, -v, -u), (v, -one, -u), (v, u, -one)]
    out = np.zeros((len(u), 3))
    for f in range(6):
        m = face == f
        out[m] = np.stack([c[m] for c in table[f]], 1)
    return out


def boundaries(per_level=400, seed=14):
    """Points on cell corners and their one-ulp neighbours, exact face ties and signed zeros.

    For every level in BOUNDARY_LEVELS: random (face, i, j) with i, j in [0, 2^level] (the far edge included), st = i / 2^level,
    uv by the inverse quadratic, the face's direction, scaled to a random valid radius; then each such point again with one
    component moved by one ulp up or down.  Ties: |x| = |y|, |x| = |z|, |y| = |z| with the third component smaller or larger,
    |x| = |y| = |z| under all eight signs, and points with +0.0 / -0.0 components."""
    rng = np.random.default_rng(seed)
    base = []
    for level in BOUNDARY_LEVELS:
        size = 1 << level
        face = rng.integers(0, 6, per_level)
        s = rng.integers(0, size + 1, per_level) / size
        t = rng.integers(0, size + 1, per_level) / size
        d = face_uv_to_xyz(face, st_to_uv(s), st_to_uv(t))
        base.append(d / np.linalg.norm(d, axis=1)[:, None] * rng.uniform(R_MIN + 1.0, R_MAX - 1.0, (per_level, 1)))
    base = np.concatenate(base)
    out = [base]
    for k in range(3):
        for toward in (np.inf, -np.inf):
            q = base.copy()
            q[:, k] = np.nextafter(q[:, k], toward)
            out.append(q)
    ties = []
    for a, b in ((0, 1), (0, 2), (1, 2)):
        c = 3 - a - b
        for lo, hi in ((-0.99, 0.99), (1.01, 3.0)):  # the tied pair largest / the third component largest
            n = 200
            t3 = rng.uniform(lo, hi, n) * rng.choice((-1.0, 1.0), n)
            r = rng.uniform(R_MIN + 1.0, R_MAX - 1.0, n)
            s = r / np.sqrt(2.0 + t3 * t3)
            p = np.zeros((n, 3))
            p[:, a] = s * rng.choice((-1.0, 1.0), n)
            p[:, b] = s * rng.choice((-1.0, 1.0), n)
            p[:, c] = t3 * s
            ties.append(p)
    for signs in itertools.product((1.0, -1.0), repeat=3):
        s = rng.uniform(R_MIN + 1.0, R_MAX - 1.0, 20) / np.sqrt(3.0)
        ties.append(np.stack([signs[0] * s, signs[1] * s, signs[2] * s], 1))
    zeros = []
    for axis in range(3):
        for sign in (1.0, -1.0):
            for z1, z2 in itertools.product((0.0, -0.0), repeat=2):
                p = np.zeros(3)
                p[axis] = sign * R
                others = [k for k in range(3) if k != axis]
                p[others[0]], p[others[1]] = z1, z2
                zeros.append(p)
    m = globe(200, seed + 1)  # one signed zero among non-zero components
    for k in range(3):
        q = m.copy()
        q[:, k] = np.where(np.arange(len(q)) % 2 == 0, 0.0, -0.0)
        q *= R / np.linalg.norm(q, axis=1)[:, None]
        zeros.extend(q)
    return np.concatenate(out + ties + [np.array(zeros)])


HEAVY_POINT = np.array([1.75e6, -4.9e6, -3.55e6])  # southern and western hemisphere (y < 0, z < 0), on face 4


def heavy(copies=10_000, singles=2000, seed=15):
    """`copies` copies of one position (one cell holding more than a 2048-point query tile at every level) interleaved with
    `singles` distinct points within a few kilometres of it (single-point cells at fine levels)."""
    rng = np.random.default_rng(seed)
    p0 = HEAVY_POINT * (R / np.linalg.norm(HEAVY_POINT))
    single = p0 + rng.uniform(-3000.0, 3000.0, (singles, 3))
    pts = np.concatenate([np.repeat(p0[None, :], copies, 0), single])
    return pts[rng.permutation(len(pts))]


def all_fixtures():
    """name -> (n, 3) float64 points."""
    return dict(corners=corners(), edges=edges(), globe=globe(), boundaries=boundaries(), heavy=heavy())


def attributes(n, seed=0):
    """Deterministic colour (n, 3) uint8 and intensity (n,) float32 for n points."""
    k = np.arange(n, dtype=np.int64) + seed
    rgb = np.stack([(k * 7) % 256, (k * 13 + 5) % 256, (k >> 8) % 256], 1).astype(np.uint8)
    return np.ascontiguousarray(rgb), ((k * 31) % 1000).astype(np.float32)
