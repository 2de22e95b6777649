"""Build cases that steer build_octree into every division mode, record width and pass encoding of csrc/build_host.hpp.

The level table (make_level_table) fixes the division mode of a whole build from its root cube:
  3  power-of-two edges: the division is an exact multiply
  2  Markstein sequence without checks: the root cube keeps every coordinate in [2^-300, 2^300), only raw inputs are checked
  1  Markstein sequence, every numerator range-checked; a flagged block repeats its tile with the IEEE operator
  0  IEEE division: an edge has an all-ones significand (or lies outside 2^+-500)
Each case picks a box and a resolution for its target mode and profile, and a cloud that reaches every level of the tree:
a chain of more than max_points_per_node points at the min corner keeps splitting down to the last level, and a few points
per level just above that chain's centre planes leave a leaf at every level, so every pass runs and every leaf encoding is
placed.  tests/test_build_modes.py checks that the cases reach what they claim; tests/test_build_modes_gpu.py builds them.
"""
import numpy as np

from tb_api import level_table

ENC_U8, ENC_U16, ENC_F32, ENC_F64 = 1, 2, 3, 4
OFFSET = (4.1e6, 6.6e5, 4.7e6)
PASS_TILE, PLACE_TILE = 1792, 2048  # kTilePoints, kPlaceTile (csrc/build_host.hpp)

# (bmin, root edge, environment) per box.  Every box is a cube: bmax = bmin + E exactly on every axis.
_E0 = float(np.nextafter(1024.0, 0.0))  # all-ones significand: div_known_ok fails on every level
BOXES = {
    "pow2": (OFFSET, 256.0, {}),                                             # mode 3
    "offset": (OFFSET, 200.0, {}),                                           # mode 2
    "zero": ((0.0, -60.0, -0.0), 200.0, {}),                                 # mode 1: the box spans zero
    "small": ((0.0, -0.25, 0.0), 0.7, {}),                                   # mode 1: edges below 1, tiny codes decode subnormal
    "checked": (OFFSET, 200.0, {"PCV_CHECKED_FAST": "1"}),                   # mode 1: per-numerator checks kept
    "pow2_checked": ((0.0, 0.0, 0.0), 256.0, {"PCV_NO_POW2": "1"}),          # mode 1: power-of-two edge, no exact scaling
    "ones": ((-1000.0, -24.0, -512.5), _E0, {}),                             # mode 0
}
BOX_MODE = {"pow2": 3, "offset": 2, "zero": 1, "small": 1, "checked": 1, "pow2_checked": 1, "ones": 0}

# Resolution as a fraction of the root edge.  narrow: levels 1-5 Float32, 6-13 Uint16, 14-22 Uint8 (16-byte records).
# wide: levels 1-7 Float64 (32-byte records), 8-15 Float32, 16-23 Uint16, 24-32 Uint8.
PROFILES = {"narrow": 1.1 * 2.0 ** -22, "wide": 1.1 * 2.0 ** -32}


def box(name):
    bmin, E, env = BOXES[name]
    bmin = np.array(bmin, np.float64)
    bmax = bmin + E
    assert np.all(bmax - bmin == E), (name, bmax - bmin, E)
    return bmin, bmax, E, dict(env)


# ---- clouds (rows of (x, y, z); every generator is deterministic in its rng) ---------------------------------------------
def _ladder(rng, bmin, E, depth, maxpts, chain):
    """`chain` points within E * 2^-(depth + 2) of the min corner (they share every node down to the last level) and 2..9 points
    per level j < depth in octant 7 of the min-corner node of level j: a leaf at every level 1..depth."""
    rows = [bmin + E * 2.0 ** -(depth + 2) * rng.random((chain, 3))]
    for j in range(depth):
        rows.append(bmin + E * 2.0 ** -j * (0.55 + 0.4 * rng.random((2 + j % 8, 3))))
    return rows


def _clustered(rng, bmin, E, n):
    cen = bmin + E * (0.05 + 0.9 * rng.random((24, 3)))
    k = rng.integers(0, 24, n)
    P = cen[k] + rng.normal(0, 1, (n, 3)) * (E * 1e-3 * (1 + 30 * rng.random(24)))[k, None]
    return np.clip(P, bmin, bmin + E)


def cloud_clean(rng, bmin, E, depth, maxpts, n):
    return np.concatenate(_ladder(rng, bmin, E, depth, maxpts, maxpts + 40) + [_clustered(rng, bmin, E, n)])


# Values that are not in div_known's proven range, or whose quotient underflows: zero of either sign, below 2^-500 and
# subnormal.  Inside the box where it touches zero, on its min corner otherwise (bmin + E * s rounds to bmin).
SPECIALS = (-0.0, 1e-200, 2.0 ** -500, float(np.nextafter(2.0 ** -500, 0.0)), 2.2250738585072014e-308, 1e-310, 3e-320, 5e-324)


def cloud_degenerate(rng, bmin, E, depth, maxpts, n):
    """Points exactly on the min corner (more than maxpts: the min-corner node keeps splitting), on the centre planes, on the max
    corner, and coordinates from SPECIALS next to the min corner, mixed axis by axis with the clean cloud."""
    rows = _ladder(rng, bmin, E, depth, maxpts, maxpts + 40)
    rows.append(np.tile(bmin, (maxpts + 1, 1)))
    centre, top = bmin + E / 2, bmin + E
    for v in (centre, top):
        rows.append(np.tile(v, (40, 1)))
        for a in range(3):  # one coordinate on the plane, the others anywhere
            r = bmin + E * rng.random((20, 3))
            r[:, a] = v[a]
            rows.append(r)
    sp = []
    for s in SPECIALS:
        for a in range(3):
            r = np.tile(bmin, (maxpts // 4 + 3, 1))
            r[:, a] = s if bmin[a] == 0.0 else bmin[a] + E * s
            r[1::2, (a + 1) % 3] = bmin[(a + 1) % 3] + E * 2.0 ** -(depth + 3)
            sp.append(r)
    # ... and spread over every node whose min is 0 on that axis, so that split Float64 nodes and leaves carry them, with random
    # subnormals: for about one in fifty the unguarded reciprocal division rounds differently from the IEEE operator
    for a in range(3):
        if bmin[a] == 0.0:
            r = bmin + E * rng.random((60 * len(SPECIALS) + 1200, 3))
            r[:, a] = np.concatenate([np.repeat(SPECIALS, 60), rng.integers(1, 2 ** 52, 1200).view(np.float64)])
            sp.append(r)
    rows += sp
    rows.append(_clustered(rng, bmin, E, n))
    P = np.concatenate(rows)
    return P[rng.permutation(len(P))]


WILD = (1e300, -1e300, np.inf, -np.inf, np.nan, 2.0 ** 399, -(2.0 ** 399))


def cloud_wild(rng, bmin, E, depth, maxpts, n):
    """The clean cloud with WILD values and points far outside the box in single coordinates and whole rows."""
    P = cloud_clean(rng, bmin, E, depth, maxpts, n)
    far = (bmin - 10 * E, bmin + 1e6, np.zeros(3))
    for v in list(WILD) + list(far):
        for a in range(3):
            P[rng.integers(0, len(P), 7), a] = v[a] if np.ndim(v) else v
    P[rng.integers(0, len(P), 5)] = np.inf
    P[rng.integers(0, len(P), 5)] = np.nan
    return P


def cloud_tiles(rng, bmin, E, depth, maxpts, n):
    """Leaves whose counts sit on the tile edges: maxpts must be 2049.  Level-1 octant 0 splits into level-2 leaves of 1791, 1792,
    1793 (partition tile), 2047, 2048 (place tile) and 2049 (= maxpts, not split) points; octant 4 into level-2 leaves of 400 + r
    points for r = 0..7; octant 2 holds one level-2 cell of maxpts + 1 points, which splits once more.  The ladder keeps the
    min-corner level-2 cell of octant 0."""
    assert maxpts == 2049
    rows = _ladder(rng, bmin, E, depth, maxpts, maxpts + 40)
    e2 = E / 4
    counts = [PASS_TILE - 1, PASS_TILE, PASS_TILE + 1, PLACE_TILE - 1, PLACE_TILE, PLACE_TILE + 1, 1000] + [400 + r for r in range(8)]
    cells = [(0, 0, 1), (0, 1, 0), (0, 1, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]
    # the 7 level-2 cells of octant 0 besides the min corner's, then the 8 level-2 cells of octant 4 (x high)
    slots = [bmin + e2 * np.array(c) for c in cells] + [bmin + np.array([2 * e2, 0, 0]) + e2 * np.array(c) for c in [(0, 0, 0)] + cells]
    for c, lo in zip(counts, slots):
        rows.append(lo + e2 * (0.05 + 0.9 * rng.random((c, 3))))
    rows.append(bmin + np.array([0, 2 * e2, 0]) + e2 * (0.05 + 0.9 * rng.random((maxpts + 1, 3))))  # octant 2, one cell: splits
    P = np.concatenate(rows)
    return P[rng.permutation(len(P))]


CLOUDS = {"clean": cloud_clean, "degenerate": cloud_degenerate, "wild": cloud_wild, "tiles": cloud_tiles}


class Case:
    def __init__(self, name, box_name, profile, cloud, maxpts=200, n=20000, intensity=False, stride=1, seed=0):
        self.name, self.box_name, self.profile, self.cloud = name, box_name, profile, cloud
        self.maxpts, self.intensity, self.stride = maxpts, intensity, stride
        self.bmin, self.bmax, self.E, self.env = box(box_name)
        self.res = self.E * PROFILES[profile]
        self.mode = BOX_MODE[box_name]
        self.wide = profile == "wide"
        depth = 32 if self.wide else 22  # the last level of the profile
        rng = np.random.default_rng(seed)
        self.P = np.ascontiguousarray(CLOUDS[cloud](rng, self.bmin, self.E, depth, maxpts, n), np.float64)
        self.n = len(self.P)
        self.rgb = rng.integers(0, 256, self.n * 3, dtype=np.uint8)
        self.inten = None
        if intensity:
            self.inten = rng.random(self.n).astype(np.float32)
            self.inten[:: 97] = np.float32(np.nan)
            self.inten[1:: 97] = np.float32(-0.0)

    def __repr__(self):
        return self.name

    def level_table(self):
        """make_level_table of this case's root cube under its environment (the caller sets self.env)."""
        return level_table(self.E, self.res, self.bmin)

    def xyz(self):
        """(x, y, z, stride) as build_octree takes them: separate arrays, or views of one row-major array for stride 3."""
        if self.stride == 3:
            flat = self.P.reshape(-1)
            return flat[0:], flat[1:], flat[2:], 3
        return [np.ascontiguousarray(self.P[:, a]) for a in range(3)] + [1]

    def columns(self):
        return [np.ascontiguousarray(self.P[:, a]) for a in range(3)]


def _cases():
    out = []
    seed = 1
    for box_name in BOXES:
        for profile in PROFILES:
            for cloud in ("clean", "degenerate", "wild"):
                # intensity on / off and AoS input alternate over the cases
                out.append(Case("%s-%s-%s" % (box_name, profile, cloud), box_name, profile, cloud, intensity=seed % 2 == 0, stride=3 if seed % 3 == 0 else 1,
                                seed=seed))
                seed += 1
    for box_name, profile in (("zero", "narrow"), ("ones", "wide"), ("offset", "narrow"), ("pow2", "wide")):
        out.append(Case("%s-%s-tiles" % (box_name, profile), box_name, profile, "tiles", maxpts=2049, intensity=True, stride=3 if seed % 2 else 1, seed=seed))
        seed += 1
    return out


CASES = _cases()


class Bits:
    """A tree (or the oracle's, oracle=True) whose node_data returns intensities as f32 bit patterns, so that compare_trees tells
    NaN from NaN and -0.0 from 0.0 as the stored bytes do."""

    def __init__(self, t, oracle=False):
        self.t, self.oracle, self.nodes = t, oracle, t.nodes
        self.has_intensity = getattr(t, "has_intensity", False)

    def node_data(self, name, with_i=True):
        x, c, i, s = self.t.node_data(name, with_i) if self.oracle else self.t.node_data(name)
        return x, c, (i.view(np.uint32) if i is not None else None), s


# ---- restatements of the kernels' choices (csrc/kernels_build.cuh) ------------------------------------------------------
def schedule(last_level):
    """BuildPlan::run's pass schedule: (level, G, Gn) with two levels per pass, one when a single level is left."""
    s, L = [], 0
    while L < last_level:
        G = min(2, last_level - L)
        s.append([L, G])
        L += G
    return [(L, G, s[i + 1][1] if i + 1 < len(s) else 0) for i, (L, G) in enumerate(s)]


def pass_encoding(enc, L, G, Gn, wide, generic=False):
    """CudaBackend::partition_launch: the one encoding of every level a pass touches (level L+1, L+2 when G == 2, and the first
    level of the next pass), or -1 for mixed encodings, wide records, Float64 or PCV_PASS_GENERIC."""
    e = enc[L + 1]
    if G == 2 and enc[L + 2] != e:
        e = -1
    if Gn > 0 and enc[min(L + G + 1, 40)] != e:
        e = -1
    return -1 if wide or e == ENC_F64 or generic else e


def div_bad(a):
    """chain_device.cuh div_bad: a numerator outside div_known's proven range (|a| in [2^-500, 2^500) or exactly +0.0 pass)."""
    b = np.asarray(a, np.float64).view(np.uint64)
    hi = ((b >> np.uint64(32)) & np.uint64(0x7FFFFFFF)).astype(np.int64)
    inrange = ((hi - 0x20B00000) & 0xFFFFFFFF) < 0x3E800000
    return ~(inrange | (b == 0))


def first_step_numerators(P, bmin, E):
    """k_ingest's numerators q - m of the first step (the root cube's digit picks m = bmin or bmin + E / 2), per coordinate."""
    e1 = E / 2
    c = (bmin + (bmin + E)) * 0.5
    with np.errstate(invalid="ignore"):
        m = np.where(P > c, bmin + e1, bmin)
        return P - m, e1


def code_of(t, enc):
    """The stored code of a quotient t (encode_axis after the division)."""
    if enc in (ENC_U8, ENC_U16):
        M = 255.0 if enc == ENC_U8 else 65535.0
        if t != t or t <= 0.0:
            return 0
        return int(min(M * t, M)) if M * t < 4294967295.0 else int(M)
    c = t if t != t else min(max(t, 0.0), 1.0)
    if enc == ENC_F32:
        return int(np.float32(c).view(np.uint32))
    return int(np.float64(c).view(np.uint64))
