"""A high-precision reference of the S2 leaf cell of a point, independent of csrc/s2.h and oracle/oracle_s2.hpp.

The face comes from exact comparisons of the double components (largest absolute component, ties to the later axis, the
negative face for a negative component).  (u, v) are the exact ratios of the components as 50-digit decimals (a normalisation
would cancel in them), st is the quadratic projection with Decimal.sqrt, and (i, j) = floor(2^30 st) clamped to [0, 2^30 - 1].
A vectorised walk of the published posToIJ / posToOrientation tables turns (face, i, j) into the leaf id.

Where the exact st lies within TIE_ST of a level-30 boundary on either axis, the double pipeline of the libraries may round to
the neighbouring leaf (or face): such points are flagged as ties, and only bit parity with the libraries' arithmetic is the
contract there."""
from decimal import Decimal, ROUND_FLOOR, localcontext

import numpy as np

MAX_LEVEL = 30
TIE_ST = Decimal(2) ** -45  # far above the double pipeline's error on st, far below one leaf (2^-30)

# The published Hilbert curve tables: posToIJ[orientation][pos] = (i bit << 1) | j bit; swapMask = 1, invertMask = 2.
POS_TO_IJ = np.array([[0, 1, 3, 2], [0, 2, 3, 1], [3, 2, 0, 1], [3, 1, 0, 2]], np.int64)
POS_TO_ORIENTATION = np.array([1, 0, 0, 3], np.int64)
IJ_TO_POS = np.argsort(POS_TO_IJ, axis=1).astype(np.int64)  # the inverse permutation of every row


def _face(x, y, z):
    ax, ay, az = abs(x), abs(y), abs(z)
    if ax > ay:
        axis = 0 if ax > az else 2
    else:
        axis = 1 if ay > az else 2
    c = (x, y, z)[axis]
    return axis + 3 if c < 0.0 else axis


def _uv(face, x, y, z):
    X, Y, Z = Decimal(x), Decimal(y), Decimal(z)  # exact: every double is a Decimal
    if face == 0:
        return Y / X, Z / X
    if face == 1:
        return -X / Y, Z / Y
    if face == 2:
        return -X / Z, -Y / Z
    if face == 3:
        return Z / X, Y / X
    if face == 4:
        return Z / Y, -X / Y
    return -Y / Z, -X / Z


_HALF, _ONE, _THREE, _SCALE = Decimal("0.5"), Decimal(1), Decimal(3), Decimal(1 << MAX_LEVEL)
_TIE = TIE_ST * _SCALE


def _ij(u):
    """(floor(2^30 st) clamped, whether st is within TIE_ST of a multiple of 2^-30)."""
    st = _HALF * (_ONE + _THREE * u).sqrt() if u >= 0 else _ONE - _HALF * (_ONE - _THREE * u).sqrt()
    scaled = st * _SCALE
    f = scaled.to_integral_value(rounding=ROUND_FLOOR)
    tie = scaled - f < _TIE or (f + 1) - scaled < _TIE
    return min(max(int(f), 0), (1 << MAX_LEVEL) - 1), tie


def face_ij(P):
    """(face, i, j, tie) of every row of P (n, 3): exact arithmetic at 50 significant digits."""
    P = np.asarray(P, np.float64).reshape(-1, 3)
    n = len(P)
    face, i, j = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(n, np.int64)
    tie = np.zeros(n, bool)
    with localcontext() as ctx:
        ctx.prec = 50
        for k, (x, y, z) in enumerate(P.tolist()):
            f = _face(x, y, z)
            u, v = _uv(f, x, y, z)
            i[k], ti = _ij(u)
            j[k], tj = _ij(v)
            face[k], tie[k] = f, ti or tj
    return face, i, j, tie


def from_face_ij(face, i, j):
    """The leaf cell ids of (face, i, j): the Hilbert curve walked from the top, starting in orientation face & swapMask."""
    face, i, j = (np.asarray(a, np.int64) for a in (face, i, j))
    orientation = face & 1
    pos = np.zeros(len(face), np.uint64)
    for k in range(MAX_LEVEL - 1, -1, -1):
        ij = (((i >> k) & 1) << 1) | ((j >> k) & 1)
        p = IJ_TO_POS[orientation, ij]
        pos |= p.astype(np.uint64) << np.uint64(2 * k)
        orientation = orientation ^ POS_TO_ORIENTATION[p]
    return (face.astype(np.uint64) << np.uint64(61)) | (pos << np.uint64(1)) | np.uint64(1)


def parent(ids, level):
    """CellID::parent(level) of leaf (or finer) ids."""
    lsb = np.uint64(1) << np.uint64(2 * (MAX_LEVEL - level))
    return (np.asarray(ids, np.uint64) & ~(lsb - np.uint64(1))) | lsb


def cell_ids(P, level=MAX_LEVEL):
    """(cell ids at `level`, tie mask) of every row of P."""
    face, i, j, tie = face_ij(P)
    return parent(from_face_ij(face, i, j), level), tie
