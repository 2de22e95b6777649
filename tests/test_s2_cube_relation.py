"""The node test of the octree's cell-union query (csrc/s2.h: s2_to_face_ij_level, s2_cube_relation), through the TEST-ONLY
sequential drivers (tests/cpu_backend/s2_cube_cpu.cpp, built into _build/libtbc.so).  Soundness is checked against the
oracle's independent from_point (oracle/oracle_s2.hpp): a cube classified Out holds no point whose leaf cell is in the union,
and a cube classified In holds only such points."""
import ctypes as C
import os

import numpy as np
import pytest

import s2_api as S

IN, CROSS, OUT = 0, 1, 2
R = 6371000.0

_SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpu_backend", "_build", "libtbc.so")
_tbc = None


def _tb():
    global _tbc
    if _tbc is None:
        L = C.CDLL(_SO)
        L.tbc_to_face_ij_level.argtypes = [C.c_uint64, C.POINTER(C.c_int32)] + [C.POINTER(C.c_uint32)] * 3
        L.tbc_cube_relation.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
        _tbc = L
    return _tbc


def face_ij_level(cid):
    f, i, j, s = C.c_int32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    _tb().tbc_to_face_ij_level(int(cid), C.byref(f), C.byref(i), C.byref(j), C.byref(s))
    return f.value, i.value, j.value, s.value


def relation(cu, m, e):
    cu = np.ascontiguousarray(cu, np.uint64)
    m = np.ascontiguousarray(np.atleast_2d(m), np.float64)
    e = np.ascontiguousarray(np.atleast_1d(e), np.float64)
    out = np.zeros(len(e), np.int32)
    _tb().tbc_cube_relation(cu.ctypes.data, len(cu), m.ctypes.data, e.ctypes.data, len(e), out.ctypes.data)
    return out


def parent(cid, level):
    return int(S.orc().orc_s2_parent(int(cid), level))


def in_union(cu, P):
    """The reference's point test, CellUnion::contains(CellID::from_point(p)), entirely in the oracle."""
    leaves = S.oracle_cell_ids(P, 30)
    contains, _ = S.union_test(cu, leaves)
    return contains


# ---- round trip --------------------------------------------------------------------------------------------------------------
def test_round_trip_every_level():
    rng = np.random.default_rng(5)
    edge = [0, 1, 2, (1 << 30) - 2, (1 << 30) - 1, 1 << 29, (1 << 29) - 1]
    cases = [(f, i, j) for f in range(6) for i in edge for j in edge]
    cases += [(int(rng.integers(6)), int(rng.integers(1 << 30)), int(rng.integers(1 << 30))) for _ in range(300)]
    for f, i, j in cases:
        leaf = int(S.tb().tbs_from_face_ij(f, i, j))
        assert leaf == int(S.orc().orc_s2_from_face_ij(f, i, j))
        for level in range(31):
            cid = parent(leaf, level) if level < 30 else leaf
            size = 1 << (30 - level)
            assert face_ij_level(cid) == (f, i & ~(size - 1), j & ~(size - 1), size), (f, i, j, level)


# ---- soundness fuzz ----------------------------------------------------------------------------------------------------------
def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


def _cube_points(m, e, rng, k=600):
    """Corners, edge and face points, the interior, and nextafter neighbours, all inside [m, m + e]."""
    hi = m + e
    ts = [np.array([(c >> a) & 1 for a in range(3)], np.float64) for c in range(8)]
    grid = np.linspace(0.0, 1.0, 5)
    ts += [np.array([a, b, c]) for a in grid for b in grid for c in (0.0, 1.0)]
    ts += [np.array([a, c, b]) for a in grid for b in grid for c in (0.0, 1.0)]
    T = np.concatenate([np.array(ts), rng.random((k, 3))])
    P = m + T * e
    P = np.concatenate([P, np.nextafter(P, np.inf), np.nextafter(P, -np.inf)])
    return np.clip(P, m, hi)


def _union_for(m, e, rng, P):
    """Mixed levels 0-30: cells of points inside the cube, their neighbours along the curve, and random cells."""
    ids = []
    leaves = S.oracle_cell_ids(P[rng.integers(len(P), size=6)], 30)
    for leaf in leaves:
        level = int(rng.integers(0, 31))
        cid = parent(int(leaf), level) if level < 30 else int(leaf)
        ids.append(cid)
        if rng.random() < 0.5:
            ids.append(int(S.orc().orc_s2_next(cid)))
    for _ in range(int(rng.integers(0, 4))):
        leaf = int(S.oracle_cell_ids(_unit(rng.normal(size=3))[None, :] * R, 30)[0])
        level = int(rng.integers(0, 31))
        ids.append(parent(leaf, level) if level < 30 else leaf)
    return S.normalize(np.array(ids, np.uint64))


def _check(m, e, cu, rng):
    m = np.asarray(m, np.float64)
    P = _cube_points(m, e, rng)
    inside = in_union(cu, P)
    rel = int(relation(cu, m, e)[0])
    if inside.any():
        assert rel != OUT, (m.tolist(), e, cu.tolist())
    if rel == IN:
        assert inside.all(), (m.tolist(), e, cu.tolist())
    return rel


def _cube_families(rng):
    """(min corner, edge) of ECEF slabs, cubes across a face edge or a face corner, cubes holding the origin, tiny cubes and
    level-20 node cubes."""
    out = []
    for _ in range(6):
        e = float(10.0 ** rng.uniform(0, 5))
        out.append((_unit(rng.normal(size=3)) * R - e / 2, e))
    for _ in range(4):
        a, b = rng.choice(3, 2, replace=False)
        d = np.zeros(3)
        d[a], d[b] = rng.choice([-1, 1]), rng.choice([-1, 1])
        d[3 - a - b] = rng.uniform(-0.5, 0.5)
        e = float(10.0 ** rng.uniform(-2, 4))
        out.append((_unit(d) * R - e * rng.uniform(0.2, 0.8, 3), e))
    for _ in range(4):
        d = rng.choice([-1.0, 1.0], 3)
        e = float(10.0 ** rng.uniform(-2, 4))
        out.append((_unit(d) * R - e * rng.uniform(0.2, 0.8, 3), e))
    for _ in range(2):
        e = float(10.0 ** rng.uniform(-3, 7))
        out.append((-e * rng.uniform(0.1, 0.9, 3), e))
    for _ in range(3):
        e = float(10.0 ** rng.uniform(-9, -3))
        out.append((_unit(rng.normal(size=3)) * R, e))
    for _ in range(3):
        root = float(2.0 ** rng.integers(14, 24))
        e = root / 2 ** 20
        c = _unit(rng.normal(size=3)) * R
        out.append((np.floor(c / e) * e, e))
    return out


@pytest.mark.parametrize("seed", range(6))
def test_soundness_fuzz(seed):
    rng = np.random.default_rng(1000 + seed)
    seen = set()
    for m, e in _cube_families(rng):
        P = _cube_points(np.asarray(m, np.float64), e, rng, k=200)
        seen.add(_check(m, e, _union_for(m, e, rng, P), rng))
    assert OUT in seen or CROSS in seen


def test_soundness_hypothesis():
    hyp = pytest.importorskip("hypothesis")
    st = pytest.importorskip("hypothesis.strategies")

    @hyp.settings(max_examples=80, deadline=None, derandomize=True, suppress_health_check=list(hyp.HealthCheck))
    @hyp.given(
        st.tuples(*[st.floats(-1.0, 1.0, allow_nan=False)] * 3),
        st.sampled_from([0.0, 1.0, R]),
        st.floats(-9.0, 6.0),
        st.integers(0, 2 ** 32 - 1),
    )
    def run(d, scale, log_e, seed):
        rng = np.random.default_rng(seed)
        e = float(10.0 ** log_e)
        m = np.asarray(d, np.float64) * scale - e * rng.uniform(0.0, 1.0, 3)
        P = _cube_points(m, e, rng, k=150)
        _check(m, e, _union_for(m, e, rng, P), rng)

    run()


# ---- pins --------------------------------------------------------------------------------------------------------------------
def test_far_side_is_out():
    c = np.array([4157222.543, 664789.307, 4774952.099])
    cu = S.oracle_cell_ids(c[None, :], 20)
    e = 1000.0
    assert relation(cu, -c - e / 2, e)[0] == OUT
    assert relation(np.zeros(0, np.uint64), c - e / 2, e)[0] == OUT  # the empty union


def test_node_inside_a_level_10_cell_is_in():
    c = np.array([4157222.543, 664789.307, 4774952.099])
    cell = S.oracle_cell_ids(c[None, :], 10)
    leaf = int(S.oracle_cell_ids(c[None, :], 30)[0])
    assert parent(leaf, 10) == int(cell[0])
    # a level-10 cell is ~10 km across; a 1 m node cube around its centre lies well inside it
    ctr = S.centre(int(cell[0])) * R
    assert relation(cell, ctr - 0.5, 1.0)[0] == IN
    assert relation(cell, np.full(3, -0.5), 1.0)[0] == CROSS  # a cube holding the origin


def test_whole_face_and_neighbour_face():
    c = np.array([4157222.543, 664789.307, 4774952.099])
    f, _, _ = S.face_ij(int(S.oracle_cell_ids(c[None, :], 30)[0]))
    face = np.array([(f << 61) | (1 << 60)], np.uint64)  # the level-0 cell of face f
    assert relation(face, c - 50.0, 100.0)[0] == IN
    other = np.array([(((f + 3) % 6) << 61) | (1 << 60)], np.uint64)  # the opposite face
    assert relation(other, c - 50.0, 100.0)[0] == OUT
