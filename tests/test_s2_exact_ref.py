"""The exact S2 leaf-cell reference (tests/s2_exact.py) against the oracle's restatement of the libraries' double arithmetic on
every edge fixture (tests/s2_edges.py), without a GPU: equal wherever the exact st lies more than 2^-45 from a level-30 boundary;
the boundary fixture must keep producing such ties, where only the product's host build of csrc/s2.h is held to the oracle."""
import numpy as np
import pytest

import s2_api as S
import s2_edges as E
import s2_exact as X

# rows of each fixture the reference walks (about 200k points of Python arithmetic in all)
SUBSAMPLE = dict(corners=slice(None, None, 8), edges=slice(None, None, 6), globe=slice(0, 80_000), boundaries=slice(None), heavy=slice(None))


@pytest.fixture(scope="module")
def fixtures():
    return E.all_fixtures()


def test_fixture_points_are_valid_ecef(fixtures):
    for name, P in fixtures.items():
        r = np.sqrt(P[:, 0] * P[:, 0] + P[:, 1] * P[:, 1] + P[:, 2] * P[:, 2])  # the split's radius test, x, y, z order
        assert ((r >= E.R_MIN) & (r <= E.R_MAX)).all(), name
        _, valid = S.product_cell_ids(P[:1000], 30)
        assert valid.all(), name
    assert len(fixtures["corners"]) == 8 * 40_000 and len(fixtures["edges"]) == 12 * 20_000 and len(fixtures["globe"]) == 1_000_000


def test_tables_and_known_cells():
    assert all(X.POS_TO_IJ[o][X.IJ_TO_POS[o][ij]] == ij for o in range(4) for ij in range(4))
    axes = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [-1, 0, 0], [0, -1, 0], [0, 0, -1]], float) * E.R
    ids, tie = X.cell_ids(axes, 0)
    assert [int(v) for v in ids] == [(f << 61) | (1 << 60) for f in range(6)]
    assert tie.all()  # a face centre is the corner of four level-1 cells
    assert int(X.cell_ids(axes[:1])[0][0]) == 0x1000000000000001
    rng = np.random.default_rng(5)
    f = rng.integers(0, 6, 3000)
    i, j = rng.integers(0, 1 << 30, 3000), rng.integers(0, 1 << 30, 3000)
    got = X.from_face_ij(f, i, j)
    assert [int(v) for v in got] == [S.orc().orc_s2_from_face_ij(int(a), int(b), int(c)) for a, b, c in zip(f, i, j)]


def test_corner_and_edge_patches_span_faces(fixtures):
    faces = S.oracle_cell_ids(fixtures["corners"], 0) >> np.uint64(61)
    for k, d in enumerate(E.corner_directions()):
        want = sorted(a if d[a] > 0 else a + 3 for a in range(3))
        assert sorted(np.unique(faces[k * 40_000:(k + 1) * 40_000]).tolist()) == want
    faces = S.oracle_cell_ids(fixtures["edges"], 0) >> np.uint64(61)
    for k, d in enumerate(E.edge_directions()):
        want = sorted(a if d[a] > 0 else a + 3 for a in range(3) if d[a] != 0)
        assert sorted(np.unique(faces[k * 20_000:(k + 1) * 20_000]).tolist()) == want
    assert len(np.unique(S.oracle_cell_ids(fixtures["globe"], 0))) == 6


@pytest.mark.parametrize("name", list(SUBSAMPLE))
def test_reference_equals_oracle_away_from_ties(fixtures, name):
    P = fixtures[name][SUBSAMPLE[name]]
    leaf, tie = X.cell_ids(P)
    for level in (30, 29, 15, 1, 0):
        want = S.oracle_cell_ids(P, level)
        assert np.array_equal(X.parent(leaf, level)[~tie], want[~tie]), level
    if name == "boundaries":
        # the fixture sits on boundaries: most points are ties, on every level's corners, and the product's host build of
        # csrc/s2.h equals the oracle on all of them (the GPU suite holds the device build to the same)
        assert tie.sum() > 0.9 * len(P) and (~tie).sum() > 0
        per_level = 400 * len(E.BOUNDARY_LEVELS)
        assert tie[:per_level].sum() > 0.99 * per_level
        differ = leaf[tie] != S.oracle_cell_ids(P, 30)[tie]
        assert 0 < differ.sum() < tie.sum()  # the exact answer may legitimately differ on a tie, but not on every one
    else:
        assert tie.sum() <= max(5, len(P) // 1000), tie.sum()
    for level in (30, 0):
        got, valid = S.product_cell_ids(P, level)
        assert valid.all() and np.array_equal(got, S.oracle_cell_ids(P, level)), level
