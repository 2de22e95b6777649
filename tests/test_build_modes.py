"""The build-mode cases of build_modes.py, on the CPU: each reaches the division mode, record width and encodings it claims
(per make_level_table), together they reach every kernel variant the build can launch, mode 1's range check really fires
(and on numerators where skipping the IEEE repeat would change a stored code), and the test backend's tree equals the
oracle's for every case."""
import numpy as np
import pytest

import build_modes as B
import oracle_api as O
from parity import compare_trees
from tb_api import TbTree, div_unguarded


@pytest.fixture(scope="module")
def oracles():
    """Oracle tree per case (built once for the module)."""
    return {c.name: O.build(*c.columns(), c.rgb.reshape(-1, 3), c.res, c.bmin, c.bmax, intensity=c.inten, max_points_per_node=c.maxpts) for c in B.CASES}


def _table(case, monkeypatch):
    for k in ("PCV_CHECKED_FAST", "PCV_NO_POW2"):
        monkeypatch.delenv(k, raising=False)
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)
    return case.level_table()


def _levels(ref):
    """Levels of the oracle tree's split nodes, and its non-root leaves that keep points: (level, num_points)."""
    names = set(ref.nodes)
    split = {len(nm) - 1 for nm in names if any(nm + str(d) in names for d in range(8))}
    leaves = [(len(nm) - 1, m["num_points"]) for nm, m in ref.nodes.items() if len(nm) > 1 and not any(nm + str(d) in names for d in range(8))]
    return split, leaves


@pytest.mark.parametrize("case", B.CASES, ids=str)
def test_case_reaches_its_mode_width_and_encodings(case, monkeypatch):
    t = _table(case, monkeypatch)
    assert t["fast"] == case.mode, (case, t["fast"])
    assert any(e == B.ENC_F64 for e in t["enc"][1:t["last_level"] + 1]) == case.wide
    assert t["last_level"] == (32 if case.wide else 22)
    used = {t["enc"][L] for L in range(1, t["last_level"] + 1)}
    assert used == ({B.ENC_U8, B.ENC_U16, B.ENC_F32} | ({B.ENC_F64} if case.wide else set())), used
    if case.mode == 0:
        assert not float(case.E).hex().startswith("0x1.0p") and float(case.E).hex().endswith("fffffffffffffp+9")
    # without the root cube (the sharded and out-of-core prefix histograms) no box is in mode 2
    assert B.level_table(case.E, case.res)["fast"] == (1 if case.mode == 2 else case.mode)


def test_coverage_of_every_kernel_variant(oracles, monkeypatch):
    """k_ingest<WIDE, FAST>, k_pass<WIDE, local, FAST, ENCU> and place_stayers<WIDE, ENC, FAST>: the variants the cases launch with
    work to do, against every variant the build instantiates."""
    reached = set()
    for case in B.CASES:
        t = _table(case, monkeypatch)
        split, leaves = _levels(oracles[case.name])
        reached.add(("k_ingest", case.wide, t["fast"]))
        for L, G, Gn in B.schedule(t["last_level"]):
            if L in split:  # the pass has active nodes
                reached.add(("k_pass", case.wide, t["fast"], B.pass_encoding(t["enc"], L, G, Gn, case.wide)))
        for L, npts in leaves:
            if npts:  # a non-root leaf with points keeps 7 of every 8 in place
                reached.add(("place_stayers", case.wide, t["enc"][L], t["fast"]))
    want = {("k_ingest", w, f) for w in (False, True) for f in range(4)}
    want |= {("k_pass", False, f, e) for f in range(4) for e in (B.ENC_U8, B.ENC_U16, B.ENC_F32, -1)} | {("k_pass", True, f, -1) for f in range(4)}
    want |= {("place_stayers", False, e, f) for e in (B.ENC_U8, B.ENC_U16, B.ENC_F32) for f in range(4)}
    want |= {("place_stayers", True, e, f) for e in (B.ENC_U8, B.ENC_U16, B.ENC_F32, B.ENC_F64) for f in range(4)}
    print("\nreached %d kernel variants:\n  %s" % (len(reached), "\n  ".join(map(str, sorted(reached, key=str)))))
    assert reached == want, ("missing", sorted(want - reached, key=str), "unexpected", sorted(reached - want, key=str))
    assert len({v for v in want if v[0] == "k_pass"}) == 20 and len({v for v in want if v[0] == "k_ingest"}) == 8


def _differs(u, v, enc):
    return B.code_of(u, enc) != B.code_of(v, enc)


def test_mode1_flag_fires_in_ingest_and_the_repeat_matters(monkeypatch):
    """k_ingest in mode 1: some first-step numerator fails div_bad, and for some of those the unguarded Markstein quotient gives
    another level-1 code than the IEEE quotient - without the IEEE repeat the build would store a different tree."""
    flagged = changed = 0
    for case in B.CASES:
        if case.mode != 1:
            continue
        t = _table(case, monkeypatch)
        a, e1 = B.first_step_numerators(case.P, case.bmin, case.E)
        bad = B.div_bad(a)
        flagged += int(bad.sum())
        ry = 1.0 / e1
        for v in np.unique(a[bad]):
            with np.errstate(all="ignore"):
                changed += _differs(div_unguarded(v, e1, ry), v / e1, t["enc"][1])
    assert flagged > 0 and changed > 0, (flagged, changed)


def _f64_nodes(ref):
    """(level, cube min, edge, codes (n, 3) float64) of every Float64 node below the root that holds points."""
    for nm, m in ref.nodes.items():
        if len(nm) > 1 and m["enc"] == B.ENC_F64 and m["num_points"]:
            yield len(nm) - 1, np.array(m["cube"][:3]), m["cube"][3], ref.node_data(nm)[0].view(np.float64).reshape(-1, 3)


def test_mode1_flag_fires_in_the_pass_and_place_kernels(oracles, monkeypatch):
    """Below the root only a Float64 level can carry a numerator outside the proven range: an oracle Float64 node holds a non-zero
    code t with t * e < 2^-500, so the pass that decodes it and the placement that rewrites it see a flagged numerator.  Where the
    node's min is 0 on that axis the decoded coordinate is t * e itself; some of those divide differently without the guard."""
    tiny, changed = 0, 0
    for case in B.CASES:
        if case.mode != 1 or not case.wide:
            continue
        _table(case, monkeypatch)
        for L, m, e, t in _f64_nodes(oracles[case.name]):
            with np.errstate(all="ignore"):
                sel = (t != 0) & (t * e < 2.0 ** -500)
            tiny += int(sel.sum())
            for a in range(3):
                if m[a] != 0.0:
                    continue
                for q in np.unique((t[:, a] * e)[sel[:, a]]):
                    for d in (e, e / 2, e / 4):  # the node's own cube (placement) and its children's (the pass)
                        changed += _differs(div_unguarded(q, d, 1.0 / d), q / d, B.ENC_F64)
    assert tiny > 0 and changed > 0, (tiny, changed)


@pytest.mark.parametrize("case", B.CASES, ids=str)
def test_test_backend_equals_oracle(case, oracles, monkeypatch):
    _table(case, monkeypatch)
    x, y, z, stride = case.xyz()
    tree = TbTree(x, y, z, case.rgb, case.res, case.bmin, case.bmax, case.maxpts, 2, intensity=case.inten, stride=stride)
    compare_trees(B.Bits(oracles[case.name], oracle=True), B.Bits(tree))
