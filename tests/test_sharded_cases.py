"""The multi-rank cases of sharded_cases.py, on the CPU: from the test backend's level-k cell of every point and the planning
helpers of distributed.py, each case reaches what it claims - non-zero sender offsets, empty senders and owners, wide fan-out,
tile-edge ranges, the shard level it runs at, the slab lifecycle - and together the fused cases launch every remote partition
kernel variant the sharded level table can reach."""
import numpy as np
import pytest

import sharded_cases as S
from tb_api import level_table


@pytest.fixture(scope="module")
def plans():
    return {c.name: S.plan(c) for c in S.ALL}


def _table(case, monkeypatch):
    """make_level_table with the root cube, as pcv_shard_ingest_device calls it (the fused pass's kernels take its mode)."""
    for k in S.ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in case.env.items():
        monkeypatch.setenv(k, v)
    _, _, _, res, bmin, bmax = case.data()
    return level_table(float(np.max(bmax - bmin)), res, bmin)


def _wide(t):
    return any(e == 4 for e in t["enc"][1:t["last_level"] + 1])


@pytest.mark.parametrize("case", S.ALL, ids=str)
def test_case_is_well_formed(case, plans):
    p = plans[case.name]
    P = case.data()[0]
    assert len(P) <= 2_000_000 and case.R in (2, 3, 4, 8)
    assert case.ranges()[0][0] == 0 and case.ranges()[-1][1] == len(P)
    assert all(a[1] == b[0] for a, b in zip(case.ranges(), case.ranges()[1:]))
    assert int(p["H"].sum()) == len(P) and int(p["M"].sum()) == len(P)
    assert np.array_equal(p["M"].sum(1), [hi - lo for lo, hi in case.ranges()])
    assert 1 <= p["k"] <= case.k


def test_every_path_runs(plans):
    ran = set()
    for c in S.ALL:
        for path in c.paths:
            ran.add("records" if path == "fused" and plans[c.name]["k"] != 2 else path)
    assert ran == set(S.PATHS), ran
    v1 = [c for R, env in S.WORLD_ENV.items() if env.get("PCV_EXCHANGE_V1") for c in S.CASES[R] if "pyx" in c.paths]
    assert v1, "no k = 3 pack + exchange under PCV_EXCHANGE_V1"
    assert any("pyx" in c.paths for R in S.CASES if R not in S.WORLD_ENV for c in S.CASES[R]), "no k = 3 pack + exchange with the sorted kernel"


def test_offsets_are_nonzero_for_every_later_sender(plans):
    """pcv_shard_pass_device's `pre` (and step (3b)'s first[d]) of sender s for cell c is the count of c on the ranks below s: some fused
    case has it non-zero for every (s > 0, c) that s sends, so an offset summed over the wrong ranks moves every remote bucket."""
    hit = []
    for c in S.ALL:
        p = plans[c.name]
        if "fused" not in c.paths or p["k"] != 2:
            continue
        H = p["Hk"].astype(np.int64)
        pairs = [(s, cell) for s in range(1, c.R) for cell in range(H.shape[1]) if H[s, cell]]
        if pairs and all(H[:s, cell].sum() > 0 for s, cell in pairs):
            hit.append(c.name)
    print("\nnon-zero offsets for every later sender: %s" % hit)
    assert {int(name[1]) for name in hit} == set(S.CASES), hit  # on every world size


def test_empty_owners_and_senders_and_fan_out(plans):
    empty_owner = [c.name for c in S.ALL if len(set(plans[c.name]["c2r"][plans[c.name]["Hk"].sum(0) > 0])) < c.R]
    empty_sender = [c.name for c in S.ALL if any(hi == lo for lo, hi in c.ranges())]
    single_point = [c.name for c in S.ALL if any(hi - lo == 1 for lo, hi in c.ranges())]
    fan3 = [c.name for c in S.ALL if max(int((plans[c.name]["M"][s] > 0).sum()) for s in range(c.R)) >= 3]
    print("\nowner without cells: %s\nsender without points: %s\nsender with one point: %s\na sender to >= 3 owners: %s" % (empty_owner, empty_sender,
                                                                                                                          single_point, fan3))
    assert "r4-two-cells" in empty_owner and plans["r4-two-cells"]["k"] == 2
    assert empty_sender and single_point and fan3


def test_range_ends_on_tile_edges():
    sizes = [hi - lo for c in S.ALL for lo, hi in c.ranges()]
    for tile in (S.PACK_TILE, S.PASS_TILE):
        assert any(s and s % tile == 0 for s in sizes) and any(s > 1 and s % tile == 1 for s in sizes), tile


def test_prefix_depths(plans):
    """k = 2 on every world size, k = 1 on most; a cloud whose sparse octant drops the shard level from 2 to 1; k = 3 for the Python path."""
    ks = {(c.R, c.k, plans[c.name]["k"]) for c in S.ALL}
    assert all((R, 2, 2) in ks for R in S.CASES), ks
    assert len({R for R, _, k in ks if k == 1}) >= 3, ks
    assert plans["r3-sparse-octant"]["k"] == 1
    assert any(c.k == 3 and plans[c.name]["k"] == 3 for c in S.ALL)


def test_record_width_intensity_and_modes(plans, monkeypatch):
    seen = set()
    for c in S.ALL:
        t = _table(c, monkeypatch)
        seen.add((_wide(t), c.intensity))
        if "/" in c.cloud:
            box_name = c.cloud.split("/")[0]
            assert t["fast"] == S.B.BOX_MODE[box_name], (c, t["fast"])
    assert seen == {(w, i) for w in (False, True) for i in (False, True)}, seen
    boxes = {c.cloud.split("/")[0] for c in S.ALL if "/" in c.cloud}
    assert {S.B.BOX_MODE[b] for b in boxes} == {0, 1, 2, 3}
    assert {c.cloud.split("/")[2] for c in S.ALL if "/" in c.cloud} == {"degenerate", "wild"}


def _need(case, plan):
    return int(plan["M"].sum(0).max())


def _cap(need):
    return ((int(need * 1.05) + 4096 + 4095) // 4096) * 4096  # slab_for (csrc/sharded_build.inl)


def test_slab_lifecycle(plans, monkeypatch):
    """The native builds of one world run on one context per node size, in order: some build regrows the slab, some wide build
    follows a narrow one and a narrow one a wide one, some build with intensity follows one without, and after an explicit release
    one more build runs."""
    regrow = narrow_after_wide = int_after_none = after_release = False
    for R, cases in S.CASES.items():
        last = {}  # per node size: (cap, wide, intensity) of the slab the previous native build left
        for c in cases:
            if not {"fused", "records"} & set(c.paths):
                continue
            wide, need = _wide(_table(c, monkeypatch)), _need(c, plans[c.name])
            prev = last.get(c.maxpts)
            if c.release_before:
                assert prev is not None
                after_release = True
            elif prev is not None:
                regrow |= prev[1] == wide and prev[2] == c.intensity and need > prev[0]
                narrow_after_wide |= prev[1] and not wide
                int_after_none |= c.intensity and not prev[2]
            keep = prev is not None and not c.release_before and prev[0] >= need and prev[1] == wide and prev[2] == c.intensity
            last[c.maxpts] = prev if keep else (_cap(need), wide, c.intensity)
    assert regrow and narrow_after_wide and int_after_none and after_release, (regrow, narrow_after_wide, int_after_none, after_release)


def test_coverage_of_every_remote_pass_variant(plans, monkeypatch):
    """k_pass<WIDE, true, FAST, -1>: the fused exchange pass of every sender with points, in the division mode of the level table
    pcv_shard_ingest_device makes (with the root cube, so mode 2 boxes stay in mode 2), against every variant pass_kernel can pick."""
    reached = set()
    for c in S.ALL:
        p = plans[c.name]
        if "fused" not in c.paths or p["k"] != 2:
            continue
        t = _table(c, monkeypatch)
        if t["last_level"] >= 2 and any(hi > lo for lo, hi in c.ranges()):
            reached.add(("k_pass", _wide(t), True, t["fast"], -1))
    want = {("k_pass", w, True, f, -1) for w in (False, True) for f in range(4)}
    print("\nremote k_pass variants reached (%d):\n  %s" % (len(reached), "\n  ".join(map(str, sorted(reached)))))
    assert reached == want, ("missing", sorted(want - reached), "unexpected", sorted(reached - want))
