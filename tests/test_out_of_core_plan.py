"""Out-of-core build: the group planner (csrc/ooc_plan.h, compiled here with g++) against a Python restatement
(distributed.usable_prefix_levels + greedy grouping of consecutive level-k cells), and the pcv_ooc_info layout.  No GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <iostream>
#include "ooc_plan.h"
int main() {
    int K; double E, res; unsigned long long maxp, budget;
    std::cin >> K >> E >> res >> maxp >> budget;
    std::vector<uint64_t> c((size_t)1 << (3 * K));
    for (auto& v : c) { unsigned long long t; std::cin >> t; v = t; }
    const pcv::OocPlan p = pcv::plan_ooc_groups(c, K, E, res, maxp, budget);
    std::cout << p.k << "\n";
    if (!p.error.empty()) { std::cout << "ERROR " << p.error << "\n"; return 0; }
    for (size_t g = 0; g < p.group_points.size(); ++g) std::cout << p.group_first[g] << " " << p.group_first[g + 1] << " " << p.group_points[g] << "\n";
    return 0;
}
"""


@pytest.fixture(scope="module")
def planner(tmp_path_factory):
    d = tmp_path_factory.mktemp("ooc_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])

    def run(counts, K, E, res, maxp, budget):
        inp = "%d %r %r %d %d\n%s\n" % (K, float(E), float(res), maxp, budget, " ".join(str(int(v)) for v in counts))
        out = subprocess.check_output([exe], input=inp, text=True).splitlines()
        k = int(out[0])
        if len(out) > 1 and out[1].startswith("ERROR "):
            return k, None, out[1][6:]
        return k, [tuple(int(t) for t in l.split()) for l in out[1:]], None

    return run


def restated(counts, K, E, res, maxp, budget):
    from point_cloud_viewer_b200 import distributed as D

    k = D.usable_prefix_levels(np.asarray(counts, np.uint64), K, E, res, maxp)
    ck = np.asarray(counts, np.uint64).reshape(8 ** k, -1).sum(1)
    groups = []  # [first cell, end cell, points]: runs of consecutive non-empty cells filled greedily up to the budget
    for cell, v in enumerate(ck.tolist()):
        if v == 0:
            continue
        if v > budget:
            return k, None, "r" + "".join(str((cell >> (3 * i)) & 7) for i in range(k - 1, -1, -1)), v
        if not groups or groups[-1][2] + v > budget:
            groups.append([cell, None, 0])
        groups[-1][2] += v
    for g in range(len(groups)):
        groups[g][1] = groups[g + 1][0] if g + 1 < len(groups) else 8 ** k
    return k, [tuple(g) for g in groups], None, None


@pytest.mark.parametrize("seed", range(12))
def test_planner_matches_python_restatement(planner, seed):
    rng = np.random.default_rng(seed)
    K = 3
    counts = rng.integers(0, 5000, 512) * (rng.random(512) < 0.6)
    if seed % 3 == 1:  # one sparse octant: its level-1 node is a leaf, so k drops
        counts.reshape(8, 64)[5] = 0
        counts[5 * 64 + 7] = 3
    if seed % 4 == 2:  # a sparse level-2 cell: k = 2
        counts.reshape(64, 8)[9] = 0
        counts[9 * 8 + 1] = 2
    maxp = int(rng.choice([50, 2000, 10 ** 9]))
    E, res = 1024.0, float(rng.choice([0.001, 1.0, 200.0]))
    biggest = int(counts.reshape(8 ** 1, -1).sum(1).max())
    for budget in (int(counts.sum()), int(counts.sum()) // 3 + 1, 5000, biggest + 1, 1):
        k, groups, err = planner(counts, K, E, res, maxp, budget)
        rk, rgroups, rcell, rcount = restated(counts, K, E, res, maxp, budget)
        assert k == rk
        if rgroups is None:
            assert err is not None and rcell in err and str(rcount) in err and str(budget) in err, err
            if k < K:
                assert "leaf" in err
        else:
            assert err is None, err
            assert groups == rgroups
            assert sum(g[2] for g in groups) == int(counts.sum())
            assert all(g[2] <= budget for g in groups)


def test_planner_k_selection_and_cell_message(planner):
    counts = np.zeros(512, np.int64)
    counts[0o000] = counts[0o777] = 900  # every level-1 and level-2 node with points has more than 100 -> k = 3
    k, groups, err = planner(counts, 3, 8.0, 0.001, 100, 1000)
    assert (k, err) == (3, None) and groups == [(0, 511, 900), (511, 512, 900)]
    counts[0o400] = 5  # a lone point group in octant 4: that level-1 node is a leaf, k = 1
    k, groups, err = planner(counts, 3, 8.0, 0.001, 100, 1000)
    assert (k, err) == (1, None) and groups == [(0, 7, 905), (7, 8, 900)]
    k, groups, err = planner(counts, 3, 8.0, 0.001, 100, 899)
    assert k == 1 and groups is None and "r0 holds 900 points, more than the 899 points" in err and "leaf" in err
    k, groups, err = planner(counts, 3, 8.0, 0.001, 100, 10 ** 6)
    assert k == 1 and groups == [(0, 8, 1805)]
    # edge <= resolution above level k stops the descent as well (generation.rs:128-150)
    counts[0o400] = 0
    k, _, _ = planner(counts, 3, 8.0, 4.0, 100, 10 ** 6)
    assert k == 1
    k, _, _ = planner(counts, 3, 8.0, 2.0, 100, 10 ** 6)
    assert k == 2


def test_ooc_info_struct_matches_the_c_compiler(tmp_path):
    """pcv_ooc_info: ctypes size and field offsets equal gcc's for include/pcv.h."""
    from point_cloud_viewer_b200 import _native as N

    fs = [f for f, _ in N.OocInfo._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "pcv.h"', "int main(void) {", 'printf("size %zu\\n", sizeof(pcv_ooc_info));']
    for f in fs:
        src.append('printf("%s %%zu\\n", offsetof(pcv_ooc_info, %s));' % (f, f))
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, str(c)])
    got = dict(l.split() for l in subprocess.check_output([exe], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(N.OocInfo)
    for f in fs:
        assert int(got[f]) == getattr(N.OocInfo, f).offset, f
