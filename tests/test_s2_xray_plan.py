"""The S2 cloud's X-ray planning (csrc/xray_plan.h s2_xray_plan, s2_xray_fixed_bytes; compiled here with g++) against a Python
restatement, and key batches cut from exact per-leaf key counts (leaves no point is drawn into count zero keys).  No GPU."""
import os
import subprocess

import numpy as np
import pytest

from test_xray_bounded_plan import batches_py, block_bytes, depth_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <iostream>
#include "xray_plan.h"
int main() {
    std::string what;
    std::cin >> what;
    if (what == "plan") {
        unsigned long long budget, fixed, leaf, tile, slice; int depth, maxg;
        std::cin >> budget >> fixed >> depth >> maxg >> leaf >> tile >> slice;
        const pcv::XrayPlan p = pcv::s2_xray_plan(budget, fixed, depth, maxg, leaf, tile, slice);
        std::cout << p.g << " " << p.key_cap << " " << p.attr_leaves << " " << p.max_loc << " " << p.sel_cap << "\n";
    } else if (what == "fixed") {
        unsigned long long nc, nt; unsigned nf;
        std::cin >> nc >> nt >> nf;
        std::cout << pcv::s2_xray_fixed_bytes(nc, nt, nf) << "\n";
    } else {
        size_t n; unsigned long long cap;
        std::cin >> n >> cap;
        std::vector<uint64_t> k(n);
        for (auto& v : k) { unsigned long long t; std::cin >> t; v = t; }
        int64_t big = -1;
        const std::vector<uint32_t> s = pcv::xray_key_batches(k, cap, &big);
        std::cout << big;
        for (uint32_t v : s) std::cout << " " << v;
        std::cout << "\n";
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    d = tmp_path_factory.mktemp("s2_xray_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: subprocess.check_output([exe], input=text, text=True).split()


def plan_py(budget, fixed, depth, maxg, leaf, tile, slice_bytes):
    chunk = max(1, (budget - fixed) // 16) if budget > fixed else 1
    g = depth_py(budget, fixed, depth, maxg, leaf, tile)
    if g < 0:
        return -1, 0, 0, chunk, 0
    used = fixed + block_bytes(g, depth - g, leaf, tile)
    rest = max(budget - used, 0)
    return g, min(rest // 4, 0xFFFFFFFE), (1 + rest // slice_bytes) if slice_bytes else 0, chunk, 0


def test_plan_matches_restatement(plan):
    rng = np.random.default_rng(11)
    for _ in range(300):
        T = int(rng.choice([16, 64, 256, 1024]))
        tile = T * T * 4
        nsub = -(-T // 32) ** 2
        leaf = tile + 8 * (nsub + 1) + int(rng.integers(600, 1200))
        fixed = int(rng.integers(0, 40)) * tile + int(rng.integers(0, 1 << 20))
        budget = fixed + int(rng.integers(0, 2000)) * tile
        depth, maxg = int(rng.integers(0, 14)), int(rng.integers(0, 11))
        sl = int(rng.choice([0, 28 * T * T]))
        got = tuple(int(v) for v in plan("plan %d %d %d %d %d %d %d" % (budget, fixed, depth, maxg, leaf, tile, sl)))
        assert got == plan_py(budget, fixed, depth, maxg, leaf, tile, sl), (budget, fixed, depth, maxg, leaf, tile, sl)
        if got[0] >= 0:  # the fixed set, the block's images and the keys or slices stay within the budget
            used = fixed + block_bytes(got[0], depth - got[0], leaf, tile)
            assert used + 4 * got[1] <= budget
            if sl:
                assert used + (got[2] - 1) * sl <= budget
        assert got[3] >= 1 and (budget <= fixed or fixed + 16 * got[3] <= budget)


def test_fixed_bytes(plan):
    for nc, nt, nf in [(0, 0, 0), (150, 640, 2), (10**6, 5 * 10**5, 7)]:
        assert int(plan("fixed %d %d %d" % (nc, nt, nf))[0]) == 32 * nt + 8 * nc + 16 * nf + 4096


def test_key_batches_from_exact_counts(plan):
    rng = np.random.default_rng(12)
    for _ in range(200):
        n = int(rng.integers(1, 60))
        keys = [int(v) if rng.random() > 0.3 else 0 for v in rng.integers(0, 5000, n)]  # some candidates draw nothing
        cap = int(rng.integers(1, 20000))
        out = [int(v) for v in plan("batches %d %d %s" % (n, cap, " ".join(map(str, keys))))]
        assert (out[0], out[1:]) == batches_py(keys, cap)
        if out[0] >= 0:  # leaf out[0] alone exceeds the key buffer
            continue
        starts = out[1:]
        assert starts[0] == 0 and starts[-1] == n
        for a, b in zip(starts[:-1], starts[1:]):
            assert b > a and sum(keys[a:b]) <= cap
