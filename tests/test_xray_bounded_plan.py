"""Bounded X-ray quadtree: the planner (csrc/xray_plan.h, compiled here with g++) against a Python restatement - block depth
from the budget, the octree sources' plan, key-batch splits, the post-order of a sparse leaf set - and the
pcv_xray_bounded_info layout.  No GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <iostream>
#include "xray_plan.h"
int main() {
    std::string what;
    std::cin >> what;
    if (what == "depth") {
        unsigned long long budget, fixed, leaf, tile; int depth, maxg;
        std::cin >> budget >> fixed >> depth >> maxg >> leaf >> tile;
        std::cout << pcv::xray_block_depth(budget, fixed, depth, maxg, leaf, tile) << "\n";
    } else if (what == "octree") {
        unsigned long long budget, fixed, window, per_loc, leaf, tile; int depth, maxg;
        std::cin >> budget >> fixed >> window >> depth >> maxg >> per_loc >> leaf >> tile;
        const pcv::XrayPlan p = pcv::xray_octree_plan(budget, fixed, window, depth, maxg, per_loc, leaf, tile);
        std::cout << p.g << " " << p.sel_cap << " " << p.max_loc << " " << p.key_cap << " " << p.attr_leaves << "\n";
    } else if (what == "batches") {
        size_t n; unsigned long long cap;
        std::cin >> n >> cap;
        std::vector<uint64_t> k(n);
        for (auto& v : k) { unsigned long long t; std::cin >> t; v = t; }
        int64_t big = -1;
        const std::vector<uint32_t> s = pcv::xray_key_batches(k, cap, &big);
        std::cout << big;
        for (uint32_t v : s) std::cout << " " << v;
        std::cout << "\n";
    } else {
        size_t n; int depth;
        std::cin >> n >> depth;
        std::vector<uint64_t> l(n);
        for (auto& v : l) { unsigned long long t; std::cin >> t; v = t; }
        for (const auto& e : pcv::xray_post_order(l, depth)) std::cout << e.first << " " << e.second << "\n";
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    d = tmp_path_factory.mktemp("xray_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: subprocess.check_output([exe], input=text, text=True).split("\n")


def block_bytes(g, above, leaf, tile):
    return 4 ** g * leaf + (4 ** g - 1) // 3 * tile + (4 * above + 1) * tile


def depth_py(budget, fixed, depth, maxg, leaf, tile):
    if budget <= fixed or block_bytes(0, depth, leaf, tile) > budget - fixed:
        return -1
    half = (budget - fixed) // 2
    g = 0
    while g < min(depth, maxg) and block_bytes(g + 1, depth - g - 1, leaf, tile) <= half:
        g += 1
    return g


def octree_plan_py(budget, fixed, window, depth, maxg, per_loc, leaf, tile):
    """(g, sel_cap, max_loc, key_cap, attr_leaves): an eighth of what fixed + window leave for the node selection, the block
    depth besides it, and the rest after the block's images for keys of 5 bytes each."""
    sel = (budget - fixed - window) // 8 if budget > fixed + window else 0
    cap = min(max(sel // 2 // 40, 64), 48 << 20)
    loc = max(1, sel // 2 // per_loc)
    held = fixed + window + sel + 40 * cap
    g = depth_py(budget, held, depth, maxg, leaf, tile)
    if g < 0:
        return g, cap, loc, 0, 0
    used = held + block_bytes(g, depth - g, leaf, tile)
    return g, cap, loc, min((budget - used) // 5, 0xFFFFFFFE) if budget > used else 0, 0


def batches_py(keys, cap):
    starts, run = [], 0
    for i, k in enumerate(keys):
        if k > cap:
            return i, []
        if not starts or run + k > cap:
            starts.append(i)
            run = 0
        run += k
    return -1, starts + [len(keys)]


def post_order_py(leaves, depth):
    """Every ancestor of a leaf (and the leaf) after its children: a recursive walk over the set."""
    exist = [set() for _ in range(depth + 1)]  # by levels above the leaves
    for l in leaves:
        for up in range(depth + 1):
            exist[up].add(l >> (2 * up))
    out = []

    def walk(up, idx):
        if up > 0:
            for k in range(4):
                if (idx << 2) + k in exist[up - 1]:
                    walk(up - 1, (idx << 2) + k)
        out.append((up, idx))

    for r in sorted(exist[depth]):
        walk(depth, r)
    return out


def test_block_depth(plan):
    for tile in (8 * 8 * 4, 32 * 32 * 4, 256 * 256 * 4):
        leaf = tile + 1000
        for depth in (0, 1, 5, 14):
            for budget in (tile, 3 * tile, 40 * tile, 10 ** 6, 10 ** 8, 80 * 2 ** 30):
                for fixed in (0, 2 * tile + 5000):
                    got = int(plan("depth %d %d %d 10 %d %d\n" % (budget, fixed, depth, leaf, tile))[0])
                    assert got == depth_py(budget, fixed, depth, 10, leaf, tile), (tile, depth, budget, fixed)


def test_octree_plan(plan):
    rng = np.random.default_rng(5)
    for _ in range(300):
        T = int(rng.choice([16, 64, 256, 1024]))
        tile = T * T * 4
        leaf = tile + 8 * (-(-T // 32) ** 2 + 1) + int(rng.integers(600, 1200))
        fixed = 2 * tile + int(rng.integers(0, 1 << 20))
        window = 0 if rng.random() < 0.5 else int(rng.integers(0, 1 << 28))
        budget = int(rng.choice([fixed, fixed + window, int(np.exp(rng.uniform(np.log(tile), np.log(80 * 2 ** 30))))]))
        depth, maxg, per_loc = int(rng.integers(0, 14)), int(rng.integers(0, 11)), int(rng.integers(100, 2000))
        got = tuple(int(v) for v in plan("octree %d %d %d %d %d %d %d %d\n" % (budget, fixed, window, depth, maxg, per_loc, leaf, tile))[0].split())
        want = octree_plan_py(budget, fixed, window, depth, maxg, per_loc, leaf, tile)
        assert got == want, (budget, fixed, window, depth, maxg, per_loc, leaf, tile)
        if got[0] >= 0:  # the fixed set, the window, the selection, the block's images and a key batch stay within the budget
            sel = (budget - fixed - window) // 8
            assert got[0] <= min(depth, maxg) and sel // 2 >= got[2] * per_loc or got[2] == 1
            assert fixed + window + sel + 40 * got[1] + block_bytes(got[0], depth - got[0], leaf, tile) + 5 * got[3] <= budget


@pytest.mark.parametrize("seed", range(6))
def test_key_batches(plan, seed):
    rng = np.random.default_rng(seed)
    keys = [int(v) for v in rng.integers(1, 5000, int(rng.integers(1, 60)))]
    for cap in (max(keys), max(keys) * 3, sum(keys), 4999, 1):
        out = [int(v) for v in plan("batches %d %d %s\n" % (len(keys), cap, " ".join(map(str, keys))))[0].split()]
        big, starts = batches_py(keys, cap)
        assert out[0] == big and out[1:] == starts
        if big < 0:
            assert all(sum(keys[a:b]) <= cap for a, b in zip(starts, starts[1:]))


@pytest.mark.parametrize("seed", range(8))
def test_post_order_of_sparse_leaves(plan, seed):
    rng = np.random.default_rng(seed)
    depth = int(rng.integers(0, 7))
    n = int(rng.integers(1, min(4 ** depth, 40) + 1))
    leaves = sorted(set(int(v) for v in rng.integers(0, 4 ** depth, n)))
    lines = plan("post %d %d %s\n" % (len(leaves), depth, " ".join(map(str, leaves))))
    got = [tuple(int(t) for t in l.split()) for l in lines if l.strip()]
    assert got == post_order_py(leaves, depth)
    pos = {e: i for i, e in enumerate(got)}
    assert len(pos) == len(got)
    for up, idx in got:
        if up > 0:
            assert all(pos[(up - 1, (idx << 2) + k)] < pos[(up, idx)] for k in range(4) if (up - 1, (idx << 2) + k) in pos)


def test_xray_bounded_info_struct_matches_the_c_compiler(tmp_path):
    """pcv_xray_bounded_info: ctypes size and field offsets equal gcc's for include/pcv.h."""
    from point_cloud_viewer_b200 import _native as N

    fs = [f for f, _ in N.XrayBoundedInfo._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "pcv.h"', "int main(void) {", 'printf("size %zu\\n", sizeof(pcv_xray_bounded_info));']
    for f in fs:
        src.append('printf("%s %%zu\\n", offsetof(pcv_xray_bounded_info, %s));' % (f, f))
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, str(c)])
    got = dict(l.split() for l in subprocess.check_output([exe], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(N.XrayBoundedInfo)
    for f in fs:
        assert int(got[f]) == getattr(N.XrayBoundedInfo, f).offset, f
