"""X-ray quadtrees over several clouds: the plan of a list of resident octrees (xray_clouds_fixed_bytes and xray_octree_plan in
csrc/xray_plan.h, compiled here with g++) and of a list of S2 clouds (summed s2_xray_fixed_bytes into s2_xray_plan) against a
Python restatement, and the C++ overloads of include/pcv.hpp over lists of clouds.  No GPU."""
import os
import subprocess

import numpy as np
import pytest

from test_xray_bounded_plan import block_bytes, depth_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <iostream>
#include "xray_plan.h"
int main() {
    std::string what;
    std::cin >> what;
    unsigned long long budget, run_fixed, per_loc, leaf, tile, slice; int depth, maxg; size_t n; unsigned nfilt;
    if (what == "octrees") {
        std::cin >> budget >> run_fixed >> nfilt >> depth >> maxg >> per_loc >> leaf >> tile >> n;
        std::vector<uint64_t> tiles(n);
        for (auto& v : tiles) { unsigned long long t; std::cin >> t; v = t; }
        const uint64_t fixed = pcv::xray_clouds_fixed_bytes(run_fixed, tiles, nfilt);
        const pcv::XrayPlan p = pcv::xray_octree_plan(budget, fixed, 0, depth, maxg, per_loc, leaf, tile, (uint32_t)n);
        std::cout << fixed << " " << p.g << " " << p.sel_cap << " " << p.max_loc << " " << p.key_cap << "\n";
    } else {
        std::cin >> budget >> run_fixed >> nfilt >> depth >> maxg >> leaf >> tile >> slice >> n;
        uint64_t fixed = run_fixed;
        for (size_t k = 0; k < n; ++k) {
            unsigned long long cells, tiles;
            std::cin >> cells >> tiles;
            fixed += pcv::s2_xray_fixed_bytes(cells, tiles, nfilt);
        }
        const pcv::XrayPlan p = pcv::s2_xray_plan(budget, fixed, depth, maxg, leaf, tile, slice);
        std::cout << fixed << " " << p.g << " " << p.max_loc << " " << p.key_cap << " " << p.attr_leaves << "\n";
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    d = tmp_path_factory.mktemp("xray_clouds_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: [int(v) for v in subprocess.check_output([exe], input=text, text=True).split()]


def octree_plan_py(budget, fixed, window, depth, maxg, per_loc, leaf, tile, clouds=1):
    """(g, sel_cap, max_loc, key_cap) of xray_octree_plan: a selection pair costs 24 B of frontier and 16 B of work list per
    cloud (the clouds' frontiers come one at a time, their work lists all stay until the place passes)."""
    pair = 24 + 16 * clouds
    sel = (budget - fixed - window) // 8 if budget > fixed + window else 0
    cap = min(max(sel // 2 // pair, 64), 48 << 20)
    loc = max(1, sel // 2 // per_loc)
    held = fixed + window + sel + pair * cap
    g = depth_py(budget, held, depth, maxg, leaf, tile)
    if g < 0:
        return g, cap, loc, 0
    used = held + block_bytes(g, depth - g, leaf, tile)
    return g, cap, loc, min((budget - used) // 5, 0xFFFFFFFE) if budget > used else 0


def clouds_fixed_py(run_fixed, tiles, nfilt):
    """The driver's fixed set, each cloud's pruning work list (16 B per tile, 16 B more) and the filter intervals (16 B each)."""
    return run_fixed + 16 * nfilt + sum(16 * t + 16 for t in tiles)


def s2_plan_py(budget, fixed, depth, maxg, leaf, tile, slice_bytes):
    g = depth_py(budget, fixed, depth, maxg, leaf, tile)
    loc = max(1, (budget - fixed) // 16) if budget > fixed else 1
    if g < 0:
        return g, loc, 0, 0
    used = fixed + block_bytes(g, depth - g, leaf, tile)
    rest = budget - used if budget > used else 0
    return g, loc, min(rest // 4, 0xFFFFFFFE), (1 + rest // slice_bytes if slice_bytes else 0)


def test_octree_clouds_plan(plan):
    rng = np.random.default_rng(11)
    for _ in range(300):
        T = int(rng.choice([16, 64, 256, 1024]))
        tile = T * T * 4
        leaf = tile + 8 * (-(-T // 32) ** 2 + 1) + int(rng.integers(600, 1200))
        run_fixed = 2 * tile + int(rng.integers(0, 1 << 20))
        tiles = [int(v) for v in rng.integers(0, 1 << 16, int(rng.integers(1, 6)))]
        nfilt = int(rng.integers(0, 4))
        fixed = clouds_fixed_py(run_fixed, tiles, nfilt)
        budget = int(rng.choice([fixed - 1, fixed, fixed + 1, int(np.exp(rng.uniform(np.log(tile), np.log(80 * 2 ** 30))))]))
        depth, maxg, per_loc = int(rng.integers(0, 14)), int(rng.integers(0, 11)), int(rng.integers(100, 2000))
        got = plan("octrees %d %d %d %d %d %d %d %d %d %s\n" % (budget, run_fixed, nfilt, depth, maxg, per_loc, leaf, tile, len(tiles), " ".join(map(str, tiles))))
        assert got[0] == fixed
        K = len(tiles)
        want = octree_plan_py(budget, fixed, 0, depth, maxg, per_loc, leaf, tile, K)
        assert tuple(got[1:]) == want, (budget, fixed, depth, maxg, K)
        if budget <= fixed:
            assert got[1] == -1  # nothing runs when the clouds' fixed set takes the whole budget
        if got[1] >= 0:  # one frontier, every cloud's work list at a full frontier, the block's images and a key batch fit
            sel = (budget - fixed) // 8
            assert fixed + sel + 24 * got[2] + 16 * K * got[2] + block_bytes(got[1], depth - got[1], leaf, tile) + 5 * got[4] <= budget


def test_one_octree_plans_as_before(plan):
    """A list of one cloud without filters holds what the single-octree run held: 16 B per pruning tile and 16 B more."""
    for tiles in (0, 1, 4097):
        got = plan("octrees %d %d 0 5 10 500 %d %d 1 %d\n" % (1 << 30, 70000, 5000, 4096, tiles))
        assert got[0] == 70000 + 16 * tiles + 16
        assert tuple(got[1:]) == octree_plan_py(1 << 30, 70000 + 16 * tiles + 16, 0, 5, 10, 500, 5000, 4096)
        # ... and the plan of xray_octree_plan without the clouds argument, which the single-octree sources call
        from test_xray_bounded_plan import octree_plan_py as single_plan_py
        assert tuple(got[1:]) == single_plan_py(1 << 30, 70000 + 16 * tiles + 16, 0, 5, 10, 500, 5000, 4096)[:4]


def test_s2_clouds_plan(plan):
    rng = np.random.default_rng(12)
    for _ in range(300):
        T = int(rng.choice([16, 64, 256]))
        tile = T * T * 4
        leaf = tile + int(rng.integers(100, 3000))
        slice_bytes = 0 if rng.random() < 0.5 else 28 * T * T
        run_fixed = 2 * tile + int(rng.integers(0, 1 << 20)) + slice_bytes
        clouds = [(int(rng.integers(1, 5000)), int(rng.integers(1, 1 << 16))) for _ in range(int(rng.integers(1, 6)))]
        nfilt = int(rng.integers(0, 4))
        fixed = run_fixed + sum(32 * t + 8 * c + 16 * nfilt + 4096 for c, t in clouds)
        budget = int(rng.choice([fixed - 1, fixed, int(np.exp(rng.uniform(np.log(tile), np.log(80 * 2 ** 30))))]))
        depth, maxg = int(rng.integers(0, 14)), int(rng.integers(0, 11))
        got = plan("s2 %d %d %d %d %d %d %d %d %d %s\n" % (budget, run_fixed, nfilt, depth, maxg, leaf, tile, slice_bytes, len(clouds),
                                                        " ".join("%d %d" % c for c in clouds)))
        assert got[0] == fixed
        assert tuple(got[1:]) == s2_plan_py(budget, fixed, depth, maxg, leaf, tile, slice_bytes)
        if budget <= fixed:
            assert got[1] == -1
        if got[1] >= 0:
            assert fixed + block_bytes(got[1], depth - got[1], leaf, tile) + 4 * got[3] <= budget


CPP = r"""
#include "pcv.hpp"
void use(const pcv::Context& ctx, const pcv::Octree& a, const pcv::Octree& b, const pcv::S2Cells& s, const pcv::S2Cells& t) {
    pcv_xray_quadtree_params pr{};
    auto tile = [](uint8_t, uint64_t, const uint8_t*, uint32_t) {};
    const std::vector<pcv::ClosedInterval> f{{0.0, 10.0}};
    pcv::build_xray_quadtree(std::vector<const pcv::Octree*>{&a, &b}, pr, f, tile);
    pcv::build_xray_quadtree(std::vector<const pcv::S2Cells*>{&s, &t}, pr, f, tile, 1 << 20);
    pcv::build_xray_quadtree_from_dir(ctx, "dir", pr, f, tile);
}
"""


def test_cpp_cloud_overloads_compile(tmp_path):
    src = tmp_path / "clouds.cpp"
    src.write_text(CPP)
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)])
