"""Inpainting planner, host side (csrc/xray_inpaint_plan.h, compiled here with g++): the adjacent leaves against the restatement
of get_adjacent_leaf_node_ids (tests/xray_inpaint_ref.py), every block's leaves, halo images, visible tiles and blend pairs
against a direct Python statement, the copy / in-place visibility difference across a piece's corner, the device bytes and
the block depth; and pcv_xray_inpaint_info's layout against gcc.  No GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import xray_inpaint_ref as R
from xray_merge_ref import Meta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <cstdio>
#include <iostream>
#include "xray_inpaint_plan.h"
using namespace pcv;
static std::vector<uint64_t> read_list() {
    size_t n;
    std::cin >> n;
    std::vector<uint64_t> v(n);
    for (auto& x : v) std::cin >> x;
    return v;
}
int main(int argc, char** argv) {
    const std::string what = argv[1];
    if (what == "adjacent") {  // stdin: D, leaves, then 4 x (present deepest nodes)
        uint32_t D;
        std::cin >> D;
        const std::vector<uint64_t> leaves = read_list();
        std::array<XrayMetaData, 4> m;
        std::array<const XrayMetaData*, 4> p{};
        for (int d = 0; d < 4; ++d) {
            int present;
            std::cin >> present >> m[d].deepest_level;
            for (uint64_t i : read_list()) m[d].nodes.emplace_back(m[d].deepest_level, i);
            if (present) p[d] = &m[d];
        }
        for (uint64_t i : xray_inpaint_adjacent(D, leaves, p)) printf("%llu ", (unsigned long long)i);
        printf("\n");
    } else if (what == "grid") {  // stdin: D j block, leaves, visible; prints the grid
        uint32_t D, j;
        uint64_t b;
        std::cin >> D >> j >> b;
        const std::vector<uint64_t> leaves = read_list(), vis = read_list();
        std::vector<uint64_t> bl;
        for (uint64_t i : leaves) if ((i >> (2 * j)) == b) bl.push_back(i);
        const XrayInpaintGrid g = xray_inpaint_grid(D, j, b, bl, leaves, [&](uint64_t i) { return std::binary_search(vis.begin(), vis.end(), i); });
        printf("%lld %lld %u\n", (long long)g.bx0, (long long)g.by0, g.B);
        auto list = [](const std::vector<uint64_t>& v) { printf("%zu", v.size()); for (uint64_t x : v) printf(" %llu", (unsigned long long)x); printf("\n"); };
        list(g.leaves);
        list(g.image_ids);
        list(g.tile_ids);
        printf("%zu", g.image_pos.size());
        for (uint32_t p : g.image_pos) printf(" %u", p);
        printf("\n%zu", g.tile_slot.size());
        for (int32_t s : g.tile_slot) printf(" %d", s);
        printf("\n%zu", g.hpairs.size());
        for (auto& p : g.hpairs) printf(" %d %d", p.first, p.second);
        printf("\n%zu", g.vpairs.size());
        for (auto& p : g.vpairs) printf(" %d %d", p.first, p.second);
        printf("\n%zu", g.leaf_image.size());
        for (int32_t s : g.leaf_image) printf(" %d", s);
        printf("\n");
    } else if (what == "bytes") {  // bytes j T k D L
        const uint32_t j = atoi(argv[2]), T = atoi(argv[3]), k = atoi(argv[4]), D = atoi(argv[5]), L = atoi(argv[6]);
        printf("%llu %llu %llu\n", (unsigned long long)xray_inpaint_block_bytes(j, T, k), (unsigned long long)xray_merge_device_bytes(D - L, T),
               (unsigned long long)xray_inpaint_device_bytes(j, T, k, D, L));
    } else if (what == "depth") {  // depth budget T k D L
        printf("%d\n", xray_inpaint_block_depth(strtoull(argv[2], nullptr, 10), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6])));
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("xray_inpaint_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    out = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", out, str(src), "-lz"])
    return out


def _run(exe, *args, stdin=""):
    return subprocess.check_output([exe] + [str(a) for a in args], input=stdin, text=True)


def _lst(v):
    return "%d %s\n" % (len(v), " ".join(map(str, v)))


def _adjacent(exe, D, leaves, nbr):
    s = "%d\n" % D + _lst(sorted(leaves))
    for m in nbr:
        s += "%d %d " % (m is not None, m.deepest if m else 0) + _lst([i for _, i in m.nodes] if m else [])
    return [int(x) for x in _run(exe, "adjacent", stdin=s).split()]


def _piece(L, r, D, keep=1.0, rng=None):
    """The leaves at level D under root (L, r), a random share `keep` of them."""
    n = D - L
    leaves = [(r << (2 * n)) + i for i in range(4 ** n)]
    if rng is not None:
        leaves = [i for i in leaves if rng.random() < keep]
    return leaves


@pytest.mark.parametrize("seed", range(8))
def test_adjacent_equals_the_restatement(exe, seed):
    rng = np.random.default_rng(seed)
    L, D = 1 + seed % 2, 3 + seed % 2
    r = int(rng.integers(0, 4 ** L))
    leaves = _piece(L, r, D, 0.6, rng)
    nbr = []
    for dx, dy in R.DIRS:
        n = R.neighbor(L, r, dx, dy)
        if n is None or rng.random() < 0.2:
            nbr.append(None)
            continue
        # a neighbour meta with its deepest nodes (and, at seed 3, a deepest level that differs: no node matches)
        deep = D + (1 if seed == 3 else 0)
        nodes = [(deep, i) for i in _piece(L, n, deep, 0.7, rng)] + [(L, n)]
        nbr.append(Meta(nodes, deepest=deep))
    got = _adjacent(exe, D, leaves, nbr)
    assert got == R.adjacent(D, set(leaves), nbr)
    if seed == 3:
        assert got == []
    # every adjacent leaf touches a leaf across a piece border
    for i in got:
        assert any(R.neighbor(D, i, -dx, -dy) in leaves for dx, dy in R.DIRS)


def _grid(exe, D, j, b, leaves, visible):
    out = _run(exe, "grid", stdin="%d %d %d\n" % (D, j, b) + _lst(sorted(leaves)) + _lst(sorted(visible))).splitlines()
    bx0, by0, B = map(int, out[0].split())
    nums = [list(map(int, l.split()))[1:] for l in out[1:]]
    return dict(bx0=bx0, by0=by0, B=B, leaves=nums[0], images=nums[1], tiles=nums[2], pos=nums[3], slot=nums[4], h=nums[5], v=nums[6], leaf_image=nums[7])


def _expected(D, j, b, leaves, visible):
    B = 1 << j
    x0, y0 = R.xy(D - j, b)
    bx0, by0 = x0 * B, y0 * B
    lim = 1 << D
    leaves = set(leaves)
    images = []
    for iy in range(B + 2):
        for ix in range(B + 2):
            x, y = bx0 - 1 + ix, by0 + B - iy
            if 0 <= x < lim and 0 <= y < lim and R.index_of(D, x, y) in leaves:
                images.append((x, y))
    need = {(x + dx, y + dy) for x, y in images for dx in (-1, 0, 1) for dy in (-1, 0, 1)}
    tiles = []
    for gy in range(B + 4):
        for gx in range(B + 4):
            x, y = bx0 - 2 + gx, by0 + B + 1 - gy
            if (x, y) in need and 0 <= x < lim and 0 <= y < lim and R.index_of(D, x, y) in visible:
                tiles.append(R.index_of(D, x, y))
    h = [(a, images.index((p[0] + 1, p[1]))) for a, p in enumerate(images) if (p[0] + 1, p[1]) in images]
    v = [(a, images.index((p[0], p[1] - 1))) for a, p in enumerate(images) if (p[0], p[1] - 1) in images]
    return [R.index_of(D, *p) for p in images], tiles, h, v


@pytest.mark.parametrize("j", [0, 1, 2])
def test_blocks_halos_and_visible_tiles(exe, j):
    rng = np.random.default_rng(j)
    D = 4
    leaves = sorted(i for i in range(4 ** D) if rng.random() < 0.7)
    visible = set(leaves) | {i for i in range(4 ** D) if rng.random() < 0.2}
    blocks = sorted({i >> (2 * j) for i in leaves})
    seen = []
    for b in blocks:
        g = _grid(exe, D, j, b, leaves, visible)
        images, tiles, h, v = _expected(D, j, b, leaves, visible)
        assert g["leaves"] == [i for i in leaves if i >> (2 * j) == b]
        assert g["images"] == images and g["tiles"] == tiles
        assert [tuple(g["h"][2 * i:2 * i + 2]) for i in range(len(h))] == h
        assert [tuple(g["v"][2 * i:2 * i + 2]) for i in range(len(v))] == v
        assert [images[s] for s in g["leaf_image"]] == g["leaves"]
        assert len(g["slot"]) == (g["B"] + 4) ** 2 and sorted(s for s in g["slot"] if s >= 0) == list(range(len(tiles)))
        seen += g["leaves"]
    assert seen == leaves  # blocks in index order cover every leaf once, in index order


def test_diagonal_across_a_piece_is_hidden_when_copying(exe):
    # piece (1, 0) = x, y in [0, 2) at level 2; its TopRight piece (1, 3) holds the tile (2, 2) diagonal to the leaf (1, 1)
    D, L = 2, 1
    leaves = _piece(L, 0, D)
    diag = R.index_of(D, 2, 2)
    right = [i for i in _piece(L, 2, D)]  # the Right piece (x in [2, 4), y in [0, 2))
    top = [i for i in _piece(L, 1, D)]
    nbr = [None, Meta([(D, i) for i in top], deepest=D), Meta([(D, i) for i in right], deepest=D), None]
    adj = _adjacent(exe, D, leaves, nbr)
    assert diag not in adj and set(adj) == {R.index_of(D, 2, y) for y in (0, 1)} | {R.index_of(D, x, 2) for x in (0, 1)}
    on_disk = set(leaves) | set(right) | set(top) | set(_piece(L, 3, D))
    corner = R.index_of(D, 1, 1)
    copy = _grid(exe, D, 0, corner, leaves, set(leaves) | set(adj))
    place = _grid(exe, D, 0, corner, leaves, on_disk)
    assert diag not in copy["tiles"] and diag in place["tiles"]
    assert set(place["tiles"]) - set(copy["tiles"]) == {diag}


def test_device_bytes_and_block_depth(exe):
    for j, T, k, D, L in ((0, 32, 3, 5, 0), (2, 64, 8, 6, 2), (0, 4096, 8, 9, 0), (1, 256, 0, 4, 4)):
        blk, walk, total = map(int, _run(exe, "bytes", j, T, k, D, L).split())
        tile = T * T * 4
        B = 1 << j
        want = tile if k == 0 else (B + 4) ** 2 * (tile + 4) + (B + 2) ** 2 * (14 * 4 * T * T + 28) + tile
        assert blk == want and total == blk + walk
        assert walk == (0 if D == L else int(_run(exe, "bytes", 0, T, 0, D, L).split()[1]))
    # one 4096 px leaf: 25 tiles of 64 MiB, 9 images of 8192^2 px at 14 bytes per pixel (256 MiB of RGBA + 640 MiB of masks
    # and transforms each), and the leaf: about 10.2 GB
    blk = int(_run(exe, "bytes", 0, 4096, 8, 9, 0).split()[0])
    assert 10.1e9 < blk < 10.3e9
    need = [int(_run(exe, "bytes", j, 64, 8, 6, 0).split()[2]) for j in range(7)]
    assert int(_run(exe, "depth", need[0] - 1, 64, 8, 6, 0)) == -1
    for j in range(6):
        assert int(_run(exe, "depth", need[j], 64, 8, 6, 0)) == j
    assert int(_run(exe, "depth", 1 << 50, 64, 8, 6, 0)) == 5  # at most 2^5 x 2^5 leaves
    assert int(_run(exe, "depth", 1 << 50, 64, 8, 6, 4)) == 2  # at most the piece
    assert int(_run(exe, "depth", 1 << 50, 64, 0, 6, 0)) == 0  # k = 0: one leaf at a time


def test_info_struct_matches_the_c_compiler(tmp_path):
    """pcv_xray_inpaint_info: ctypes size and field offsets equal gcc's for include/pcv.h."""
    from point_cloud_viewer_b200 import _native as N

    fields = [f for f, _ in N.XrayInpaintInfo._fields_]
    c = tmp_path / "layout.c"
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pcv.h"\nint main(void) {\n    printf("%zu", sizeof(pcv_xray_inpaint_info));\n' +
                 "".join('    printf(" %%zu", offsetof(pcv_xray_inpaint_info, %s));\n' % f for f in fields) + "    printf(\"\\n\");\n    return 0;\n}\n")
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, str(c)])
    got = list(map(int, subprocess.check_output([exe], text=True).split()))
    assert got[0] == C.sizeof(N.XrayInpaintInfo)
    assert got[1:] == [getattr(N.XrayInpaintInfo, f).offset for f in fields]
