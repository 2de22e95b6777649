"""X-ray quadtrees from an octree directory: the window planner (csrc/xray_dir_plan.h, compiled here with g++) against a Python
restatement - the node table from meta.pb, windows, window bytes, the block depth under a budget scan - windows that hold every
node the oracle's nodes_in_location returns for every leaf of their block (random octrees, random query_from_global rotations,
points on block edges), and the pcv_xray_dir_info layout.  No GPU."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import oracle_api as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <cfloat>
#include <iostream>
#include <iomanip>
#include "xray_dir_plan.h"
#include "xray_png.hpp"
using namespace pcv;
static void put_loc(const pcv_location& l) {
    const double* v = (const double*)&l.aabb_min;  // every double field of pcv_location, in order
    std::cout << l.kind;
    for (size_t k = 0; k < (sizeof(pcv_location) - 8) / 8; ++k) std::cout << " " << v[k];
    std::cout << "\n";
}
int main() {
    std::cout << std::setprecision(17);
    std::string what;
    std::cin >> what;
    if (what == "depth") {
        unsigned long long budget, fixed, leaf, tile, per_loc; int depth, gmax;
        std::cin >> budget >> fixed >> depth >> gmax >> leaf >> tile >> per_loc;
        std::vector<unsigned long long> w(gmax + 1);
        for (auto& v : w) std::cin >> v;
        std::cout << xray_dir_block_depth(budget, fixed, depth, gmax, leaf, tile, per_loc, [&](int g) { return (uint64_t)w[g]; }) << "\n";
        return 0;
    }
    // windows <dir> <T> <px> <B> <has_q> [qfg x7]: the node table, then per block at level B: its geometry, its window, its
    // window bytes and the locations of its leaves
    std::string dir; unsigned T; double px; int B, has_q; double qfg[7];
    std::cin >> dir >> T >> px >> B >> has_q;
    if (has_q) for (double& v : qfg) std::cin >> v;
    std::string buf;
    read_whole_file(dir + "/meta.pb", buf);
    MetaHeader h; std::vector<ParsedNode> pn; int version = 0;
    decode_meta(buf, h, pn, version);
    double obmin[3], obmax[3]; std::vector<pcv_node_meta> nodes; uint64_t np = 0, xb = 0;
    octree_nodes_from_meta(h, pn, obmin, obmax, nodes, np, xb);
    std::cout << nodes.size() << " " << np << " " << xb << "\n";
    for (const auto& m : nodes)
        std::cout << node_name(m.id_high, m.id_low) << " " << m.num_points << " " << m.position_encoding << " " << m.cube_min[0] << " " << m.cube_min[1] << " "
                  << m.cube_min[2] << " " << m.cube_edge << " " << m.point_offset << " " << m.xyz_byte_offset << "\n";
    const std::vector<int32_t> ch = octree_children(nodes);
    double bmin[3], bmax[3];  // the quadtree's frame, as xray_api.inl's quad_driver_init
    for (int a = 0; a < 3; ++a) bmin[a] = obmin[a], bmax[a] = obmax[a];
    const double* q = has_q ? qfg : nullptr;
    if (q) {
        double lo[3], hi[3];
        for (int k = 0; k < 8; ++k) {
            const V3 p = iso_apply(q, V3{(k & 1) ? obmax[0] : obmin[0], (k & 2) ? obmax[1] : obmin[1], (k & 4) ? obmax[2] : obmin[2]});
            const double v[3] = {p.x, p.y, p.z};
            for (int a = 0; a < 3; ++a) lo[a] = k == 0 ? v[a] : std::fmin(lo[a], v[a]), hi[a] = k == 0 ? v[a] : std::fmax(hi[a], v[a]);
        }
        for (int a = 0; a < 3; ++a) bmin[a] = lo[a], bmax[a] = hi[a];
    }
    QuadRect rect; uint8_t deepest = 0;
    quadtree_rect_and_levels(bmin, bmax, T, px, rect, deepest);
    double big = 0;
    for (int a = 0; a < 3; ++a) big = std::fmax(big, std::fmax(std::fabs(obmin[a]), std::fabs(obmax[a])));
    big = std::fmax(big, std::fmax(std::fabs(rect.min_x), std::fabs(rect.min_y)) + rect.edge);
    if (q) for (int a = 0; a < 3; ++a) big = std::fmax(big, std::fmax(std::fabs(bmin[a]), std::fabs(bmax[a])));
    const double margin = std::ldexp(rect.edge, -B) / 1024. + 64. * (double)(deepest + 1) * big * DBL_EPSILON;
    std::cout << (int)deepest << "\n";
    for (uint64_t b = 0; b < (1ull << (2 * B)); ++b) {
        const QueryGeom g = make_query_geom(xray_block_location(rect, B, b, bmin, bmax, margin, q));
        std::cout << "block " << b << " " << g.naxes;
        for (int k = 0; k < g.naxes; ++k) std::cout << " " << g.axes[k][0] << " " << g.axes[k][1] << " " << g.axes[k][2];
        for (int k = 0; k < 8; ++k) std::cout << " " << g.corners[k][0] << " " << g.corners[k][1] << " " << g.corners[k][2];
        std::cout << "\n";
        const std::vector<uint32_t> w = xray_window(nodes, ch, g);
        std::cout << w.size();
        for (uint32_t i : w) std::cout << " " << i;
        const WindowSize ws = xray_window_size(nodes, w, true);
        std::cout << "\n" << ws.bytes << " " << ws.points << " " << ws.xyz_bytes << "\n";
        const int g_ = deepest - B;
        for (uint64_t l = b << (2 * g_); l < ((b + 1) << (2 * g_)); ++l) {
            const QuadRect r = quad_rect_of(QuadId{deepest, l}, rect);
            const double tmin[3] = {r.min_x, r.min_y, bmin[2]}, tmax[3] = {r.min_x + r.edge, r.min_y + r.edge, bmax[2]};
            put_loc(xray_location(tmin, tmax, q));
        }
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    d = tmp_path_factory.mktemp("xray_dir_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: subprocess.check_output([exe], input=text, text=True).split("\n")


# ---- Python restatement -------------------------------------------------------------------------------------------------
def block_bytes(g, above, leaf, tile):
    return 4 ** g * leaf + (4 ** g - 1) // 3 * tile + (4 * above + 1) * tile


def block_depth(budget, fixed, depth, maxg, leaf, tile):
    if budget <= fixed or block_bytes(0, depth, leaf, tile) > budget - fixed:
        return -1
    half = (budget - fixed) // 2
    g = 0
    while g < min(depth, maxg) and block_bytes(g + 1, depth - g - 1, leaf, tile) <= half:
        g += 1
    return g


def dir_block_depth(budget, fixed, depth, gmax, leaf, tile, per_loc, wmax):
    for g in range(gmax, -1, -1):
        w = wmax[g]
        if w == 2 ** 64 - 1 or fixed + w >= budget:
            continue
        sel = (budget - fixed - w) // 8
        cap = min(max(sel // 2 // 40, 64), 48 << 20)
        if block_depth(budget, fixed + w + sel + 40 * cap, depth, g, leaf, tile) >= g:
            return g
    return -1


def sat_out(axes, corners, m, e):
    cube = np.array([[m[0] + (e if i & 1 else 0), m[1] + (e if i & 2 else 0), m[2] + (e if i & 4 else 0)] for i in range(8)])
    for ax in axes:
        pa, pb = corners @ ax, cube @ ax
        if pb.min() > pa.max() or pb.max() < pa.min():
            return True
    return False


def window_py(nodes, axes, corners):
    """Nodes whose cube and every ancestor's cube are not Out (nodes_in_location's BFS semantics), by testing every node."""
    names = {n["name"]: i for i, n in enumerate(nodes)}
    out = []
    for i, n in enumerate(nodes):
        name, ok = n["name"], True
        while ok and name:
            if name not in names or sat_out(axes, corners, nodes[names[name]]["m"], nodes[names[name]]["e"]):
                ok = False
            name = name[:-1] if len(name) > 1 else ""
        if ok:
            out.append(i)
    return out


ENC_BPC = {1: 1, 2: 2, 3: 4, 4: 8}


def window_bytes_py(nodes, win):
    xb = pts = 0
    for i in win:
        xb = (xb + 15) & ~15
        xb += nodes[i]["n"] * 3 * ENC_BPC[nodes[i]["enc"]]
        pts += nodes[i]["n"]
    return xb + 32 + max(3 * pts, 16) + 4 * pts + 98 * len(win), pts, xb


def parse(lines, B):
    it = iter(lines)
    nn, npts, xb = map(int, next(it).split())
    nodes = []
    for _ in range(nn):
        f = next(it).split()
        nodes.append(dict(name=f[0], n=int(f[1]), enc=int(f[2]), m=tuple(float(v) for v in f[3:6]), e=float(f[6]), poff=int(f[7]), xoff=int(f[8])))
    deepest = int(next(it))
    blocks = []
    for line in it:
        if not line.startswith("block"):
            continue
        f = line.split()
        na = int(f[2])
        vals = [float(v) for v in f[3:]]
        axes = np.array(vals[:3 * na]).reshape(na, 3)
        corners = np.array(vals[3 * na:]).reshape(8, 3)
        w = [int(v) for v in next(it).split()[1:]]
        size = tuple(int(v) for v in next(it).split())
        locs = []
        blocks.append(dict(axes=axes, corners=corners, win=w, size=size, locs=locs))
        nleaf = 4 ** (deepest - B)
        for _ in range(nleaf):
            f = next(it).split()
            loc = O.Location()
            loc.kind = int(f[0])
            vals = [float(v) for v in f[1:]]
            arr = (C.c_double * len(vals)).from_buffer_copy(np.array(vals, np.float64).tobytes())
            C.memmove(C.addressof(loc) + O.Location.aabb_min.offset, arr, C.sizeof(arr))
            locs.append(loc)
    return dict(nodes=nodes, npts=npts, xyz_bytes=xb, deepest=deepest, blocks=blocks)


def octree_dir(tmp_path, seed, n=6000, mppn=300):
    rng = np.random.default_rng(seed)
    x, y, z = rng.uniform(0.0, 64.0, n), rng.uniform(0.0, 64.0, n), rng.uniform(0.0, 8.0, n)
    x[: n // 10] = np.round(x[: n // 10] / 16.0) * 16.0  # points on block edges
    y[n // 10: n // 5] = np.round(y[n // 10: n // 5] / 8.0) * 8.0
    keep = ~((x > 40) & (y > 40))
    x, y, z = x[keep], y[keep], z[keep]
    rgb = rng.integers(0, 256, (len(x), 3), dtype=np.uint8)
    inten = rng.uniform(0, 100, len(x)).astype(np.float32)
    ref = O.build(x, y, z, rgb, 1.0 / 256, (0.0, 0.0, 0.0), (64.0, 64.0, 8.0), intensity=inten, max_points_per_node=mppn)
    d = str(tmp_path / ("o%d" % seed))
    os.makedirs(d)
    ref.write_dir(d)
    return ref, d


def random_qfg(rng):
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    ang = rng.uniform(-math.pi, math.pi)
    s = math.sin(ang / 2)
    return [float(v) for v in rng.uniform(-50, 50, 3)] + [ax[0] * s, ax[1] * s, ax[2] * s, math.cos(ang / 2)]


@pytest.mark.parametrize("seed", range(5))
def test_windows_against_restatement_and_oracle(plan, tmp_path, seed):
    ref, d = octree_dir(tmp_path, seed)
    rng = np.random.default_rng(100 + seed)
    qfg = None if seed % 2 == 0 else random_qfg(rng)
    T, px = 8, 1.0
    B = 1 + seed % 2
    cmd = "windows %s %d %r %d %d" % (d, T, px, B, 0 if qfg is None else 1)
    if qfg is not None:
        cmd += " " + " ".join(repr(v) for v in qfg)
    out = parse(plan(cmd + "\n"), B)
    nodes = out["nodes"]
    # the node table as load_dir lays it out: sorted by NodeId, cubes of the oracle, 16-byte aligned positions
    assert sorted(n["name"] for n in nodes) == sorted(ref.nodes)
    xo = po = 0
    for n in nodes:
        m = ref.nodes[n["name"]]
        assert (n["n"], n["enc"]) == (m["num_points"], m["enc"]) and n["m"] + (n["e"],) == m["cube"]
        xo = (xo + 15) & ~15
        assert (n["poff"], n["xoff"]) == (po, xo)
        po += n["n"]
        xo += n["n"] * 3 * ENC_BPC[n["enc"]]
    assert (out["npts"], out["xyz_bytes"]) == (po, xo)
    assert len(out["blocks"]) == 4 ** B
    smaller = 0
    for blk in out["blocks"]:
        assert blk["win"] == window_py(nodes, blk["axes"], blk["corners"])
        assert blk["size"] == window_bytes_py(nodes, blk["win"])
        names = {nodes[i]["name"] for i in blk["win"]}
        for loc in blk["locs"]:
            assert set(ref.nodes_in_location(loc)) <= names
        smaller += len(blk["win"]) < len(nodes)
    assert smaller > 0  # windows prune


def test_block_depth_budget_scan(plan):
    rng = np.random.default_rng(1)
    U = 2 ** 64 - 1
    for _ in range(60):
        gmax = int(rng.integers(0, 8))
        depth = gmax + int(rng.integers(0, 4))
        tile = int(rng.choice([256, 4096, 65536]))
        leaf, per_loc = tile + 1200, 1100
        w = sorted((int(v) for v in rng.integers(10 ** 4, 10 ** 8, gmax + 1)))  # windows shrink with g
        if rng.random() < 0.3:
            w[-1] = U
        fixed = 2 * tile + 5000
        for budget in [int(v) for v in np.geomspace(10 ** 4, 10 ** 10, 25)]:
            got = int(plan("depth %d %d %d %d %d %d %d %s\n" % (budget, fixed, depth, gmax, leaf, tile, per_loc, " ".join(map(str, w))))[0])
            assert got == dir_block_depth(budget, fixed, depth, gmax, leaf, tile, per_loc, w), (budget, w)


def test_xray_dir_info_struct_matches_the_c_compiler(tmp_path):
    """pcv_xray_dir_info: ctypes size and field offsets equal gcc's for include/pcv.h."""
    from point_cloud_viewer_b200 import _native as N

    fs = [f for f, _ in N.XrayDirInfo._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "pcv.h"', "int main(void) {", 'printf("size %zu\\n", sizeof(pcv_xray_dir_info));']
    for f in fs:
        src.append('printf("%s %%zu\\n", offsetof(pcv_xray_dir_info, %s));' % (f, f))
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, str(c)])
    got = dict(l.split() for l in subprocess.check_output([exe], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(N.XrayDirInfo)
    for f in fs:
        assert int(got[f]) == getattr(N.XrayDirInfo, f).offset, f
