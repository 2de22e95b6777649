"""X-ray quadtrees from several octree directories: the host-only planning of csrc/xray_dir_plan.h (compiled here with g++) against
a Python restatement - the occupancy pass's (directory, node) work list and its chunks under the chunk, node and tile caps; the
bytes of a block's windows over several directories; the block depth under a budget scan with several directories' work
lists - and windows over the union of several random octrees' boxes, under random query_from_global rotations and with points on
block edges, that hold every node the oracle's nodes_in_location returns for every leaf of their block, in every directory.
No GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_api as O
from test_xray_dir_plan import ENC_BPC, block_depth, random_qfg, window_bytes_py, window_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <cfloat>
#include <iostream>
#include <iomanip>
#include "xray_dir_plan.h"
#include "xray_png.hpp"
using namespace pcv;
static std::vector<std::vector<pcv_node_meta>> read_tables(size_t nd) {
    std::vector<std::vector<pcv_node_meta>> t(nd);
    for (auto& v : t) {
        size_t n;
        std::cin >> n;
        v.resize(n);
        for (auto& m : v) {
            long long np; int enc;
            std::cin >> np >> enc;
            m = pcv_node_meta{};
            m.num_points = np;
            m.position_encoding = enc;
        }
    }
    return t;
}
static std::vector<const std::vector<pcv_node_meta>*> ptrs(const std::vector<std::vector<pcv_node_meta>>& t) {
    std::vector<const std::vector<pcv_node_meta>*> p;
    for (const auto& v : t) p.push_back(&v);
    return p;
}
int main() {
    std::cout << std::setprecision(17);
    std::string what;
    std::cin >> what;
    if (what == "chunks") {  // chunks <ndirs> <tables> <budget> <tile_points> <set_bytes>
        size_t nd;
        std::cin >> nd;
        const auto t = read_tables(nd);
        unsigned long long budget, set_bytes; unsigned tile_points;
        std::cin >> budget >> tile_points >> set_bytes;
        uint64_t largest = 0;
        const std::vector<DirNode> work = xray_occupancy_work(ptrs(t), &largest);
        const OccupancyPlan p = xray_occupancy_plan(budget, largest, tile_points, set_bytes);
        std::cout << largest << " " << p.chunk << " " << p.node_cap << " " << p.tile_cap << " " << p.need << "\n" << work.size();
        for (const DirNode& w : work) std::cout << " " << w.dir << " " << w.node;
        const std::vector<size_t> starts = xray_occupancy_chunks(ptrs(t), work, p, tile_points);
        std::cout << "\n" << starts.size();
        for (size_t s : starts) std::cout << " " << s;
        std::cout << "\n";
    } else if (what == "bytes") {  // bytes <ndirs> <tables> then per directory: has_intensity, window size, window
        size_t nd;
        std::cin >> nd;
        const auto t = read_tables(nd);
        std::vector<char> hi(nd);
        std::vector<std::vector<uint32_t>> w(nd);
        for (size_t k = 0; k < nd; ++k) {
            int h; size_t n;
            std::cin >> h >> n;
            hi[k] = (char)h;
            w[k].resize(n);
            for (auto& v : w[k]) std::cin >> v;
        }
        const WindowsSize s = xray_windows_size(ptrs(t), hi, w);
        std::cout << s.bytes << " " << s.points << " " << s.max_points << " " << s.max_dir << "\n";
    } else if (what == "depth") {
        unsigned long long budget, fixed, leaf, tile, per_loc; int depth, gmax; unsigned clouds;
        std::cin >> budget >> fixed >> depth >> gmax >> leaf >> tile >> per_loc >> clouds;
        std::vector<unsigned long long> w(gmax + 1);
        for (auto& v : w) std::cin >> v;
        std::cout << xray_dir_block_depth(budget, fixed, depth, gmax, leaf, tile, per_loc, [&](int g) { return (uint64_t)w[g]; }, clouds) << "\n";
    } else if (what == "windows") {
        // windows <ndirs> <dir>... <T> <px> <B> <has_q> [qfg x7]: over the union of the directories' boxes, per block at level B
        // its geometry, every directory's window and the locations of its leaves
        size_t nd;
        std::cin >> nd;
        std::vector<std::string> dirs(nd);
        for (auto& d : dirs) std::cin >> d;
        unsigned T; double px; int B, has_q; double qfg[7];
        std::cin >> T >> px >> B >> has_q;
        if (has_q) for (double& v : qfg) std::cin >> v;
        std::vector<std::vector<pcv_node_meta>> nodes(nd);
        std::vector<std::vector<int32_t>> ch(nd);
        double obmin[3] = {0, 0, 0}, obmax[3] = {0, 0, 0};
        for (size_t k = 0; k < nd; ++k) {
            std::string buf;
            read_whole_file(dirs[k] + "/meta.pb", buf);
            MetaHeader h; std::vector<ParsedNode> pn; int version = 0;
            decode_meta(buf, h, pn, version);
            double mn[3], mx[3]; uint64_t np = 0, xb = 0;
            octree_nodes_from_meta(h, pn, mn, mx, nodes[k], np, xb);
            ch[k] = octree_children(nodes[k]);
            for (int a = 0; a < 3; ++a) {  // the union of the boxes, as unite_boxes
                obmin[a] = k == 0 ? mn[a] : std::fmin(obmin[a], mn[a]);
                obmax[a] = k == 0 ? mx[a] : std::fmax(obmax[a], mx[a]);
            }
            std::cout << nodes[k].size() << "\n";
            for (const auto& m : nodes[k])
                std::cout << node_name(m.id_high, m.id_low) << " " << m.num_points << " " << m.position_encoding << " " << m.cube_min[0] << " "
                          << m.cube_min[1] << " " << m.cube_min[2] << " " << m.cube_edge << "\n";
        }
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
            for (size_t k = 0; k < nd; ++k) {
                const std::vector<uint32_t> w = xray_window(nodes[k], ch[k], g);
                std::cout << w.size();
                for (uint32_t i : w) std::cout << " " << i;
                std::cout << "\n";
            }
            const int g_ = deepest - B;
            for (uint64_t l = b << (2 * g_); l < ((b + 1) << (2 * g_)); ++l) {
                const QuadRect r = quad_rect_of(QuadId{deepest, l}, rect);
                const double tmin[3] = {r.min_x, r.min_y, bmin[2]}, tmax[3] = {r.min_x + r.edge, r.min_y + r.edge, bmax[2]};
                const pcv_location loc = xray_location(tmin, tmax, q);
                const double* v = (const double*)&loc.aabb_min;  // every double field of pcv_location, in order
                std::cout << loc.kind;
                for (size_t k = 0; k < (sizeof(pcv_location) - 8) / 8; ++k) std::cout << " " << v[k];
                std::cout << "\n";
            }
        }
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    d = tmp_path_factory.mktemp("xray_dirs_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: subprocess.check_output([exe], input=text, text=True).split("\n")


def _tables_text(tables):
    out = []
    for t in tables:
        out.append(str(len(t)))
        out += ["%d %d" % (n, e) for n, e in t]
    return " ".join(out)


def _xyz_bytes(n, e):
    return n * 3 * ENC_BPC[e]


# ---- Python restatement -------------------------------------------------------------------------------------------------
def occupancy_py(tables, budget, tile_points, set_bytes):
    work = [(k, i) for k, t in enumerate(tables) for i, (n, _) in enumerate(t) if n > 0]
    largest = max([_xyz_bytes(*tables[k][i]) for k, i in work], default=0)
    chunk = max(min(64 << 20, budget // 8), ((largest + 15) & ~15) + 16)
    node_cap = max(64, chunk // 512)
    tile_cap = node_cap + chunk // (3 * tile_points) + 1
    need = chunk + 64 * node_cap + 16 * tile_cap + set_bytes
    starts, nbytes, nt = [0], 0, 0
    for j, (k, i) in enumerate(work):
        n, e = tables[k][i]
        b = (_xyz_bytes(n, e) + 15) & ~15
        t = (n + tile_points - 1) // tile_points
        if j > starts[-1] and (nbytes + b > chunk or j - starts[-1] >= node_cap or nt + t > tile_cap):
            starts.append(j)
            nbytes = nt = 0
        nbytes += b
        nt += t
    starts.append(len(work))
    return largest, (chunk, node_cap, tile_cap, need), work, starts


def windows_bytes_py(tables, has_i, wins):
    total = pts = maxp = maxd = 0
    for k, w in enumerate(wins):
        if not w:
            continue
        nodes = [dict(n=n, enc=e) for n, e in tables[k]]
        b, p, _ = window_bytes_py(nodes, w)
        if not has_i[k]:
            b -= 4 * p
        total += b
        pts += p
        if p > maxp:
            maxp, maxd = p, k
    return total, pts, maxp, maxd


def dir_block_depth_py(budget, fixed, depth, gmax, leaf, tile, per_loc, wmax, clouds):
    pair = 24 + 16 * clouds
    for g in range(gmax, -1, -1):
        w = wmax[g]
        if w == 2 ** 64 - 1 or fixed + w >= budget:
            continue
        sel = (budget - fixed - w) // 8
        cap = min(max(sel // 2 // pair, 64), 48 << 20)
        if block_depth(budget, fixed + w + sel + pair * cap, depth, g, leaf, tile) >= g:
            return g
    return -1


def _random_tables(rng, nd):
    tables = []
    for _ in range(nd):
        nn = int(rng.integers(0, 400))
        kinds = rng.random(nn)
        pts = np.where(kinds < 0.15, 0, np.where(kinds < 0.97, rng.integers(1, 6000, nn), rng.integers(10 ** 5, 3 * 10 ** 6, nn)))
        tables.append([(int(p), int(rng.integers(1, 5))) for p in pts])
    return tables


@pytest.mark.parametrize("seed", range(12))
def test_occupancy_chunks(plan, seed):
    rng = np.random.default_rng(seed)
    tables = _random_tables(rng, int(rng.integers(1, 6)))
    for budget in (1 << 20, 24 << 20, 300 << 20, 4 << 30):
        tile_points = int(rng.choice([64, 2048]))
        set_bytes = int(rng.integers(0, 1 << 20))
        out = plan("chunks %d %s %d %d %d\n" % (len(tables), _tables_text(tables), budget, tile_points, set_bytes))
        largest, chunk, node_cap, tile_cap, need = map(int, out[0].split())
        f = list(map(int, out[1].split()))
        work = list(zip(f[1::2], f[2::2]))
        starts = list(map(int, out[2].split()))[1:]
        wl, wplan, wwork, wstarts = occupancy_py(tables, budget, tile_points, set_bytes)
        assert (largest, (chunk, node_cap, tile_cap, need), work, starts) == (wl, wplan, wwork, wstarts)
        # every node with points exactly once, in directory order; every chunk within its caps
        assert len(work) == sum(1 for t in tables for n, _ in t if n > 0) and work == sorted(work)
        for a, b in zip(starts, starts[1:]):
            assert b > a
            nodes = [tables[k][i] for k, i in work[a:b]]
            assert len(nodes) <= node_cap
            assert sum((_xyz_bytes(n, e) + 15) & ~15 for n, e in nodes) <= chunk
            assert sum((n + tile_points - 1) // tile_points for n, _ in nodes) <= tile_cap


@pytest.mark.parametrize("seed", range(8))
def test_windows_bytes(plan, seed):
    rng = np.random.default_rng(50 + seed)
    nd = int(rng.integers(1, 6))
    tables = _random_tables(rng, nd)
    for _ in range(10):
        has_i = [int(v) for v in rng.integers(0, 2, nd)]
        wins = []
        for t in tables:
            if not t or rng.random() < 0.25:
                wins.append([])
            else:
                wins.append(sorted(int(v) for v in rng.choice(len(t), int(rng.integers(1, len(t) + 1)), replace=False)))
        cmd = "bytes %d %s " % (nd, _tables_text(tables))
        cmd += " ".join("%d %d %s" % (h, len(w), " ".join(map(str, w))) for h, w in zip(has_i, wins))
        got = tuple(map(int, plan(cmd + "\n")[0].split()))
        assert got == windows_bytes_py(tables, has_i, wins)
    # no window: nothing to load
    assert tuple(map(int, plan("bytes 2 %s 1 0 0 0\n" % _tables_text(tables[:1] * 2))[0].split())) == (0, 0, 0, 0)


def test_block_depth_budget_scan(plan):
    rng = np.random.default_rng(7)
    U = 2 ** 64 - 1
    for _ in range(60):
        gmax = int(rng.integers(0, 8))
        depth = gmax + int(rng.integers(0, 4))
        tile = int(rng.choice([256, 4096, 65536]))
        leaf, per_loc = tile + 1200, 1100
        w = sorted((int(v) for v in rng.integers(10 ** 4, 10 ** 8, gmax + 1)))
        if rng.random() < 0.3:
            w[-1] = U
        fixed = 2 * tile + 5000
        clouds = int(rng.integers(1, 9))
        for budget in [int(v) for v in np.geomspace(10 ** 4, 10 ** 10, 25)]:
            got = int(plan("depth %d %d %d %d %d %d %d %d %s\n" % (budget, fixed, depth, gmax, leaf, tile, per_loc, clouds, " ".join(map(str, w))))[0])
            want = dir_block_depth_py(budget, fixed, depth, gmax, leaf, tile, per_loc, w, clouds)
            assert got == want, (budget, w, clouds)


def _octree_dir(tmp_path, seed, box, n, mppn):
    rng = np.random.default_rng(seed)
    lo, hi = np.array(box[:3]), np.array(box[3:])
    p = lo + rng.uniform(0.0, 1.0, (n, 3)) * (hi - lo)
    p[: n // 10, 0] = np.round(p[: n // 10, 0] / 16.0) * 16.0  # points on block edges
    p[n // 10: n // 5, 1] = np.round(p[n // 10: n // 5, 1] / 8.0) * 8.0
    p = np.clip(p, lo, hi)
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    inten = rng.uniform(0, 100, n).astype(np.float32)
    ref = O.build(p[:, 0].copy(), p[:, 1].copy(), p[:, 2].copy(), rgb, 1.0 / 256, tuple(lo), tuple(hi), intensity=inten, max_points_per_node=mppn)
    d = str(tmp_path / ("o%d" % seed))
    os.makedirs(d)
    ref.write_dir(d)
    return ref, d


def _parse(lines, nd, B):
    it = iter(lines)
    tables = []
    for _ in range(nd):
        nn = int(next(it))
        nodes = []
        for _ in range(nn):
            f = next(it).split()
            nodes.append(dict(name=f[0], n=int(f[1]), enc=int(f[2]), m=tuple(float(v) for v in f[3:6]), e=float(f[6])))
        tables.append(nodes)
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
        wins = [[int(v) for v in next(it).split()[1:]] for _ in range(nd)]
        locs = []
        for _ in range(4 ** (deepest - B)):
            f = next(it).split()
            loc = O.Location()
            loc.kind = int(f[0])
            vals = [float(v) for v in f[1:]]
            arr = (C.c_double * len(vals)).from_buffer_copy(np.array(vals, np.float64).tobytes())
            C.memmove(C.addressof(loc) + O.Location.aabb_min.offset, arr, C.sizeof(arr))
            locs.append(loc)
        blocks.append(dict(axes=axes, corners=corners, wins=wins, locs=locs))
    return tables, deepest, blocks


@pytest.mark.parametrize("seed", range(5))
def test_windows_of_several_directories_hold_the_oracles_nodes(plan, tmp_path, seed):
    """Three octrees with different boxes, cubes and max_points_per_node over the union of their boxes: every directory's window
    of a block is the restatement's and holds every node of that directory the oracle selects for any leaf of the block."""
    rng = np.random.default_rng(200 + seed)
    specs = [((0.0, 0.0, 0.0, 64.0, 64.0, 8.0), 5000, 300), ((30.0, 20.0, -2.0, 90.0, 50.0, 6.0), 4000, 150),
             ((-10.0, 40.0, 1.0, 20.0, 70.0, 3.0), 3000, 600)]
    refs, dirs = [], []
    for k, (box, n, mppn) in enumerate(specs):
        r, d = _octree_dir(tmp_path, 10 * seed + k, box, n, mppn)
        refs.append(r)
        dirs.append(d)
    order = list(rng.permutation(3))
    refs, dirs = [refs[k] for k in order], [dirs[k] for k in order]
    qfg = None if seed % 2 == 0 else random_qfg(rng)
    T, px, B = 8, 1.0, 1 + seed % 2
    cmd = "windows 3 %s %d %r %d %d" % (" ".join(dirs), T, px, B, 0 if qfg is None else 1)
    if qfg is not None:
        cmd += " " + " ".join(repr(v) for v in qfg)
    tables, deepest, blocks = _parse(plan(cmd + "\n"), 3, B)
    assert len(blocks) == 4 ** B
    for k in range(3):
        assert sorted(n["name"] for n in tables[k]) == sorted(refs[k].nodes)
    pruned = empty = 0
    for blk in blocks:
        for k in range(3):
            w = blk["wins"][k]
            assert w == window_py(tables[k], blk["axes"], blk["corners"])
            names = {tables[k][i]["name"] for i in w}
            for loc in blk["locs"]:
                assert set(refs[k].nodes_in_location(loc)) <= names
            pruned += len(w) < len(tables[k])
            empty += not w
    assert pruned > 0  # windows prune
    if qfg is None:
        assert empty > 0  # some block misses a whole directory: its window is empty and is not loaded

