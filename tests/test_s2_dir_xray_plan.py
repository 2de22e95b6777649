"""X-ray quadtrees from S2 directories: the host-only planner (csrc/s2_dir_xray_plan.h, compiled here with g++) against a Python
restatement - the scan pass's chunks, which cut cells larger than a chunk and cover every point exactly once; window bytes for
every strategy and filter combination; the block depth under a budget scan - and the meta.pb opener shared with load_s2_dir
(open_s2_dir_cells in csrc/s2_disk.hpp), which rejects what load_s2_dir rejects with the same codes and messages.  No GPU."""
import os
import struct
import subprocess

import numpy as np
import pytest

from test_s2_xray_plan import plan_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HARNESS = r"""
#include <iostream>
#include "s2_dir_xray_plan.h"
#include "s2_disk.hpp"
using namespace pcv;
int main() {
    std::string what;
    while (std::cin >> what) {
        if (what == "chunks") {
            size_t n; unsigned long long chunk, maxp;
            std::cin >> n >> chunk >> maxp;
            std::vector<uint64_t> counts(n);
            for (auto& v : counts) std::cin >> v;
            std::vector<S2Piece> pieces;
            const std::vector<size_t> starts = s2_scan_chunks(counts, chunk, maxp, pieces);
            std::cout << starts.size();
            for (size_t s : starts) std::cout << " " << s;
            std::cout << "\n" << pieces.size();
            for (const auto& p : pieces) std::cout << " " << p.cell << " " << p.first << " " << p.count;
            std::cout << "\n";
        } else if (what == "bytes") {
            unsigned long long points, cells, tiles; int strategy; unsigned nfilt;
            std::cin >> points >> cells >> tiles >> strategy >> nfilt;
            std::cout << s2_window_bytes(points, cells, tiles, strategy, nfilt) << "\n";
        } else if (what == "depth") {
            unsigned long long budget, fixed, leaf, tile, slice; int depth, gmax;
            std::cin >> budget >> fixed >> depth >> gmax >> leaf >> tile >> slice;
            std::vector<unsigned long long> w(gmax + 1);
            for (auto& v : w) std::cin >> v;
            std::cout << s2_dir_block_depth(budget, fixed, depth, gmax, leaf, tile, slice, [&](int g) { return (uint64_t)w[g]; }) << "\n";
        } else if (what == "open") {
            std::string dir;
            std::cin >> dir;
            S2DirCells dc;
            std::string err;
            const int rc = open_s2_dir_cells(dir, dc, err);
            std::cout << rc << "\n" << err << "\n" << dc.ids.size() << " " << dc.n << " " << dc.level << " " << dc.m.has_color << " " << dc.m.has_intensity;
            for (size_t k = 0; k < dc.ids.size(); ++k) std::cout << " " << dc.ids[k] << " " << dc.counts[k] << " " << dc.starts[k];
            std::cout << "\n";
        }
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    d = tmp_path_factory.mktemp("s2_dir_xray_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: subprocess.check_output([exe], input=text, text=True).split("\n")


# ---- chunks ------------------------------------------------------------------------------------------------------------------
def chunks_py(counts, chunk, maxp):
    pieces, starts, used = [], [0], 0
    for k, c in enumerate(counts):
        first = 0
        while first < c:
            if used == chunk or len(pieces) - starts[-1] == maxp:
                starts.append(len(pieces))
                used = 0
            take = min(c - first, chunk - used)
            pieces.append((k, first, take))
            first += take
            used += take
    if len(pieces) > starts[-1]:
        starts.append(len(pieces))
    return starts, pieces


@pytest.mark.parametrize("seed", range(8))
def test_scan_chunks_cover_every_point_once(plan, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 200))
    counts = [int(v) for v in rng.integers(0, 5000, n)]
    counts[int(rng.integers(0, n))] = int(rng.integers(20000, 60000))  # a cell far larger than a chunk
    chunk, maxp = int(rng.integers(1, 9000)), int(rng.integers(1, 40))
    out = plan("chunks %d %d %d %s\n" % (n, chunk, maxp, " ".join(map(str, counts))))
    s = [int(v) for v in out[0].split()]
    p = [int(v) for v in out[1].split()]
    starts = s[1:]
    pieces = [(p[1 + 3 * i], p[2 + 3 * i], p[3 + 3 * i]) for i in range(p[0])]
    assert (starts, pieces) == chunks_py(counts, chunk, maxp)
    # every point of every cell exactly once, in order; every chunk within its bounds
    cover = {}
    for cell, first, cnt in pieces:
        assert cnt > 0 and first == cover.get(cell, 0)
        cover[cell] = first + cnt
    assert all(cover.get(k, 0) == c for k, c in enumerate(counts))
    for a, b in zip(starts, starts[1:]):
        assert 0 < b - a <= maxp and sum(x[2] for x in pieces[a:b]) <= chunk
    assert sum(1 for c in counts if c > chunk) == 0 or any(x[1] > 0 for x in pieces)  # some cell was cut


def test_scan_chunks_empty(plan):
    out = plan("chunks 3 100 10 0 0 0\n")
    assert out[0].split() == ["1", "0"] and out[1].split() == ["0"]


# ---- window bytes ------------------------------------------------------------------------------------------------------------
def window_bytes_py(points, cells, tiles, strategy, nfilt):
    fixed = 32 * tiles + 8 * cells + 4096  # s2_xray_fixed_bytes without the filters (the run holds them)
    return 24 * points + (3 * points if strategy == 1 else 0) + (4 * points if strategy == 2 or nfilt else 0) + 120 * cells + fixed


@pytest.mark.parametrize("strategy", [0, 1, 2, 3])
@pytest.mark.parametrize("nfilt", [0, 2])
def test_window_bytes(plan, strategy, nfilt):
    rng = np.random.default_rng(strategy * 10 + nfilt)
    for _ in range(20):
        pts, cells = int(rng.integers(0, 1 << 33)), int(rng.integers(1, 100000))
        tiles = cells + pts // 2048
        got = int(plan("bytes %d %d %d %d %d\n" % (pts, cells, tiles, strategy, nfilt))[0])
        assert got == window_bytes_py(pts, cells, tiles, strategy, nfilt)
    # XRay without filters: positions only
    assert int(plan("bytes 1000 1 1 0 0\n")[0]) == 24000 + 120 + 32 + 8 + 4096


# ---- block depth -------------------------------------------------------------------------------------------------------------
def dir_depth_py(budget, fixed, depth, gmax, leaf, tile, slice_bytes, w):
    for g in range(gmax, -1, -1):
        if w[g] != 2**64 - 1 and plan_py(budget, fixed + w[g], depth, g, leaf, tile, slice_bytes)[0] == g:
            return g
    return -1


def test_block_depth_under_a_budget_scan(plan):
    rng = np.random.default_rng(5)
    tile = 64 * 64 * 4
    leaf = tile + 8 * 5 + 400
    seen = set()
    for budget in [int(v) for v in np.geomspace(64 << 10, 1 << 30, 120)]:
        depth = int(rng.integers(0, 12))
        gmax = min(depth, 10)
        fixed = int(rng.integers(1 << 12, 1 << 16))
        # windows shrink as blocks get smaller; now and then one is too large to hold
        w = [int(budget * rng.uniform(0.01, 0.6) * 4.0 ** (g - gmax)) for g in range(gmax + 1)]
        if rng.random() < 0.2:
            w[int(rng.integers(0, gmax + 1))] = 2**64 - 1
        slice_bytes = 28 * 64 * 64 if rng.random() < 0.5 else 0
        got = int(plan("depth %d %d %d %d %d %d %d %s\n" % (budget, fixed, depth, gmax, leaf, tile, slice_bytes, " ".join(map(str, w))))[0])
        assert got == dir_depth_py(budget, fixed, depth, gmax, leaf, tile, slice_bytes, w), budget
        seen.add(got)
    assert -1 in seen and len(seen) >= 4


# ---- meta.pb: what load_s2_dir rejects, with its codes and messages ---------------------------------------------------------
def _varint(v):
    out = b""
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out += bytes([b | 0x80])
        else:
            return out + bytes([b])


def _key(f, w):
    return _varint((f << 3) | w)


def _bytes(f, b):
    return _key(f, 2) + _varint(len(b)) + b


def _meta(cells, version=13, attrs=(("color", 27), ("intensity", 11)), s2=True, box=((1.0, 2.0, 3.0), (4.0, 5.0, 6.0))):
    vec = lambda v: b"".join(_key(i + 1, 1) + struct.pack("<d", x) for i, x in enumerate(v))
    out = _key(1, 0) + _varint(version) + _bytes(4, _bytes(3, vec(box[0])) + _bytes(4, vec(box[1])))
    if s2:
        body = b"".join(_bytes(1, _key(1, 0) + _varint(i) + _key(2, 0) + _varint(n)) for i, n in cells)
        body += b"".join(_bytes(2, _bytes(1, name.encode()) + _key(2, 0) + _varint(t)) for name, t in attrs)
        out += _bytes(7, body)
    return out


def _token(cid):
    return ("%016x" % cid).rstrip("0") or "X"


L20 = [0x89C2590000000000 | (1 << 20), 0x89C25A0000000000 | (1 << 20), 0x1000000000000000 | (1 << 20)]  # three level-20 cells
BAD = 0x89C2590000000000 | (1 << 21)  # its lowest set bit is not a level's


def _open(plan, d):
    out = plan("open %s\n" % d)
    head = out[2].split()
    return int(out[0]), out[1], head


def test_meta_opener(plan, tmp_path):
    d = tmp_path / "ok"
    d.mkdir()
    (d / "meta.pb").write_bytes(_meta([(L20[0], 5), (L20[2], 7), (L20[1], 0)]))
    rc, err, head = _open(plan, d)
    assert rc == 0 and err == ""
    nc, n, level, rgb, inten = (int(v) for v in head[:5])
    assert (nc, n, level, rgb, inten) == (3, 12, 20, 1, 1)
    rows = [tuple(int(v) for v in head[5 + 3 * k: 8 + 3 * k]) for k in range(nc)]
    assert rows == [(L20[2], 7, 0), (L20[0], 5, 7), (L20[1], 0, 12)]  # id order, first slots


@pytest.mark.parametrize("case", ["missing", "version", "not_s2", "invalid_id", "twice", "attribute", "garbage"])
def test_meta_opener_rejects_as_load_s2_dir(plan, tmp_path, case):
    d = tmp_path / case
    d.mkdir()
    want = {
        "missing": (-3, "cannot read %s/meta.pb" % d),
        "version": (-1, "No S2 point cloud supported with version 11"),
        "not_s2": (-1, "This meta does not describe S2 point clouds"),
        "invalid_id": (-1, "invalid S2 cell id %x in meta.pb" % BAD),
        "twice": (-1, "cell %s is listed twice" % _token(L20[1])),
        "attribute": (-1, "unsupported attribute 'normal' (color: U8Vec3 and intensity: F32 are carried)"),
        "garbage": (-1, "Could not parse meta.pb"),
    }[case]
    if case != "missing":
        data = {
            "version": _meta([(L20[0], 1)], version=11),
            "not_s2": _meta([], s2=False),
            "invalid_id": _meta([(L20[1], 1), (BAD, 1)]),
            "twice": _meta([(L20[1], 1), (L20[0], 2), (L20[1], 3)]),
            "attribute": _meta([(L20[0], 1)], attrs=(("normal", 11),)),
            "garbage": _key(7, 2) + _varint(50) + b"\x01",
        }[case]
        (d / "meta.pb").write_bytes(data)
    rc, err, _ = _open(plan, d)
    assert (rc, err) == want
