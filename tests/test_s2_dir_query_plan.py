"""Point queries straight from an S2 directory, host side: the budget planning of csrc/s2_dir_query_plan.h (compiled here with
g++) against a Python restatement over random cell tables - open's least budget, the box scan's chunk, and the locations per
selection of a batch - and the scan's invariant that the chunks s2_scan_chunks cuts (cells larger than a chunk included) never
hold more work tiles than the chunk reserves, at every room the smallest budget open accepts leaves.  No GPU."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE, ALIGN = 2048, 256
CELL = 64 + 8 + 48  # kS2WindowCellBytes
PROJ, GEOM = 416, 4096  # any per-location sizes: the planner takes them as arguments

HARNESS = r"""
#include <iostream>
#include "s2_dir_query_plan.h"
using namespace pcv;
int main() {
    std::string what;
    while (std::cin >> what) {
        if (what == "open") {  // open <nc> <proj> <geom>
            unsigned long long nc, proj, geom;
            std::cin >> nc >> proj >> geom;
            std::cout << s2_dir_open_bytes(nc, proj, geom) << "\n";
        } else if (what == "scan") {  // scan <room>
            unsigned long long room;
            std::cin >> room;
            uint64_t chunk = 0, pieces = 0;
            const bool ok = s2_dir_scan_chunk(room, chunk, pieces);
            std::cout << ok << " " << chunk << " " << pieces << " " << s2_dir_scan_bytes(chunk, pieces) << "\n";
        } else if (what == "loc") {  // loc <nloc> <nc> <proj> <room>
            unsigned long long nloc, nc, proj, room;
            std::cin >> nloc >> nc >> proj >> room;
            std::cout << s2_dir_loc_chunk(nloc, nc, proj, room) << " " << s2_dir_select_bytes(1, nc, proj) << "\n";
        } else if (what == "tiles") {  // tiles <chunk> <pieces> <ncells> counts...: the most work tiles of any chunk
            unsigned long long chunk, pieces, nc;
            std::cin >> chunk >> pieces >> nc;
            std::vector<uint64_t> counts(nc);
            for (auto& c : counts) std::cin >> c;
            std::vector<S2Piece> pcs;
            const std::vector<size_t> st = s2_scan_chunks(counts, chunk, pieces, pcs);
            uint64_t most = 0, pts = 0;
            for (size_t k = 0; k + 1 < st.size(); ++k) {
                uint64_t t = 0;
                for (size_t j = st[k]; j < st[k + 1]; ++j) t += (pcs[j].count + kDirTile - 1) / kDirTile, pts += pcs[j].count;
                most = std::max(most, t);
            }
            std::cout << most << " " << pts << "\n";
        }
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("s2_dir_query_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: [l.split() for l in subprocess.check_output([exe], input=text, text=True).split("\n") if l]


# ---- Python restatement ---------------------------------------------------------------------------------------------------
def al(v, a):
    return (v + a - 1) // a * a


def min_chunk():  # dir_min_chunk_bytes: one tile at the widest encoding, with its survivors
    p, x = TILE, TILE * 24
    b = al(x + 32, ALIGN) + al(3 * p, ALIGN) + al(4 * p, ALIGN) + al(64, ALIGN) + al(8, ALIGN) + al(16, ALIGN) + al(4, ALIGN) + ALIGN
    return b + al(24 * p, ALIGN) + al(3 * p, ALIGN) + al(4 * p, ALIGN) + al(8 * p, ALIGN)


def select_bytes(nloc, nc, proj):
    return nloc * (proj + 8 + 8 * nc) + 36


def open_bytes(nc, proj, geom):
    return CELL * nc + select_bytes(1, nc, proj) + geom + 4096 + min_chunk()


def scan_bytes(chunk, pieces):
    return 24 * chunk + pieces * 68 + (pieces + chunk // TILE + 1) * 16


def scan_chunk(room):
    chunk = (64 << 20) // 24
    while True:
        pieces = max(64, chunk // 64)
        if scan_bytes(chunk, pieces) <= room:
            return True, chunk, pieces
        if chunk <= TILE:
            return False, chunk, pieces
        chunk = max(TILE, chunk // 2)


def loc_chunk(nloc, nc, proj, room):
    per = proj + 8 + 8 * nc
    if room < 36 + per:
        return 0
    return min(nloc, (room - 36) // per, 65535, max(1, (1 << 25) // max(nc, 1)))


def test_open_bytes(harness):
    rng = np.random.default_rng(5)
    cases = [(0, PROJ, GEOM), (1, PROJ, GEOM)] + [(int(rng.integers(0, 1 << 24)), int(rng.integers(1, 2000)), int(rng.integers(1, 9000))) for _ in range(200)]
    out = harness("".join("open %d %d %d\n" % c for c in cases))
    for c, o in zip(cases, out):
        assert int(o[0]) == open_bytes(*c), c


def test_scan_chunk(harness):
    rng = np.random.default_rng(6)
    rooms = [0, 1, scan_bytes(TILE, 64) - 1, scan_bytes(TILE, 64), 1 << 40] + [int(v) for v in np.exp(rng.uniform(np.log(1e4), np.log(1e10), 300))]
    out = harness("".join("scan %d\n" % r for r in rooms))
    for r, o in zip(rooms, out):
        ok, chunk, pieces, b = int(o[0]), int(o[1]), int(o[2]), int(o[3])
        assert (bool(ok), chunk, pieces) == scan_chunk(r), r
        assert b == scan_bytes(chunk, pieces)
        if ok:
            assert b <= r and chunk >= TILE and pieces >= 64
            assert chunk == (64 << 20) // 24 or scan_bytes(min(2 * chunk, (64 << 20) // 24), max(64, min(2 * chunk, (64 << 20) // 24) // 64)) > r


def test_loc_chunk(harness):
    rng = np.random.default_rng(7)
    cases = [(1, 1, PROJ, 0), (2000, 5000, PROJ, select_bytes(1, 5000, PROJ)), (2000, 5000, PROJ, select_bytes(1, 5000, PROJ) - 1), (70000, 1, PROJ, 1 << 40)]
    for _ in range(300):
        nc = int(rng.integers(1, 1 << 22))
        cases.append((int(rng.integers(1, 100000)), nc, PROJ, int(rng.integers(0, 1 << 33))))
    out = harness("".join("loc %d %d %d %d\n" % c for c in cases))
    for c, o in zip(cases, out):
        m = int(o[0])
        assert m == loc_chunk(*c), c
        nloc, nc, proj, room = c
        if m:
            assert select_bytes(m, nc, proj) <= room and m <= min(nloc, 65535)
        else:
            assert select_bytes(1, nc, proj) > room


def test_scan_fits_smallest_budget(harness):
    """At the smallest budget open accepts, the first polyhedral call has the room open reserved beyond the cell table; the scan's
    chunk fits it, and no chunk s2_scan_chunks cuts holds more tiles than the chunk reserves - cells larger than a chunk, cells
    of one point and empty cells included."""
    rng = np.random.default_rng(8)
    text, want = "", []
    for trial in range(40):
        nc = int(rng.integers(1, 3000))
        kind = trial % 4
        counts = rng.integers(0, 5, nc) if kind == 0 else rng.integers(1, 3 * TILE, nc) if kind == 1 else rng.integers(0, 200000, nc)
        if kind == 3:
            counts[rng.integers(0, nc, 3)] = 3_000_000  # larger than any chunk at this budget
        room = open_bytes(nc, PROJ, GEOM) - CELL * nc
        ok, chunk, pieces = scan_chunk(room)
        assert ok and scan_bytes(chunk, pieces) <= room
        text += "tiles %d %d %d %s\n" % (chunk, pieces, nc, " ".join(str(int(c)) for c in counts))
        want.append((chunk, pieces, int(counts.sum())))
    for (chunk, pieces, total), o in zip(want, harness(text)):
        most, pts = int(o[0]), int(o[1])
        assert pts == total
        assert most <= pieces + chunk // TILE + 1
