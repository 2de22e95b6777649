"""Batched point queries that return their points straight from directories, host side: the planning header
(csrc/dir_query_batch_points_plan.h, with the chunk planner and the chunk tile order of csrc/dir_query_plan.h, compiled here with
g++).  Over random (location, node) pair sets - duplicate locations, locations flagged In, nodes without points, tiles without
survivors, nodes split across chunks by small chunk budgets - every work tile appears once, and its destination equals a brute-force
ordering of all tiles by (location, node, first point) with each location starting at its offset.  No GPU."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 2048
IN = 0x80000000

HARNESS = r"""
#include <algorithm>
#include <iostream>
#include "dir_query_batch_points_plan.h"
using namespace pcv;
// the survivors of a tile, a function of (location, node, first point) that both sides evaluate
static uint32_t survivors(uint32_t loc, uint32_t node, uint64_t first, uint32_t count) {
    const uint64_t h = (uint64_t)(loc & kDbpLocMask) * 7919u + (uint64_t)node * 104729u + (first / kDirTile) * 13u;
    return h % 5 == 0 ? 0u : (uint32_t)(h % (count + 1));
}
int main() {
    uint32_t nn, nloc, np;
    unsigned long long budget, tile_bytes;
    while (std::cin >> nn >> nloc >> budget >> tile_bytes) {
        std::vector<uint64_t> n(nn);
        std::vector<uint32_t> bpc(nn);
        for (uint32_t i = 0; i < nn; ++i) std::cin >> n[i] >> bpc[i];
        std::cin >> np;
        std::vector<std::pair<uint32_t, uint32_t>> pairs(np);  // (node, location): pairs_by_node's order
        for (auto& p : pairs) std::cin >> p.second >> p.first;
        std::sort(pairs.begin(), pairs.end());
        std::vector<uint32_t> visit, pair_loc;
        std::vector<uint64_t> pair_begin(nn + 1, 0);
        for (size_t j = 0; j < pairs.size(); ++j) {
            pair_loc.push_back(pairs[j].second);
            pair_begin[pairs[j].first + 1]++;
            if (j == 0 || pairs[j].first != pairs[j - 1].first) visit.push_back(pairs[j].first);
        }
        for (uint32_t i = 0; i < nn; ++i) pair_begin[i + 1] += pair_begin[i];
        auto info = [&](uint32_t i) { return DirPlanNode{n[i], bpc[i], (uint32_t)(pair_begin[i + 1] - pair_begin[i])}; };
        std::vector<DirChunk> chunks;
        if (!plan_dir_chunks(visit, info, true, false, budget, chunks, tile_bytes)) {
            std::cout << "refused\n";
            continue;
        }
        std::vector<uint32_t> cnt, tloc, tnode;
        std::vector<uint64_t> tfirst;
        std::vector<uint64_t> kept(nloc, 0);
        for (const DirChunk& ch : chunks)
            dir_chunk_tiles(ch, &pair_loc, &pair_begin, nullptr, [&](uint32_t k, uint32_t loc, uint32_t f, uint32_t c) {
                const DirPiece& pc = ch.pieces[k];
                const uint32_t s = survivors(loc, pc.node, pc.first + f, c);
                cnt.push_back(s), tloc.push_back(loc & kDbpLocMask), tnode.push_back(pc.node), tfirst.push_back(pc.first + f);
                kept[loc & kDbpLocMask] += s;
            });
        std::vector<uint64_t> off(nloc + 1, 0), dest(cnt.size(), ~0ull);
        for (uint32_t l = 0; l < nloc; ++l) off[l + 1] = off[l] + kept[l];
        const uint64_t nt = dbp_tile_dests(chunks, pair_loc, pair_begin, cnt.data(), off.data(), nloc, dest.data());
        uint64_t split = 0;
        for (size_t c = 1; c < chunks.size(); ++c) split += chunks[c].pieces.front().first != 0;
        std::cout << chunks.size() << " " << split << " " << nt << " " << dbp_work_tiles(visit, info) << " " << cnt.size() << "\n";
        for (size_t t = 0; t < cnt.size(); ++t) std::cout << tloc[t] << " " << tnode[t] << " " << tfirst[t] << " " << cnt[t] << " " << dest[t] << "\n";
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    d = tmp_path_factory.mktemp("dir_query_batch_points_plan")
    src, exe = d / "h.cpp", str(d / "h")
    src.write_text(HARNESS)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])

    def call(n, bpc, pairs, nloc, budget, tile_bytes=8):
        lines = ["%d %d %d %d" % (len(n), nloc, budget, tile_bytes), " ".join("%d %d" % (a, b) for a, b in zip(n, bpc)), str(len(pairs))]
        lines += ["%d %d" % p for p in pairs]
        out = subprocess.check_output([exe], input="\n".join(lines) + "\n", text=True).split("\n")
        if out[0] == "refused":
            return None
        nchunks, split, nt, work, ntiles = map(int, out[0].split())
        tiles = np.array([list(map(int, l.split())) for l in out[1: 1 + ntiles]], dtype=np.int64).reshape(-1, 5)
        return dict(chunks=nchunks, split=split, nt=nt, work=work, tiles=tiles)

    return call


def _survivors(loc, node, first, count):
    h = (loc & ~IN) * 7919 + node * 104729 + (first // TILE) * 13
    return 0 if h % 5 == 0 else h % (count + 1)


def _brute(n, pairs, nloc):
    """Every (location, node, tile) in (location, node, first) order, each location's survivors from its offset on."""
    tiles = []
    for loc, node in pairs:
        for f in range(0, n[node], TILE):
            c = min(TILE, n[node] - f)
            tiles.append(((loc & ~IN), node, f, _survivors(loc, node, f, c)))
    tiles.sort()
    kept = np.zeros(nloc, np.int64)
    for l, _, _, s in tiles:
        kept[l] += s
    off = np.concatenate([[0], np.cumsum(kept)])
    run, want = off[:-1].copy(), {}
    for l, node, f, s in tiles:
        want[(l, node, f)] = (s, int(run[l]))
        run[l] += s
    return want


def _check(got, n, pairs, nloc):
    want = _brute(n, pairs, nloc)
    assert got["nt"] == got["work"] == len(got["tiles"]) == len(want)
    seen = {}
    for l, node, f, s, dest in got["tiles"].tolist():
        assert (l, node, f) not in seen
        seen[(l, node, f)] = (s, dest)
    assert seen == want


def _random_case(rng, nn, nloc, density, max_pts):
    n = [int(v) for v in rng.integers(0, max_pts, nn)]
    for k in rng.choice(nn, nn // 6, replace=False):
        n[k] = 0  # nodes without points: no tiles
    bpc = [int(v) for v in rng.choice([1, 2, 4, 8], nn)]
    pairs = [(l | (IN if rng.random() < 0.2 else 0), node) for l in range(nloc) for node in range(nn) if rng.random() < density]
    return n, bpc, pairs


@pytest.mark.parametrize("seed", range(8))
def test_destinations_equal_the_brute_force_order(run, seed):
    rng = np.random.default_rng(seed)
    n, bpc, pairs = _random_case(rng, int(rng.integers(5, 40)), int(rng.integers(1, 12)), 0.4, 5 * TILE)
    nloc = 1 + max([p[0] & ~IN for p in pairs], default=0)
    for budget in (1 << 28, 1 << 20, 3 << 18):
        got = run(n, bpc, pairs, nloc, budget)
        assert got is not None
        _check(got, n, pairs, nloc)


def test_nodes_split_across_chunks_and_duplicate_locations(run):
    """Large nodes under a small budget: pieces of one node in consecutive chunks; locations 0 and 3 visit the same nodes."""
    rng = np.random.default_rng(11)
    n = [int(v) for v in rng.integers(TILE, 40 * TILE, 12)]
    bpc = [4] * 12
    nodes = sorted(rng.choice(12, 8, replace=False).tolist())
    pairs = [(0, k) for k in nodes] + [(1 | IN, k) for k in nodes[::2]] + [(2, k) for k in nodes[1::3]] + [(3, k) for k in nodes]
    got = run(n, bpc, pairs, 4, 1 << 20)
    assert got["chunks"] > 3 and got["split"] > 0
    _check(got, n, pairs, 4)
    seg = {}
    for l, node, f, s, dest in got["tiles"].tolist():
        seg.setdefault(l, []).append((node, f, s, dest))
    a, b = sorted(seg[0]), sorted(seg[3])
    assert [x[:2] for x in a] == [y[:2] for y in b]


def test_empty_pairs_and_no_survivors(run):
    got = run([100, 0, 5000], [2, 2, 2], [], 3, 1 << 28)
    assert got["nt"] == 0 and len(got["tiles"]) == 0 and got["chunks"] == 0
    got = run([0, 0], [8, 8], [(0, 0), (1, 1)], 2, 1 << 28)
    assert got["nt"] == 0


def test_destination_bytes_shrink_the_chunks(run):
    """The per-tile destination bytes count in the chunk budget: more chunks with them than without, the same destinations."""
    rng = np.random.default_rng(5)
    n, bpc, pairs = _random_case(rng, 30, 40, 0.9, 3 * TILE)
    with_d, without = run(n, bpc, pairs, 40, 1 << 20, 8), run(n, bpc, pairs, 40, 1 << 20, 0)
    assert with_d["chunks"] >= without["chunks"]
    _check(with_d, n, pairs, 40)
    _check(without, n, pairs, 40)
