"""Batched point queries that return their points, host side: the planning header (csrc/query_batch_points_plan.h, compiled here
with g++) - the sort key of a (location, node) pair orders pairs by location, then node index, within the bits the sort looks
at; the slabs cover the work list in order with at most kQbpSlabTiles tiles each; the offsets are the exclusive scan of the
counts; the scratch bound.  No GPU."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLAB_TILES = 1 << 18

HARNESS = r"""
#include <iostream>
#include "query_batch_points_plan.h"
using namespace pcv;
int main() {
    std::string what;
    while (std::cin >> what) {
        if (what == "consts") {
            std::cout << kQbpSlabTiles << " " << kQbpTileBytes << " " << kQbpPairBytes << " " << qbp_slab_bytes() << "\n";
        } else if (what == "bits") {  // bits <nloc> <nnodes>
            unsigned long long nl, nn;
            std::cin >> nl >> nn;
            const QbpKeyBits kb = qbp_key_bits(nl, nn);
            std::cout << kb.node_bits << " " << kb.end_bit << "\n";
        } else if (what == "key") {  // key <nloc> <nnodes> <loc> <node>
            unsigned long long nl, nn;
            uint32_t l, n;
            std::cin >> nl >> nn >> l >> n;
            std::cout << qbp_key(l, n, qbp_key_bits(nl, nn)) << "\n";
        } else if (what == "slabs") {  // slabs <ntiles> <slab_tiles>
            unsigned long long nt, st;
            std::cin >> nt >> st;
            const auto v = qbp_slabs(nt, st);
            std::cout << v.size();
            for (const auto& s : v) std::cout << " " << s.first << " " << s.n;
            std::cout << "\n";
        } else if (what == "offsets") {  // offsets <n> counts...
            uint32_t n;
            std::cin >> n;
            std::vector<uint64_t> c(n), off(n + 1);
            for (auto& v : c) std::cin >> v;
            const uint64_t t = qbp_offsets(c.data(), n, off.data());
            std::cout << t;
            for (auto v : off) std::cout << " " << v;
            std::cout << "\n";
        }
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    d = tmp_path_factory.mktemp("query_batch_points_plan")
    src, exe = d / "h.cpp", str(d / "h")
    src.write_text(HARNESS)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: subprocess.check_output([exe], input=text, text=True).split("\n")[:-1]


def test_constants_and_scratch_bound(run):
    slab, tile, pair, slab_bytes = map(int, run("consts")[0].split())
    assert slab == SLAB_TILES
    assert tile == 16 + 2048 // 8 + 4 + 4  # QTile, survivor mask, count, offset
    assert pair == 5 * 8
    assert slab_bytes == slab * tile == 73400320  # 70 MiB of slab scratch, whatever the batch
    assert slab * 2048 < 2 ** 32  # slab-local offsets fit in u32


@pytest.mark.parametrize("nloc,nn", [(1, 1), (2, 2), (3, 5), (1000, 4681), (65535, 1 << 20), (1 << 32, 1 << 32), (7, 1 << 31)])
def test_key_bits(run, nloc, nn):
    nb, end = map(int, run("bits %d %d" % (nloc, nn))[0].split())
    assert nb == max(1, (nn - 1).bit_length()) and end - nb == max(1, (nloc - 1).bit_length())
    assert end <= 64
    # the largest key sits inside the bits the sort looks at
    top = int(run("key %d %d %d %d" % (nloc, nn, nloc - 1, nn - 1))[0])
    assert top < 2 ** end


def test_keys_order_pairs_by_location_then_node(run):
    rng = np.random.default_rng(5)
    nloc, nn = 37, 1001
    pairs = [(int(l), int(n)) for l, n in zip(rng.integers(0, nloc, 300), rng.integers(0, nn, 300))]
    keys = [int(v) for v in run("".join("key %d %d %d %d\n" % (nloc, nn, l, n) for l, n in pairs))]
    assert [p for _, p in sorted(zip(keys, pairs))] == sorted(pairs)
    assert len(set(keys)) == len(set(pairs))


@pytest.mark.parametrize("ntiles,slab", [(0, SLAB_TILES), (1, SLAB_TILES), (SLAB_TILES, SLAB_TILES), (SLAB_TILES + 1, SLAB_TILES), (10, 3), (3 * SLAB_TILES + 17, SLAB_TILES)])
def test_slabs_cover_the_work_list_in_order(run, ntiles, slab):
    v = list(map(int, run("slabs %d %d" % (ntiles, slab))[0].split()))
    k, parts = v[0], list(zip(v[1::2], v[2::2]))
    assert k == len(parts) == -(-ntiles // slab)
    nxt = 0
    for first, n in parts:
        assert first == nxt and 0 < n <= slab
        nxt += n
    assert nxt == ntiles


def test_offsets(run):
    counts = [0, 5, 0, 0, 12, 1, 2 ** 40, 3]
    v = list(map(int, run("offsets %d %s" % (len(counts), " ".join(map(str, counts))))[0].split()))
    assert v[0] == sum(counts)
    assert v[1:] == [0] + list(np.cumsum(counts, dtype=np.uint64).astype(int))
    assert list(map(int, run("offsets 0")[0].split())) == [0, 0]
