"""Point queries straight from an octree directory, host side: the chunk planner (csrc/dir_query_plan.h, compiled here with g++)
against a Python restatement and its invariants over random visit lists, the host /nodes_data formatter against the oracle's
blob over a directory the oracle wrote, and the pcv_dir_query_stats layout.  No GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_api as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE, ALIGN = 2048, 256

HARNESS = r"""
#include <cstdio>
#include <iostream>
#include "dir_query_plan.h"
#include "xray_dir_plan.h"
using namespace pcv;
int main() {
    std::string what;
    std::cin >> what;
    if (what == "min") {
        std::cout << dir_min_chunk_bytes() << "\n";
        return 0;
    }
    if (what == "plan") {  // plan <has_i> <store> <budget> <nvisit> then (node n bpc mult) per visited node
        int has_i, store; unsigned long long budget; size_t nv;
        std::cin >> has_i >> store >> budget >> nv;
        std::vector<uint32_t> visit(nv);
        std::vector<DirPlanNode> info(nv);
        for (size_t k = 0; k < nv; ++k) std::cin >> visit[k] >> info[k].n >> info[k].bpc >> info[k].mult;
        std::vector<DirChunk> ch;
        const bool ok = plan_dir_chunks(visit, [&](uint32_t v) { return info[std::find(visit.begin(), visit.end(), v) - visit.begin()]; }, has_i, store, budget, ch);
        if (!ok) { std::cout << "fail\n"; return 0; }
        std::cout << ch.size() << "\n";
        for (const auto& c : ch) {
            std::cout << c.pieces.size() << " " << c.points << " " << c.xyz_bytes << " " << c.tiles << " "
                      << dir_chunk_bytes(c.points, c.xyz_bytes, c.pieces.size(), c.tiles, has_i, store);
            for (const auto& p : c.pieces) std::cout << " " << p.node << " " << p.first << " " << p.count;
            std::cout << "\n";
        }
        return 0;
    }
    // blob <dir> <out> <k> then k (hi lo): the reply laid out by nodes_blob_layout / nodes_blob_header, files read with stdio
    std::string dir, outp; uint32_t k;
    std::cin >> dir >> outp >> k;
    std::vector<uint64_t> ids(2 * k);
    for (auto& v : ids) std::cin >> v;
    std::string buf;
    read_whole_file(dir + "/meta.pb", buf);
    MetaHeader h; std::vector<ParsedNode> pn; int version = 0;
    decode_meta(buf, h, pn, version);
    double bmin[3], bmax[3]; std::vector<pcv_node_meta> nodes; uint64_t np = 0, xb = 0;
    octree_nodes_from_meta(h, pn, bmin, bmax, nodes, np, xb);
    std::vector<BlobPart> parts; uint64_t size = 0;
    const int64_t bad = nodes_blob_layout(nodes, ids.data(), k, parts, size);
    if (bad >= 0) { std::cout << "bad " << bad << "\n"; return 0; }
    std::vector<uint8_t> out(size, 0);
    for (const auto& p : parts) {
        nodes_blob_header(nodes[p.node], out.data() + p.header_at);
        const std::string s = dir + "/" + node_name(nodes[p.node].id_high, nodes[p.node].id_low);
        std::string f;
        read_whole_file(s + ".xyz", f);
        std::copy(f.begin(), f.end(), out.begin() + p.xyz_at);
        read_whole_file(s + ".rgb", f);
        std::copy(f.begin(), f.end(), out.begin() + p.rgb_at);
    }
    FILE* fo = fopen(outp.c_str(), "wb");
    fwrite(out.data(), 1, out.size(), fo);
    fclose(fo);
    std::cout << "ok " << size << "\n";
    return 0;
}
"""


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("dir_query_plan")
    src = d / "plan.cpp"
    src.write_text(HARNESS)
    exe = str(d / "plan")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", exe, str(src)])
    return lambda text: subprocess.check_output([exe], input=text, text=True).split("\n")


# ---- Python restatement ---------------------------------------------------------------------------------------------------
def al(v, a):
    return (v + a - 1) // a * a


def chunk_bytes(points, xyz, pieces, tiles, has_i, store):
    b = al(xyz + 32, ALIGN) + al(3 * points, ALIGN) + (al(4 * points, ALIGN) if has_i else 0)
    b += al(64 * pieces, ALIGN) + al(8 * pieces, ALIGN) + al(16 * tiles, ALIGN) + al(4 * tiles, ALIGN) + ALIGN
    if store:
        b += al(24 * points, ALIGN) + al(3 * points, ALIGN) + al(4 * points, ALIGN) + al(8 * points, ALIGN)
    return b


def plan_py(visit, has_i, store, budget):
    out, cur = [], dict(pieces=[], points=0, xyz=0, tiles=0)

    def cost(c, bpc, mult, cnt):
        return chunk_bytes(c["points"] + cnt, c["xyz"] + al(cnt * 3 * bpc, 16), len(c["pieces"]) + 1, c["tiles"] + -(-cnt // TILE) * mult, has_i, store)

    for node, n, bpc, mult in visit:
        first = 0
        while first < n:
            left = n - first
            t = 0  # the most whole tiles that fit, by linear search
            while t < -(-left // TILE) and cost(cur, bpc, mult, min(left, (t + 1) * TILE)) <= budget:
                t += 1
            if t == 0:
                if not cur["pieces"]:
                    return None
                out.append(cur)
                cur = dict(pieces=[], points=0, xyz=0, tiles=0)
                continue
            cnt = min(left, t * TILE)
            cur["pieces"].append((node, first, cnt))
            cur["points"] += cnt
            cur["xyz"] += al(cnt * 3 * bpc, 16)
            cur["tiles"] += -(-cnt // TILE) * mult
            first += cnt
    if cur["pieces"]:
        out.append(cur)
    return out


def run_plan(harness, visit, has_i, store, budget):
    text = "plan %d %d %d %d\n" % (has_i, store, budget, len(visit)) + "".join("%d %d %d %d\n" % v for v in visit)
    lines = [l for l in harness(text) if l]
    if lines[0] == "fail":
        return None
    chunks = []
    for l in lines[1:]:
        v = [int(t) for t in l.split()]
        chunks.append(dict(npieces=v[0], points=v[1], xyz=v[2], tiles=v[3], bytes=v[4], pieces=[tuple(v[5 + 3 * k: 8 + 3 * k]) for k in range(v[0])]))
    assert len(chunks) == int(lines[0])
    return chunks


def random_visit(rng):
    nodes = sorted(rng.choice(100000, int(rng.integers(1, 60)), replace=False))
    out = []
    for v in nodes:
        r = rng.random()
        n = int(rng.integers(1, 40)) if r < 0.3 else int(rng.integers(1, 30000)) if r < 0.9 else int(rng.integers(30000, 400000))
        out.append((int(v), n, int(rng.choice([1, 2, 4, 8])), int(rng.integers(1, 5)) if rng.random() < 0.5 else 1))
    return out


def test_min_chunk(harness):
    assert int(harness("min\n")[0]) == chunk_bytes(TILE, TILE * 24, 1, 1, True, True)


@pytest.mark.parametrize("seed", range(12))
def test_planner_against_restatement_and_invariants(harness, seed):
    rng = np.random.default_rng(seed)
    visit = random_visit(rng)
    has_i, store = bool(seed % 2), seed % 3 != 0
    if store:
        visit = [(v, n, b, 1) for v, n, b, _ in visit]  # the single-location form
    total = sum(n for _, n, _, _ in visit)
    mn = chunk_bytes(TILE, TILE * 24, 1, 1, True, True)
    split_seen = False
    for budget in [int(b) for b in np.geomspace(mn // 4, 40 * mn, 9)] + [mn]:
        got = run_plan(harness, visit, has_i, store, budget)
        want = plan_py(visit, has_i, store, budget)
        if want is None:
            assert got is None, budget
            assert budget < mn or any(m > 1 for _, _, _, m in visit)
            continue
        assert got is not None and len(got) == len(want), budget
        for g, w in zip(got, want):
            assert g["pieces"] == w["pieces"] and (g["points"], g["xyz"], g["tiles"]) == (w["points"], w["xyz"], w["tiles"])
            # the byte bound, intensity counted when present
            assert g["bytes"] == chunk_bytes(w["points"], w["xyz"], len(w["pieces"]), w["tiles"], has_i, store) <= budget
        # every visited point in exactly one piece, pieces in visit order, pieces start at tile multiples
        pieces = [p for c in got for p in c["pieces"]]
        at = {}
        order = []
        for node, first, cnt in pieces:
            assert first == at.get(node, 0) and cnt > 0
            assert first % TILE == 0
            at[node] = first + cnt
            if not order or order[-1] != node:
                order.append(node)
        assert order == [v for v, _, _, _ in visit]
        assert all(at[v] == n for v, n, _, _ in visit) and sum(c["points"] for c in got) == total
        # a node larger than what a chunk holds is split, at tile boundaries
        for v, n, b, m in visit:
            mine = [p for p in pieces if p[0] == v]
            if chunk_bytes(n, al(n * 3 * b, 16), 1, -(-n // TILE) * m, has_i, store) > budget:
                assert len(mine) > 1
                split_seen = True
            assert all(cnt % TILE == 0 for _, _, cnt in mine[:-1])
    assert split_seen or total < 2 * TILE


def test_budget_below_min_chunk_is_rejected(harness):
    mn = chunk_bytes(TILE, TILE * 24, 1, 1, True, True)
    visit = [(0, 5 * TILE, 8, 1)]
    assert run_plan(harness, visit, True, True, mn - 1) is None
    got = run_plan(harness, visit, True, True, mn)
    assert got is not None and [c["points"] for c in got] == [TILE] * 5


def test_nodes_blob_matches_oracle(harness, tmp_path):
    rng = np.random.default_rng(7)
    n = 20000
    x, y, z = rng.uniform(0, 50, n), rng.uniform(0, 50, n), rng.uniform(0, 5, n)
    x[:5000] = 10.0 + rng.integers(0, 3, 5000)  # dense columns: nodes at several levels and encodings
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    ref = O.build(x, y, z, rgb, 1.0 / 512, (0.0, 0.0, 0.0), (50.0, 50.0, 5.0), max_points_per_node=500)
    d = str(tmp_path / "oct")
    os.makedirs(d)
    ref.write_dir(d)
    names = [nm for nm in ref.order if ref.nodes[nm]["num_points"] > 0]
    assert len(names) > 10
    pick = [names[i] for i in rng.permutation(len(names))[:40]] + names[:3]
    ids = [v for nm in pick for v in O.id_from_str(nm)]
    outp = str(tmp_path / "blob.bin")
    res = harness("blob %s %s %d %s\n" % (d, outp, len(pick), " ".join(str(int(v)) for v in ids)))[0].split()
    assert res[0] == "ok"
    got = open(outp, "rb").read()
    assert got == ref.nodes_data_blob(pick) and len(got) == int(res[1])
    # an unknown id is reported with its position in the request
    bad = pick[:2] + ["r" + "7" * 12]
    ids = [v for nm in bad for v in O.id_from_str(nm)]
    assert harness("blob %s %s %d %s\n" % (d, outp, 3, " ".join(str(int(v)) for v in ids)))[0] == "bad 2"


def test_dir_query_stats_struct_matches_the_c_compiler(tmp_path):
    """pcv_dir_query_stats: ctypes size and field offsets equal gcc's for include/pcv.h."""
    from point_cloud_viewer_b200 import _native as N

    fs = [f for f, _ in N.DirQueryStats._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "pcv.h"', "int main(void) {", 'printf("size %zu\\n", sizeof(pcv_dir_query_stats));']
    for f in fs:
        src.append('printf("%s %%zu\\n", offsetof(pcv_dir_query_stats, %s));' % (f, f))
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, str(c)])
    got = dict(l.split() for l in subprocess.check_output([exe], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(N.DirQueryStats)
    for f in fs:
        assert int(got[f]) == getattr(N.DirQueryStats, f).offset, f
