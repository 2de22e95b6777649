"""Merging partial X-ray quadtrees, host side (csrc/xray_png.hpp, csrc/xray_merge_plan.h, compiled here with g++): the PNG reader
against Pillow and hand-built PNGs, the meta decoder against python-protobuf, and the merge planner against a Python
restatement of validate_and_merge_metadata, Node::parent and create_non_leaf_nodes (tests/xray_merge_ref.py).  No GPU."""
import io
import math
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest
from PIL import Image

from proto_meta import XrayMeta
from xray_merge_ref import Meta as M, plan as plan_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, INVALID, NOT_FOUND, UNSUPPORTED = 0, -1, -4, -6

HARNESS = r"""
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include "xray_merge_plan.h"
using namespace pcv;
int main(int argc, char** argv) {
    const std::string what = argv[1];
    if (what == "png") {  // png <in> <out>: "code w h why", the pixels into <out>
        std::string f;
        read_whole_file(argv[2], f);
        uint32_t w = 0, h = 0;
        std::vector<uint8_t> px;
        std::string why;
        const int rc = decode_png_rgba(f, w, h, px, &why);
        printf("%d %u %u %s\n", rc, w, h, why.c_str());
        if (rc == 0) write_whole_file(argv[3], px.data(), px.size());
    } else if (what == "encode") {  // encode <w> <h> <rgba in> <png out>
        std::string px;
        read_whole_file(argv[4], px);
        std::string png;
        encode_png_rgba((const uint8_t*)px.data(), (uint32_t)atoi(argv[2]), (uint32_t)atoi(argv[3]), png);
        write_whole_file(argv[5], png.data(), png.size());
    } else if (what == "meta") {  // meta <in>: "ok version min_x min_y edge deepest tile n level index ..."
        std::string f;
        read_whole_file(argv[2], f);
        XrayMetaData m;
        int version = 0;
        const bool ok = decode_xray_meta(f, m, version);
        printf("%d %d %a %a %a %u %u %zu", ok ? 1 : 0, version, m.min_x, m.min_y, m.edge, m.deepest_level, m.tile_size, m.nodes.size());
        for (const auto& n : m.nodes) printf(" %u %llu", n.first, (unsigned long long)n.second);
        printf("\n");
    } else if (what == "plan") {  // stdin: n, then per meta "deepest tile min_x min_y edge nnodes (level index)*"
        size_t n;
        std::cin >> n;
        std::vector<XrayMetaData> metas(n);
        for (auto& m : metas) {
            std::string x, y, e;
            size_t k;
            std::cin >> m.deepest_level >> m.tile_size >> x >> y >> e >> k;
            m.min_x = strtod(x.c_str(), nullptr), m.min_y = strtod(y.c_str(), nullptr), m.edge = strtod(e.c_str(), nullptr);
            m.nodes.resize(k);
            for (auto& nd : m.nodes) std::cin >> nd.first >> nd.second;
        }
        const XrayMergePlan p = xray_merge_plan(metas);
        printf("%d %u %u %s\n", p.code, p.metas, p.empty, p.error.c_str());
        if (p.code) return 0;
        printf("%u %u %u %a %a %a\n%zu", p.root_level, p.deepest_level, p.tile_size, p.rect.min_x, p.rect.min_y, p.rect.edge, p.roots.size());
        for (size_t i = 0; i < p.roots.size(); ++i) printf(" %llu %zu", (unsigned long long)p.roots[i], p.root_meta[i]);
        printf("\n%zu", p.walk.size());
        for (const auto& w : p.walk) printf(" %u %llu", w.first, (unsigned long long)w.second);
        printf("\n%zu", p.nodes.size());
        for (const auto& w : p.nodes) printf(" %u %llu", w.first, (unsigned long long)w.second);
        printf("\n");
    } else if (what == "bytes") {  // bytes <L> <T>
        printf("%llu\n", (unsigned long long)xray_merge_device_bytes((uint32_t)atoi(argv[2]), (uint32_t)atoi(argv[3])));
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("xray_merge_host")
    src = d / "merge.cpp"
    src.write_text(HARNESS)
    out = str(d / "merge")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "point_cloud_viewer_b200", "csrc"), "-o", out, str(src), "-lz"])
    return out


def _run(exe, *args, stdin=None):
    return subprocess.check_output([exe] + [str(a) for a in args], input=stdin, text=True)


# ---- PNG reader ------------------------------------------------------------------------------------------------------------

def _decode(exe, tmp_path, png_bytes):
    p = tmp_path / "in.png"
    p.write_bytes(png_bytes)
    o = tmp_path / "out.rgba"
    if o.exists():
        o.unlink()
    head = _run(exe, "png", p, o).split(" ", 3)
    code, w, h = int(head[0]), int(head[1]), int(head[2])
    px = np.frombuffer(o.read_bytes(), np.uint8).reshape(h, w, 4) if code == 0 else None
    return code, px


def _chunk(t, data):
    return struct.pack(">I", len(data)) + t + data + struct.pack(">I", zlib.crc32(t + data) & 0xFFFFFFFF)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def _filter_row(f, row, prev, bpp=4):
    row = row.astype(np.int32)
    prev = prev.astype(np.int32) if prev is not None else np.zeros_like(row)
    out = np.zeros_like(row)
    for i in range(len(row)):
        a = row[i - bpp] if i >= bpp else 0
        b = prev[i]
        c = prev[i - bpp] if i >= bpp else 0
        pred = [0, a, b, (a + b) >> 1, _paeth(a, b, c)][f]
        out[i] = (row[i] - pred) & 0xFF
    return bytes([f]) + out.astype(np.uint8).tobytes()


def _png(px, filters=None, idat_splits=1, color_type=6, bit_depth=8, interlace=0, raw=None, extra_chunks=()):
    h, w = px.shape[:2]
    if raw is None:
        rows = []
        flat = px.reshape(h, -1)
        for y in range(h):
            rows.append(_filter_row(filters[y % len(filters)] if filters else 0, flat[y], flat[y - 1] if y else None))
        raw = b"".join(rows)
    z = zlib.compress(raw, 6)
    ihdr = struct.pack(">IIBBBBB", w, h, bit_depth, color_type, 0, 0, interlace)
    out = b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", ihdr)
    for c in extra_chunks:
        out += c
    step = max(1, math.ceil(len(z) / idat_splits))
    for i in range(0, len(z), step):
        out += _chunk(b"IDAT", z[i:i + step])
    return out + _chunk(b"IEND", b"")


def test_png_equals_pillow_on_this_projects_tiles(exe, tmp_path):
    rng = np.random.default_rng(1)
    for w, h in ((1, 1), (7, 3), (256, 256)):
        px = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        px[: h // 2, :, 3] = 0  # a background region, as X-ray tiles have
        raw = tmp_path / "px.rgba"
        raw.write_bytes(px.tobytes())
        png = tmp_path / "tile.png"
        _run(exe, "encode", w, h, raw, png)
        code, got = _decode(exe, tmp_path, png.read_bytes())
        assert code == OK
        ref = np.asarray(Image.open(png).convert("RGBA"))
        assert np.array_equal(got, ref) and np.array_equal(got, px)


def test_png_all_filter_types_and_split_idat(exe, tmp_path):
    rng = np.random.default_rng(2)
    px = rng.integers(0, 256, (23, 17, 4), dtype=np.uint8)
    px[5:9] = px[4]  # repeated rows: Up filters to zero
    for filters, splits in (([0], 1), ([1], 3), ([2], 2), ([3], 5), ([4], 1), ([0, 1, 2, 3, 4], 7), ([4, 3, 2, 1, 0], 64)):
        data = _png(px, filters, splits, extra_chunks=[_chunk(b"gAMA", struct.pack(">I", 45455)), _chunk(b"tEXt", b"Software\x00test")])
        code, got = _decode(exe, tmp_path, data)
        assert code == OK, (filters, splits)
        assert np.array_equal(got, px), (filters, splits)
        assert np.array_equal(np.asarray(Image.open(io.BytesIO(data)).convert("RGBA")), px)


def test_png_pillow_written_files(exe, tmp_path):
    rng = np.random.default_rng(3)
    px = rng.integers(0, 256, (64, 64, 4), dtype=np.uint8)
    px[10:30, 10:30] = (255, 255, 255, 255)
    for opt in ({}, {"optimize": True}, {"compress_level": 1}):
        buf = io.BytesIO()
        Image.fromarray(px, "RGBA").save(buf, "PNG", **opt)
        code, got = _decode(exe, tmp_path, buf.getvalue())
        assert code == OK and np.array_equal(got, px)


def test_png_rejects(exe, tmp_path):
    px = np.zeros((4, 4, 4), np.uint8)
    good = _png(px, [0])
    assert _decode(exe, tmp_path, good)[0] == OK
    h, w = 4, 4
    cases = {
        "16-bit": (_png(px, raw=b"".join(b"\x00" + bytes(w * 8) for _ in range(h)), bit_depth=16), UNSUPPORTED),
        "palette": (_png(px, raw=b"".join(b"\x00" + bytes(w) for _ in range(h)), color_type=3), UNSUPPORTED),
        "rgb": (_png(px, raw=b"".join(b"\x00" + bytes(w * 3) for _ in range(h)), color_type=2), UNSUPPORTED),
        "grey": (_png(px, raw=b"".join(b"\x00" + bytes(w) for _ in range(h)), color_type=0), UNSUPPORTED),
        "interlaced": (_png(px, [0], interlace=1), UNSUPPORTED),
    }
    bad_crc = bytearray(good)
    bad_crc[8 + 8 + 13] ^= 1  # IHDR's CRC
    cases["bad crc"] = (bytes(bad_crc), INVALID)
    bad_idat_crc = bytearray(good)
    idat = good.index(b"IDAT")
    bad_idat_crc[idat + 4] ^= 0x40  # first byte of the zlib stream; the CRC no longer matches
    cases["bad idat crc"] = (bytes(bad_idat_crc), INVALID)
    z = zlib.compress(b"".join(b"\x00" + bytes(w * 4) for _ in range(h)))
    trunc = b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 6, 0, 0, 0)) + _chunk(b"IDAT", z[:-6]) + _chunk(b"IEND", b"")
    cases["truncated stream"] = (trunc, INVALID)
    short = zlib.compress(b"".join(b"\x00" + bytes(w * 4) for _ in range(h - 1)))
    cases["short stream"] = (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 6, 0, 0, 0)) + _chunk(b"IDAT", short) + _chunk(b"IEND", b""),
                             INVALID)
    cases["truncated file"] = (good[:-20], INVALID)
    cases["bad filter type"] = (_png(px, raw=b"".join(b"\x05" + bytes(w * 4) for _ in range(h))), INVALID)
    cases["not a png"] = (b"GIF89a" + bytes(40), INVALID)
    for name, (data, want) in cases.items():
        assert _decode(exe, tmp_path, data)[0] == want, name


# ---- meta decoder ----------------------------------------------------------------------------------------------------------

def _meta(exe, tmp_path, data):
    p = tmp_path / "meta.pb"
    p.write_bytes(data)
    f = _run(exe, "meta", p).split()
    nodes = [(int(f[8 + 2 * i]), int(f[9 + 2 * i])) for i in range(int(f[7]))]
    return int(f[0]), int(f[1]), float.fromhex(f[2]), float.fromhex(f[3]), float.fromhex(f[4]), int(f[5]), int(f[6]), nodes


def test_meta_v3_and_v2_equal_protobuf(exe, tmp_path):
    rng = np.random.default_rng(4)
    for trial in range(20):
        m = XrayMeta()
        v2 = trial % 2 == 1
        m.version = 2 if v2 else 3
        if v2:
            m.bounding_rect.deprecated_min.x = float(rng.normal() * 1e4)
            m.bounding_rect.deprecated_min.y = float(rng.normal() * 1e4)
            m.bounding_rect.deprecated_edge_length = float(rng.uniform(1, 1e5))
        else:
            m.bounding_rect.min.x = float(rng.normal() * 1e6)
            m.bounding_rect.min.y = float(rng.normal() * 1e6)
            m.bounding_rect.edge_length = float(rng.uniform(1, 1e7))
        m.deepest_level = int(rng.integers(0, 20))
        m.tile_size = int(rng.choice([256, 512, 4096]))
        for _ in range(int(rng.integers(0, 30))):
            n = m.nodes.add()
            n.level = int(rng.integers(0, 20))
            n.index = int(rng.integers(0, 4 ** n.level))
        ok, version, x, y, e, deepest, tile, nodes = _meta(exe, tmp_path, m.SerializeToString())
        back = XrayMeta.FromString(m.SerializeToString())
        rect = back.bounding_rect
        want = (rect.deprecated_min.x, rect.deprecated_min.y, rect.deprecated_edge_length) if v2 else (rect.min.x, rect.min.y, rect.edge_length)
        assert ok == 1 and version == m.version
        assert (x, y, e) == want  # f32 fields widened to f64 exactly
        assert (deepest, tile) == (m.deepest_level, m.tile_size)
        assert nodes == [(n.level, n.index) for n in back.nodes]


def test_meta_rejects_other_versions_and_truncation(exe, tmp_path):
    m = XrayMeta()
    m.bounding_rect.min.x = 1.5
    m.bounding_rect.edge_length = 8.0
    m.deepest_level = 3
    m.tile_size = 256
    n = m.nodes.add()
    n.level, n.index = 2, 7
    for v in (1, 4, 0):
        m.version = v
        assert _meta(exe, tmp_path, m.SerializeToString())[0] == 0, v
    m.version = 3
    data = m.SerializeToString()
    assert _meta(exe, tmp_path, data)[0] == 1
    for cut in range(1, len(data)):
        ok = _meta(exe, tmp_path, data[:cut])[0]
        try:  # a prefix protobuf itself parses can still be a valid message (a field boundary)
            XrayMeta.FromString(data[:cut])
            parses = True
        except Exception:
            parses = False
        if not parses:
            assert ok == 0, cut


# ---- planner ---------------------------------------------------------------------------------------------------------------

def plan_cpp(exe, metas):
    lines = [str(len(metas))]
    for m in metas:
        lines.append("%d %d %s %s %s %d %s" % (m.deepest, m.tile, m.rect[0].hex(), m.rect[1].hex(), m.rect[2].hex(), len(m.nodes),
                                               " ".join("%d %d" % n for n in m.nodes)))
    out = _run(exe, "plan", stdin="\n".join(lines) + "\n").split("\n")
    head = out[0].split(" ", 3)
    code = int(head[0])
    if code:
        return code, head[3], int(head[1]), int(head[2])
    L, deepest, tile, x, y, e = out[1].split()
    r = [int(v) for v in out[2].split()]
    roots = [(int(L), r[1 + 2 * i]) for i in range(r[0])]
    w = [int(v) for v in out[3].split()]
    walk = [(w[1 + 2 * i], w[2 + 2 * i]) for i in range(w[0])]
    n = [int(v) for v in out[4].split()]
    nodes = [(n[1 + 2 * i], n[2 + 2 * i]) for i in range(n[0])]
    return OK, (int(L), int(deepest), int(tile), (float.fromhex(x), float.fromhex(y), float.fromhex(e)), roots, walk, nodes), int(head[1]), int(head[2])


def _subtree(level, index, deepest):
    out = [(level, index)]
    for l in range(level + 1, min(deepest, level + 2) + 1):
        out += [(l, (index << (2 * (l - level))) + k) for k in range(4 ** (l - level)) if k % 3 != 1]
    return out


def test_validation_errors_in_the_references_order(exe):
    a, b, c = _subtree(2, 5, 6), _subtree(2, 6, 6), _subtree(1, 1, 6)
    cases = [
        ([], NOT_FOUND, "No subquadtrees meta files found."),
        ([M([]), M([], deepest=5, tile=512)], INVALID, "All subquadtress are empty."),
        ([M(a), M(a), M(c), M(b, deepest=7)], INVALID, "Not all roots are unique."),
        ([M(a), M(c), M(b, deepest=7, tile=512)], INVALID, "Not all roots have the same level."),
        ([M(a), M(b, tile=512), M([], deepest=7)], INVALID, "Not all meta files have the same deepest level."),
        ([M(a), M(b), M([], tile=512)], INVALID, "Not all meta files have the same tile size."),
    ]
    for metas, code, msg in cases:
        assert plan_py(metas) == (code, msg)
        got = plan_cpp(exe, metas)
        assert got[:2] == (code, msg), msg
        assert got[2] == len(metas) and got[3] == sum(1 for m in metas if not m.nodes)
    # beyond the reference: roots outside their level, levels a NodeId cannot hold, tiles of 0 px
    assert plan_cpp(exe, [M([(1, 4)])])[0] == INVALID
    assert plan_cpp(exe, [M([(3, 1)], deepest=40)])[0] == UNSUPPORTED
    assert plan_cpp(exe, [M([(1, 1)], tile=0)])[0] == UNSUPPORTED


def test_rect_walk_bits_on_random_non_dyadic_rects(exe):
    rng = np.random.default_rng(5)
    for _ in range(200):
        L = int(rng.integers(0, 25))
        idx = int(rng.integers(0, 4 ** L)) if L else 0
        rect = (float(rng.normal() * 10 ** rng.uniform(0, 7)), float(rng.normal() * 10 ** rng.uniform(0, 7)), float(rng.uniform(0.001, 1e4)))
        metas = [M([], deepest=L + 3), M([(L, idx), (L + 1, 4 * idx + 2)], deepest=L + 3, rect=rect)]
        want = plan_py(metas)
        got = plan_cpp(exe, metas)
        assert got[0] == OK
        assert [v.hex() for v in got[1][3]] == [v.hex() for v in want[1][3]]


@pytest.mark.parametrize("L", [1, 2, 3, 4])
def test_parent_sets_and_walk_order(exe, L):
    rng = np.random.default_rng(10 + L)
    for trial in range(15):
        n = 4 ** L
        k = int(rng.integers(1, min(n, 40) + 1))
        roots = sorted(set(int(v) for v in rng.integers(0, n, k)))
        # several sub-roots share one meta file's directory; some metas are empty; the order of metas is shuffled
        metas = [M([(L, r), (L + 1, 4 * r + int(rng.integers(0, 4)))], deepest=L + 2) for r in roots]
        metas += [M([], deepest=L + 2) for _ in range(int(rng.integers(0, 3)))]
        rng.shuffle(metas)
        code, want = plan_py(metas)
        assert code == OK
        got = plan_cpp(exe, metas)
        assert got[0] == OK
        gL, deepest, tile, rect, groots, walk, nodes = got[1]
        assert (gL, deepest, tile) == want[:3] and groots == want[4] and nodes == want[6]
        assert set(walk) == want[5] and len(walk) == len(want[5])
        pos = {nd: i for i, nd in enumerate(walk)}
        for (l, i) in walk:  # every parent after its built children; siblings in index order; the root last
            for c in range(4):
                ch = (l + 1, 4 * i + c)
                if ch in pos:
                    assert pos[ch] < pos[(l, i)]
        assert walk[-1] == (0, 0)
        for lv in range(L):
            lvl = [i for l, i in walk if l == lv]
            assert lvl == sorted(lvl)


def _taps_py(T):
    """make_lanczos3_table(2T, T)'s sizes: T samples, each reading right - left inputs."""
    ratio, support, taps = 2.0, 6.0, 0
    for o in range(T):
        x = (o + 0.5) * ratio
        left = min(max(math.floor(x - support), 0), 2 * T - 1)
        right = min(max(math.ceil(x + support), left + 1), 2 * T)
        taps += right - left
    return 4 * 4 * T + 4 * taps


def test_device_bytes_formula(exe):
    for L in (0, 1, 2, 3, 7):
        for T in (1, 2, 7, 256, 1024, 4096):
            got = int(_run(exe, "bytes", L, T))
            want = 0 if L == 0 else (4 * L + 1) * T * T * 4 + 2 * T * T * 4 + _taps_py(T)
            assert got == want, (L, T)
