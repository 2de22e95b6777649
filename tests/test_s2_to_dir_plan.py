"""Streamed S2 directories, host side: the batch planner (csrc/s2_stream_plan.h) against a Python restatement, the
pcv_s2_dir_build_info layout against gcc's, and the directory writer (csrc/s2_dir_writer.hpp) fed synthetic batches.  Both
headers are compiled here with g++ through tests/cpu_backend/s2_dir_writer_cpu.cpp."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLACK, MAX_BATCH = 1 << 20, 1 << 24


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("sdw") / "libsdw.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-shared", "-fPIC", "-pthread", "-o", out, os.path.join(ROOT, "tests", "cpu_backend", "s2_dir_writer_cpu.cpp")])
    L = C.CDLL(out)
    L.sdw_new.restype = C.c_void_p
    L.sdw_new.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int]
    for f in ("sdw_free", "sdw_begin"):
        getattr(L, f).argtypes = [C.c_void_p]
    L.sdw_submit.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.sdw_wait.argtypes = [C.c_void_p, C.c_uint64]
    L.sdw_finish.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.sdw_error.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
    L.sdw_stats.argtypes = [C.c_void_p, C.c_void_p]
    L.sdw_plan.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    return L


# ---- planner -----------------------------------------------------------------------------------------------------------------
def plan_py(budget, free, n, attr, sort_pp, sort_fixed, chunk, granule, src):
    """plan_s2_stream restated."""
    budget = budget or free - free // 8
    per = 4 * attr + 16 + 8 + 16 + sort_pp
    fixed = sort_fixed + SLACK
    g = max(1, granule)
    full = max(g, chunk // g * g)
    need = max(g, (n + g - 1) // g * g)
    cap = min(MAX_BATCH, 0xFFFFFFFE) // g * g
    if budget < fixed + g * (per + src):
        return None, fixed + g * (per + src)
    room = budget - fixed
    c = min(full, need)
    if room >= c * src + c * per:
        b = (room - c * src) // per // c * c
        b = min(b, (need + c - 1) // c * c)
        b = max(c, min(b, cap // c * c))
    else:
        b = room // (per + src) // g * g
        c = b
    return (budget, b, c, per, fixed, fixed + c * src + b * per), None


def plan_c(lib, *args):
    i = np.array(args, np.uint64)
    o = np.zeros(6, np.uint64)
    err = C.create_string_buffer(256)
    rc = lib.sdw_plan(i.ctypes.data, o.ctypes.data, err, 256)
    return rc, tuple(int(v) for v in o), err.value.decode()


def test_planner_matches_restatement(lib):
    host_chunk = lambda attr: max(4096, ((64 << 20) // attr) // 4096 * 4096)  # noqa: E731  (host_chunk_points)
    cases = 0
    for attr in (24, 27, 28, 31):
        for src_kind in ("host", 12, 31, 57, 200):  # host arrays, or PLY records of that many bytes
            if src_kind == "host":
                chunk, granule, src = host_chunk(attr), 4096, 2 * attr
            else:
                t = min(4096, max(256, (65536 // src_kind) & ~255))
                chunk, granule, src = max(t, ((64 << 20) // src_kind) // t * t), t, 2 * src_kind + attr + 1
            for n in (1, 1000, 300_000, 10**8, 5 * 10**9):
                for budget in (0, 1 << 20, 50 << 20, 300 << 20, 2 << 30, 20 << 30, 70 << 30):
                    for sort_pp, sort_fixed in ((12, 5000), (13, 1 << 16)):
                        free = 79 << 30
                        want, minimum = plan_py(budget, free, n, attr, sort_pp, sort_fixed, chunk, granule, src)
                        rc, got, err = plan_c(lib, budget, free, n, attr, sort_pp, sort_fixed, chunk, granule, src)
                        if want is None:
                            assert rc == 1 and "cannot hold one batch of %d points: at least %d bytes" % (granule, minimum) in err
                            continue
                        assert rc == 0 and got == want
                        b, c = got[1], got[2]
                        assert b % c == 0 and c % granule == 0 and 0 < b < 2**32 and got[5] <= got[0]
                        cases += 1
    assert cases > 1000


def test_planner_budget_error_names_the_budget_and_minimum(lib):
    rc, _, err = plan_c(lib, 1000, 0, 10**6, 31, 12, 4096, 2162688, 4096, 62)
    assert rc == 1 and err.startswith("a device budget of 1000 bytes") and "at least" in err


def test_info_struct_matches_the_c_compiler(tmp_path):
    """pcv_s2_dir_build_info: ctypes size and field offsets equal gcc's for include/pcv.h."""
    from point_cloud_viewer_b200 import _native as N

    fs = [f for f, _ in N.S2DirBuildInfo._fields_]
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "pcv.h"', "int main(void) {", 'printf("size %zu\\n", sizeof(pcv_s2_dir_build_info));']
    for f in fs:
        src.append('printf("%s %%zu\\n", offsetof(pcv_s2_dir_build_info, %s));' % (f, f))
    src.append("return 0; }")
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = str(tmp_path / "layout")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, str(c)])
    got = dict(l.split() for l in subprocess.check_output([exe], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(N.S2DirBuildInfo)
    for f in fs:
        assert int(got[f]) == getattr(N.S2DirBuildInfo, f).offset, f


# ---- writer ------------------------------------------------------------------------------------------------------------------
def _token(cid):
    t = "%016x" % cid
    return t.rstrip("0") or "X"


def _batches(rng, nb, ids):
    """Synthetic batches: every batch holds a random subset of `ids` (sorted), 1..50 points each; cells span batches."""
    out = []
    for _ in range(nb):
        sub = np.sort(rng.choice(ids, size=rng.integers(1, len(ids) + 1), replace=False)).astype(np.uint64)
        counts = rng.integers(1, 50, len(sub)).astype(np.uint64)
        m = int(counts.sum())
        out.append((sub, counts, rng.random(m * 3), rng.integers(0, 256, m * 3, dtype=np.uint8), rng.random(m).astype(np.float32)))
    return out


def _drive(lib, d, batches, threads, rgb=True, inten=True, finish=True):
    w = lib.sdw_new(os.fsencode(d), threads, int(rgb), int(inten))
    try:
        rc = lib.sdw_begin(w)
        for k, (ids, counts, xyz, col, it) in enumerate(batches if rc == 0 else ()):
            rc = lib.sdw_submit(w, k, xyz.ctypes.data, col.ctypes.data if rgb else None, it.ctypes.data if inten else None, ids.ctypes.data,
                                counts.ctypes.data, len(ids))
            if rc:
                break
            if k >= 1:
                lib.sdw_wait(w, k - 1)
        err = C.create_string_buffer(512)
        if finish and rc == 0:
            rc = lib.sdw_finish(w, (C.c_double * 3)(1, 2, 3), (C.c_double * 3)(4, 5, 6))
        else:
            lib.sdw_wait(w, len(batches))
        lib.sdw_error(w, err, 512)
        st = np.zeros(3, np.uint64)
        lib.sdw_stats(w, st.ctypes.data)
        return rc, err.value.decode(), st
    finally:
        lib.sdw_free(w)


def _expected(batches):
    """Every cell's file = its runs concatenated in batch order."""
    want = {}
    for ids, counts, xyz, col, it in batches:
        o = 0
        for cid, cnt in zip(ids.tolist(), counts.tolist()):
            e = want.setdefault(cid, [b"", b"", b"", 0])
            e[0] += xyz[3 * o:3 * (o + cnt)].tobytes()
            e[1] += col[3 * o:3 * (o + cnt)].tobytes()
            e[2] += it[o:o + cnt].tobytes()
            e[3] += cnt
            o += cnt
    return want


@pytest.mark.parametrize("threads", [1, 8])
def test_writer_files_are_runs_in_batch_order(lib, tmp_path, threads):
    from proto_meta import Meta

    rng = np.random.default_rng(threads)
    ids = np.array(sorted(rng.choice(2**40, 40, replace=False) * 2**20 + 2**19), np.uint64)  # level-20-like ids
    batches = _batches(rng, 9, ids)
    d = str(tmp_path / "out")
    os.makedirs(d)
    # a pre-existing longer file of a cell the cloud holds, a file of a cell it does not hold, and an old meta.pb
    open(os.path.join(d, _token(int(ids[0])) + ".xyz"), "wb").write(b"\x01" * 100000)
    open(os.path.join(d, "ffff.xyz"), "wb").write(b"keep")
    open(os.path.join(d, "meta.pb"), "wb").write(b"old")
    w = lib.sdw_new(os.fsencode(d), threads, 1, 1)
    try:
        assert lib.sdw_begin(w) == 0
        assert not os.path.exists(os.path.join(d, "meta.pb"))  # removed before any cell file is written
        for k, (bid, counts, xyz, col, it) in enumerate(batches):
            assert lib.sdw_submit(w, k, xyz.ctypes.data, col.ctypes.data, it.ctypes.data, bid.ctypes.data, counts.ctypes.data, len(bid)) == 0
        lib.sdw_wait(w, len(batches) - 1)
        assert not os.path.exists(os.path.join(d, "meta.pb"))  # absent until finish
        assert lib.sdw_finish(w, (C.c_double * 3)(1, 2, 3), (C.c_double * 3)(4, 5, 6)) == 0
        st = np.zeros(3, np.uint64)
        lib.sdw_stats(w, st.ctypes.data)
    finally:
        lib.sdw_free(w)
    want = _expected(batches)
    for cid, (xb, rb, ib, cnt) in want.items():
        stem = os.path.join(d, _token(cid))
        assert open(stem + ".xyz", "rb").read() == xb
        assert open(stem + ".rgb", "rb").read() == rb
        assert open(stem + ".intensity", "rb").read() == ib
    assert open(os.path.join(d, "ffff.xyz"), "rb").read() == b"keep"
    assert not os.path.exists(os.path.join(d, "meta.pb.tmp"))
    m = Meta.FromString(open(os.path.join(d, "meta.pb"), "rb").read())
    assert [(c.id, c.num_points) for c in m.s2.cells] == sorted((k, v[3]) for k, v in want.items())
    assert [m.bounding_box.min.x, m.bounding_box.max.z] == [1.0, 6.0]
    assert int(st[0]) == sum(len(v[0]) + len(v[1]) + len(v[2]) for v in want.values())
    assert int(st[1]) == 3 * sum(len(b[0]) for b in batches) and int(st[2]) == len(want)


def test_writer_one_attribute_set_and_thread_counts_agree(lib, tmp_path):
    rng = np.random.default_rng(7)
    ids = np.array(sorted(rng.choice(2**30, 12, replace=False) * 2**34 + 2**33), np.uint64)
    batches = _batches(rng, 5, ids)
    outs = []
    for threads in (1, 8):
        d = str(tmp_path / ("t%d" % threads))
        rc, err, _ = _drive(lib, d, batches, threads, rgb=False, inten=False)
        assert rc == 0, err
        outs.append({f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))})
    assert outs[0] == outs[1]
    assert all(f.endswith(".xyz") or f == "meta.pb" for f in outs[0])


def test_writer_unwritable_directory_is_an_io_error(lib, tmp_path):
    blocker = tmp_path / "file"
    blocker.write_bytes(b"x")
    rng = np.random.default_rng(3)
    batches = _batches(rng, 2, np.array([2**63 + 2**19], np.uint64))
    rc, err, _ = _drive(lib, str(blocker / "sub"), batches, 4)
    assert rc == 1 and err.startswith("cannot ") and str(blocker / "sub") in err
    # a directory whose cell files cannot be created: the first file is named
    d = tmp_path / "ro"
    d.mkdir()
    (d / (_token(2**63 + 2**19) + ".xyz")).mkdir()  # a directory where the cell's file would go
    rc, err, _ = _drive(lib, str(d), batches, 4)
    assert rc == 1 and err == "cannot write %s/%s.xyz" % (d, _token(2**63 + 2**19))
    assert not os.path.exists(d / "meta.pb")
