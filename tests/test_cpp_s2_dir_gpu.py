"""pcv::S2CellsDir (include/pcv.hpp) exercised once from C++: tests/cpp/test_s2_dir.cpp against pcv::S2Cells::from_directory."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_s2_cells_dir(tmp_path):
    exe = str(tmp_path / "test_s2_dir")
    lib_dir = os.path.join(ROOT, "point_cloud_viewer_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", os.path.join(ROOT, "tests", "cpp", "test_s2_dir.cpp"), "-o", exe, "-L" + lib_dir, "-l:libpcv_b200.so",
                           "-Wl,-rpath," + lib_dir])
    r = subprocess.run([exe, str(tmp_path / "s2")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr
