import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the oracle (checker), the test-only CPU backend and - if nvcc is present - the CUDA library."""
    import __graft_entry__ as g

    g.build_oracle()
    g.build_test_backend()
    if os.path.exists(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")):
        g.build_library()
    yield


@pytest.fixture(scope="session")
def ctx():
    import point_cloud_viewer_b200 as pcv

    c = pcv.Context(0)
    yield c
    c.close()
