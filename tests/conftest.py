import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA sm_90a device (run with -m gpu)")


@pytest.fixture(scope="session")
def built_lib():
    """Build (if stale) and load libyamb200.so; works without a GPU."""
    import __graft_entry__ as g
    g.build()
    from yet_another_mobilenet_series_b200 import native
    return native.lib()


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
