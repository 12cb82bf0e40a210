import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session")
def oracle():
    """CPU oracle (oracle/vlcal_oracle.c) -- the checker, never the thing under test in -m gpu runs."""
    from oracle import oracle as O

    O.build()
    return O


@pytest.fixture(scope="session")
def vlcal():
    """The product package; the C-ABI library must be built (there is no fallback)."""
    import direct_visual_lidar_calibration_b200 as V

    if not os.path.exists(V.library_path()):
        V.build_library()
    V.load_library()
    return V


@pytest.fixture(scope="session")
def gpu(vlcal):
    if vlcal.device_count() < 1:
        pytest.fail("GPU test selected but no CUDA device is visible (the product has no CPU fallback)")
    return vlcal
