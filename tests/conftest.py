import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _have_gpu():
    try:
        import orb_slam_b200
        return orb_slam_b200.lib().orbfe_device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def gpu_required():
    if not _have_gpu():
        pytest.fail("GPU test selected but no CUDA device / liborbfe.so: there is no CPU fallback")
