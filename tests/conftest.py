import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _has_gpu() -> bool:
    try:
        from aurora_b200 import _native as N

        return N.load().aur_device_count() > 0
    except Exception:
        return False


@pytest.fixture(scope="session")
def gpu_available():
    return _has_gpu()


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU (or without the library) must fail loudly, not skip
    # silently; `-m "not gpu"` never touches the device.
    pass
