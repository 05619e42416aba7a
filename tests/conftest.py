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
        from dampr_b200 import device
        return device.device_count() > 0
    except Exception:
        return False


HAVE_GPU = None


@pytest.fixture(scope="session")
def ctx():
    """One device context per test session (cuda:0). Fails loudly when there is no GPU."""
    from dampr_b200 import device
    c = device.Ctx(0)
    yield c
    c.close()
