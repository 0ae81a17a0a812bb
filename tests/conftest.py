import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


def _have_gpu():
    import particlesfm_b200
    return particlesfm_b200.device_count() > 0


@pytest.fixture(scope="session")
def gpu():
    if not _have_gpu():
        pytest.fail("a test marked gpu ran without a CUDA device / built libpsfm_b200.so — "
                    "the product has no CPU fallback")
    return True
