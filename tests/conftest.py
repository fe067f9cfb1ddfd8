import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) and the built libwhisper_b200.so")


def _has_gpu():
    try:
        from whisper_b200 import capi
        return capi.lib().wsp_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without a GPU should say so instead of failing in 40 different ways
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device visible")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def ref_available():
    from oracle import ref
    return ref.available()


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
