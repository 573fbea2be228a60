import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device of compute capability 9.0 (H100)")


def _has_gpu():
    try:
        from skdist_b200 import _lib
        return _lib.load().skd_device_count() > 0
    except Exception:
        return False


HAS_GPU = _has_gpu()


def pytest_collection_modifyitems(config, items):
    if HAS_GPU:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture
def fake_engine():
    """Route skdist_b200.engine.get_engine() to the oracle-backed stand-in (host-logic tests)."""
    from skdist_b200 import engine
    from tests.fake_engine import FakeEngine
    engine.set_engine_factory(FakeEngine)
    yield
    engine.set_engine_factory(None)
