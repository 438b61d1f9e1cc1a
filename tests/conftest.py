import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _has_gpu() -> bool:
    try:
        from porepy_b200 import _lib
        return _lib.load().pb_device_count() >= 1
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    # GPU tests selected on a box without a GPU fail loudly instead of silently passing
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords and not config.getoption("-m"):
            item.add_marker(skip)
