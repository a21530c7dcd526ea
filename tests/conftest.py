import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")
    # build the product library and the oracle if they are missing (CPU-only cross compile)
    need = [os.path.join(ROOT, "goleft_b200", "libgoleft_b200.so"), os.path.join(ROOT, "oracle", "_build", "liboracle.so")]
    if not all(os.path.exists(p) for p in need):
        subprocess.check_call(["make", "-s", "lib", "oracle"], cwd=ROOT)


def _has_gpu():
    try:
        from goleft_b200 import capi
        return capi.device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def ctx():
    from goleft_b200 import capi
    c = capi.Ctx(0)
    yield c
    c.close()
