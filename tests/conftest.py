import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def _has_gpu():
    try:
        from directxtex_b200 import capi
        return capi.lib.dxb200_device_count() > 0
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    """ctypes handle on oracle/_ref/libdxtex_ref.so (the unmodified reference, built by oracle/Makefile).
    Built here when /root/reference is mounted; on the GPU box the prebuilt .so travels with the repo."""
    from tests import oracle_lib
    return oracle_lib.load_ref()


@pytest.fixture(scope="session")
def emul():
    from tests import oracle_lib
    return oracle_lib.load_emul()
