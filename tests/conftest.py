import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _cuda_device_present() -> bool:
    """True when libvello_b200.so can create a renderer (= a CUDA device is usable). No torch import."""
    try:
        from vello_b200.renderer import Renderer
        r = Renderer()
        r.close()
        return True
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests are skipped (not failed) on a box without a CUDA device; the product itself still raises there."""
    gpu_items = [it for it in items if it.get_closest_marker("gpu")]
    if gpu_items and not _cuda_device_present():
        skip = pytest.mark.skip(reason="no CUDA device / libvello_b200.so could not create a renderer")
        for it in gpu_items:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle.vbo import Oracle
    return Oracle(threads=4)


@pytest.fixture(scope="session")
def oracle_libm():
    from oracle.vbo import Oracle
    return Oracle(libm=True, threads=4)
