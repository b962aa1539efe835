import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with `-m gpu` on a GPU machine)")


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """The C-ABI library is a build product (git-ignored); build it once if it is missing."""
    from visdial_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()


def _cuda_device_count():
    try:
        import ctypes
        rt = ctypes.CDLL("libcudart.so")
    except OSError:
        try:
            import ctypes
            import glob
            cands = sorted(glob.glob("/usr/local/cuda/lib64/libcudart.so*"))
            rt = ctypes.CDLL(cands[0]) if cands else None
        except OSError:
            rt = None
    if rt is None:
        return 0
    n = ctypes.c_int(0)
    return n.value if rt.cudaGetDeviceCount(ctypes.byref(n)) == 0 else 0


def pytest_collection_modifyitems(config, items):
    """Plain `pytest tests` on a box without a GPU skips the gpu-marked tests instead of failing them one by one."""
    if not any("gpu" in it.keywords for it in items):
        return
    if _cuda_device_count() > 0:
        return
    skip = pytest.mark.skip(reason="no CUDA device (gpu-marked tests run with `-m gpu` on an H100)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)
