import ctypes
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on a machine with an H100)")


def _oracle_lib_path():
    return os.path.join(ROOT, "oracle", "_build", "liboracle.so")


@pytest.fixture(scope="session")
def oracle():
    """Backend over the CPU oracle (test infrastructure; the product never loads it)."""
    from risingwave_b200.executor import Backend
    p = _oracle_lib_path()
    src = os.path.join(ROOT, "oracle", "oracle.cc")
    if not os.path.exists(p) or os.path.getmtime(p) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    return Backend(ctypes.CDLL(p), "rwo_")


@pytest.fixture(scope="session")
def cuda():
    """Backend over librwgpu.so (the product). Fails loudly if not built / no device."""
    from risingwave_b200.executor import Backend
    b = Backend.cuda()
    b.lib.rwgpu_device_check.restype = ctypes.c_int32
    rc = b.lib.rwgpu_device_check()
    assert rc == 0, "no CUDA device visible to librwgpu.so"
    return b
