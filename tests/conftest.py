import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ORACLE_SO = os.path.join(ROOT, "oracle", "libazoracle.so")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def _build_oracle():
    srcs = [os.path.join(ROOT, "oracle", f) for f in os.listdir(os.path.join(ROOT, "oracle"))
            if f.endswith((".cpp", ".hpp"))] + [os.path.join(ROOT, "include", "agogo_b200.h")]
    if (not os.path.exists(ORACLE_SO)) or any(os.path.getmtime(s) > os.path.getmtime(ORACLE_SO) for s in srcs):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL)


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle bound through the same ctypes layer as the product (tests only)."""
    from agogo_b200 import _capi
    _build_oracle()
    return _capi.load(ORACLE_SO)


@pytest.fixture(scope="session")
def engine_lib():
    """The product CUDA library; GPU tests only."""
    from agogo_b200 import _capi
    return _capi.load()
