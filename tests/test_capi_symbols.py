"""The product library loads without a GPU, exports every symbol include/agogo_b200.h declares, and
refuses loudly (AZ_ERR_CUDA) to create an engine when there is no CUDA device — no CPU fallback."""
import ctypes as C
import os
import re
import subprocess

import pytest

from agogo_b200 import _capi as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "agogo_b200.h")).read()
    return sorted(set(re.findall(r"^(?:int|void|const char\*)\s+(az_[a-z_0-9]+)\s*\(", src, flags=re.M)))


def test_header_and_binding_agree():
    assert set(K.SYMBOLS) == set(_declared())


@pytest.fixture(scope="module")
def product():
    if not os.path.exists(K.PRODUCT_LIB):
        from agogo_b200 import build
        build.build()
    return K.load()


def test_product_exports_every_declared_symbol(product):
    for name in _declared():
        assert hasattr(product.dll, name), name
    assert "sm_90a" in product.build_info()


def test_oracle_exports_every_declared_symbol(oracle):
    for name in _declared():
        assert hasattr(oracle.dll, name), name


def _has_gpu():
    try:
        return subprocess.run(["nvidia-smi", "-L"], capture_output=True, timeout=20).returncode == 0
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="this check is for GPU-less hosts")
def test_product_fails_loudly_without_gpu(product):
    from tests import helpers as H
    with pytest.raises(K.AZError) as ei:
        product.create(K.make_desc(K.GAME_MNK, 3, 3, 3, sims=2, nn=H.tiny_nn(3, 3, 10)))
    assert ei.value.code == -2 and "no CPU fallback" in str(ei.value)


def test_product_never_references_the_oracle():
    """Nothing under agogo_b200/ (the shipped package) may import, link or name the oracle."""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "agogo_b200")):
        if "build" in dirpath.split(os.sep):
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "libazoracle" not in txt and "oracle/" not in txt.replace("oracle/dual.hpp", "").replace("oracle/wq.hpp", ""), (dirpath, f)
