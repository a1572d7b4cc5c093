"""The conv kernel's MMA pipeline: its SASS shape (CPU, from the built library) and the exact bits it produces at the
headline width (GPU, against tests/golden/tower_c3_bits.npz written by tools/make_tower_golden.py)."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "agogo_b200", "libagogo_b200.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "tower_c3_bits.npz")
K_STEPS_PER_BLOCK = 4  # a K block of the wgmma kernels is 64 channels: four k16 wgmma steps
TC_PASSES = 3  # the pass count of every tensor-core kernel but the diagnostic k_conv3x3_tc instantiations


def _cuobjdump():
    return shutil.which("cuobjdump") or next((p for p in ["/usr/local/cuda/bin/cuobjdump"] if os.path.exists(p)), None)


def _sass_functions(tool):
    out = subprocess.run([tool, "-sass", LIB], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return funcs


def _passes(name):
    """Tensor passes per K block of a wgmma kernel, or None for any other function."""
    if "k_conv3x3_tc" in name:
        m = re.search(r"k_conv3x3_tcILi(\d+)ELb([01])ELi(\d)E", name)
        assert m, name
        return int(m.group(3))
    return TC_PASSES if "k_dw_tc" in name or "k_net_small" in name else None


def test_conv_kernel_one_warpgroup_arrive_per_k_block():
    """Every wgmma kernel (each k_conv3x3_tc and k_dw_tc instantiation, and k_net_small with one K-block loop per layer
    width) issues each K block as one batch: one WARPGROUP.ARRIVE, then all passes x k16 HGMMAs with nothing in between,
    and only the last one waits on the scoreboard (gsb0)."""
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built library and cuobjdump")
    kernels = {n: (_passes(n), body) for n, body in _sass_functions(tool).items() if _passes(n) is not None}
    names = " ".join(kernels)
    assert "k_conv3x3_tc" in names, "no k_conv3x3_tc in the library"
    for kernel in ("k_dw_tcILi64E", "k_dw_tcILi128E", "k_dw_tcILi256E", "k_net_small"):
        assert kernel in names, "no %s in the library" % kernel
    for name, (passes, body) in kernels.items():
        ins = [ln for ln in body if "WARPGROUP.ARRIVE" in ln or "HGMMA" in ln]
        arrives = sum("WARPGROUP.ARRIVE" in ln for ln in ins)
        hgmma = [ln for ln in ins if "HGMMA" in ln]
        assert arrives >= 1, name
        assert len(hgmma) == arrives * passes * K_STEPS_PER_BLOCK, (name, arrives, len(hgmma))
        assert sum("gsb0" in ln for ln in hgmma) == arrives, name
        # each ARRIVE opens a run of passes x k16 HGMMAs that ends on the gsb0 one
        run = []
        for ln in ins:
            if "WARPGROUP.ARRIVE" in ln:
                assert not run, name
            else:
                run.append(ln)
                if "gsb0" in ln:
                    assert len(run) == passes * K_STEPS_PER_BLOCK, (name, len(run))
                    run = []


@pytest.mark.gpu
def test_tower_and_train_bits_match_golden(engine_lib):
    """Tower outputs at C3 dims for n in {1, 3, 64, 512} and the parameters after one training step (raw-mode conv,
    backward-filter) equal, bit for bit, what the kernels produced when the fixture was written."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_tower_golden as M
    gold = np.load(GOLDEN)
    res = M.compute(engine_lib)
    assert sorted(res) == sorted(gold.files)
    for k, v in res.items():
        g = gold[k]
        assert v.shape == g.shape and v.dtype == g.dtype, k
        assert v.tobytes() == g.tobytes(), k
