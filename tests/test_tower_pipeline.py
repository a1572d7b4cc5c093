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
TC_PASSES = 3  # the pass count on fp16 hi/lo planes (hi*hi + hi*lo + lo*hi); one fp16 plane runs hi*hi alone
# the conv kernels each object's dispatch can reach, as (name, template arguments): tower_tc.cu (dispatch_conv) runs
# <BN, PAIR> = <256|128, true> and <256|128|64, false> on both operand forms (two planes, one) and the 192-row fused
# kernel; train_tc.cu runs the raw-mode conv and the backward-filter kernel at BN = 256, 128 and 64
REACHABLE_CONV = {
    "tower_tc": sorted([("k_conv3x3_tc", (bn, pair, ops)) for ops in (2, 1)
                        for bn, pair in ((256, 1), (128, 1), (256, 0), (128, 0), (64, 0))] + [("k_conv3x3_m192", (256, 1))]),
    "train_tc": sorted([("k_conv3x3_tc", (bn, 0, 2)) for bn in (256, 128, 64)] + [("k_dw_tc", (bn,)) for bn in (256, 128, 64)]),
}


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
    """Tensor passes per K block of a wgmma kernel, from its operand-plane count (two planes: three passes, one plane:
    one), or None for any other function."""
    if "k_conv3x3_tc" in name:
        m = re.search(r"k_conv3x3_tcILi(\d+)ELb([01])ELi([12])EE", name)
        assert m, name
        return TC_PASSES if m.group(3) == "2" else 1
    if "k_smallnet_fp16" in name:
        return 1
    return TC_PASSES if re.search(r"k_conv3x3_m192|k_dw_tc|k_net_small", name) else None


def test_library_holds_exactly_the_reachable_conv_kernels():
    """The tower object holds the 10 k_conv3x3_tc instantiations and the one k_conv3x3_m192 its dispatch can launch, and
    the training object its 3 k_conv3x3_tc and 3 k_dw_tc: no kernel that nothing launches."""
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built library and cuobjdump")
    found = {}
    for name in _sass_functions(tool):
        # _ZN<len>_GLOBAL__N__<hash>_<len>_<unit>_cu_<hash><len><kernel>I<template arguments>E...
        m = re.search(r"_([a-z_]+)_cu_[0-9a-f]+\d(k_conv3x3_tc|k_conv3x3_m192|k_dw_tc)I((?:L[ib]\d+E)+)E", name)
        if m:
            found.setdefault(m.group(1), []).append((m.group(2), tuple(int(v) for v in re.findall(r"\d+", m.group(3)))))
    assert {unit: sorted(k) for unit, k in found.items()} == REACHABLE_CONV, found


def test_conv_kernel_one_warpgroup_arrive_per_k_block():
    """Every wgmma kernel (each k_conv3x3_tc, k_conv3x3_m192 and k_dw_tc instantiation, and k_net_small and
    k_smallnet_fp16 with one K-block loop per layer width) issues each K block as one batch: one WARPGROUP.ARRIVE, then
    all passes x k16 HGMMAs with nothing in between, and only the last one waits on the scoreboard (gsb0)."""
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built library and cuobjdump")
    kernels = {n: (_passes(n), body) for n, body in _sass_functions(tool).items() if _passes(n) is not None}
    names = " ".join(kernels)
    assert "k_conv3x3_tc" in names, "no k_conv3x3_tc in the library"
    for kernel in ("k_conv3x3_m192", "k_dw_tcILi64E", "k_dw_tcILi128E", "k_dw_tcILi256E", "k_net_small", "k_smallnet_fp16"):
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
