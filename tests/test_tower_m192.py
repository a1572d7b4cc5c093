"""k_conv3x3_m192: the fused residual-block conv on 192-row tiles (three consumer warpgroups, 384 threads).

On the per-sample layout its M rows are the board points alone (a TMA im2col map skips the zero column and the tile
tail).  Each output row is accumulated by the same (tap, chunk, k16, pass) sequence of wgmmas as on the 128-row kernel,
and the window values off the board are zeros either way, so the two kernels must give the same bits.
CPU: the kernel's SASS shape and resources, and a restatement of the dispatch rule.  GPU: tower outputs (az_infer_tower) and policy/value (az_infer) of AZ_TC_M192=0 and the default, bit for bit."""
import collections
import os
import re
import subprocess

import numpy as np
import pytest

from agogo_b200 import _capi as K
from tests import helpers as H
from tests import pyref_dual as D
from tests.test_tc_layers import _desc, _planes, tower_layout
from tests.test_tower_pipeline import K_STEPS_PER_BLOCK, LIB, TC_PASSES, _cuobjdump, _sass_functions

M192 = "k_conv3x3_m192ILi256ELb1EE"
BM192 = 192
MAX_REGS = 168  # 384 threads x 168 = 64512 of the SM's 65536 registers, one CTA per SM


# the dispatch rule, restated (tower_tc.cu: tc_tower_alloc, dispatch_conv): every fused layer with BN = 256 (K >= 128);
# M rows per sample: the board points on the per-sample layout, the flat positions otherwise
def m192_applies(m, n, k, layers):
    lay = tower_layout(m, n, k, layers)
    return dict(lay, m192=k >= 128 and not lay["small"], rows=m * n if lay["per_sample"] else lay["S"])


Case = collections.namedtuple("Case", "name kind m n k layers n_big n_mid")
CASES = [
    Case("wq19-k256", K.GAME_WQ, 19, 19, 256, 2, 300, 37),  # per-sample (im2col); several tiles per CTA
    Case("wq19-k128", K.GAME_WQ, 19, 19, 128, 2, 64, 9),
    Case("mnk19x12-k128", K.GAME_MNK, 19, 12, 128, 2, 12, 5),  # per-sample, H != W
    Case("wq13-k256", K.GAME_WQ, 13, 13, 256, 2, 100, 13),  # flat
    Case("wq13-k128", K.GAME_WQ, 13, 13, 128, 2, 64, 7),    # flat
    Case("wq19-k64", K.GAME_WQ, 19, 19, 64, 2, 12, 5),      # fused BN = 128: the 128-row kernel
]


def test_m192_kernel_sass_shape():
    """One WARPGROUP.ARRIVE and 12 HGMMAs per K block, only the last on gsb0; no local memory, at most 168 registers."""
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built library and cuobjdump")
    funcs = _sass_functions(tool)
    names = [n for n in funcs if M192 in n]
    assert len(names) == 1, names
    body = funcs[names[0]]
    assert not any(re.search(r"\b(STL|LDL)\b", ln) for ln in body), "local memory"
    ins = [ln for ln in body if "WARPGROUP.ARRIVE" in ln or "HGMMA" in ln]
    arrives = sum("WARPGROUP.ARRIVE" in ln for ln in ins)
    hgmma = [ln for ln in ins if "HGMMA" in ln]
    assert arrives == 1 and len(hgmma) == TC_PASSES * K_STEPS_PER_BLOCK, (arrives, len(hgmma))
    assert "gsb0" in hgmma[-1] and sum("gsb0" in ln for ln in hgmma) == 1
    assert all("64x256x16" in ln for ln in hgmma), hgmma[0]
    res = subprocess.run([tool, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    m = re.search(re.escape(M192) + r"\S*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", res)
    assert m, "no resource line for %s" % M192
    regs, stack, local = map(int, m.groups())
    assert regs <= MAX_REGS and stack == 0 and local == 0, (regs, stack, local)


def test_m192_dispatch_cases_cover_the_rule():
    """The GPU cases below reach every branch of the rule: the per-sample layout (im2col) at K = 256 and 128 and with
    H != W, the flat layout at K = 256 and 128, and a K = 64 net that keeps the 128-row kernel; the middle batch ends
    inside a 192-row tile, and a tile straddles two samples."""
    seen = set()
    for c in CASES:
        r = m192_applies(c.m, c.n, c.k, c.layers)
        if not r["m192"]:
            seen.add("k%d 128-row" % c.k)
            continue
        seen.add("%s k%d%s" % ("per-sample" if r["per_sample"] else "flat", c.k, " H != W" if c.m != c.n else ""))
        assert (c.n_mid * r["rows"]) % BM192 and r["rows"] % BM192, c.name
        assert c.n_big > c.n_mid > 1
    assert {"per-sample k256", "per-sample k128", "per-sample k128 H != W", "flat k256", "flat k128", "k64 128-row"} <= seen, seen
    c3 = m192_applies(19, 19, 256, 20)  # the C3 headline: 963 tiles of 192 board points for 512 samples, not 1024
    assert c3["m192"] and c3["per_sample"] and -(-512 * c3["rows"] // BM192) == 963


def _run(engine_lib, monkeypatch, c, flag, params, planes):
    monkeypatch.setenv("AZ_TC_M192", flag)
    e = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, c.layers, c.n_big))
    if params is None:
        params = H.tame_gammas([e], 0, 17, target=0.9)
    else:
        e.net_set(0, params)
    e.set_inferer(0, K.INF_DUAL)
    e.profile(True)
    kind = e.profile(False)["kernel_kind"]
    outs = []
    for nn in (c.n_big, c.n_mid, 1):
        outs.append((e.infer_tower(0, planes[:nn]), *e.infer(0, planes[:nn])))
    e.close()
    return kind, outs, params


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_m192_bits_equal_128_row_kernel(engine_lib, monkeypatch, c):
    """Same weights and planes on AZ_TC_M192=0 and the default: tower output, policy and value bit-identical at a full
    batch, a middle batch and n = 1 (n descending on each engine); kernel_kind 8 exactly where the rule applies."""
    planes = _planes(c.kind, np.random.default_rng(5), c.n_big, c.m, c.n)
    kind0, ref, params = _run(engine_lib, monkeypatch, c, "0", None, planes)
    kind1, new, _ = _run(engine_lib, monkeypatch, c, "1", params, planes)
    assert kind0 == 0 and kind1 == (8 if m192_applies(c.m, c.n, c.k, c.layers)["m192"] else 0), (kind0, kind1)
    for nn, a, b in zip((c.n_big, c.n_mid, 1), ref, new):
        for x, y in zip(a, b):
            assert np.isfinite(x).all(), (c.name, nn)
            assert x.shape == y.shape and (x.view(np.uint32) == y.view(np.uint32)).all(), (c.name, nn)


@pytest.mark.gpu
def test_m192_activation_overflow_is_reported(engine_lib):
    """At act_scale_log2 = 20 an output of the fused layers beyond fp16's range raises AZ_ERR_PANIC "activation
    overflow" from the 192-row kernel.  Zero planes and biases pin where it happens: the init conv outputs
    relu(2^-8) * 2^20 = 4096, in range; the fused layers add a bias of 1 before the ReLU, so their outputs reach the
    order of 2^20, out of range.  (Non-zero planes would already overflow when packed at this scale.)"""
    planes = np.zeros((4, 18 * 19 * 19), np.float32)
    e = engine_lib.create(_desc(K.GAME_WQ, 19, 19, 256, 2, 4, act=20))
    H.tame_gammas([e], 0, 3, target=0.9)
    tensors = D.unpack(e, 0)
    for name, t in tensors:
        if name.endswith("_conv_β") and ("FilterInit" in name or "Shared Layer" in name):
            t[...] = 2.0 ** -8 if "FilterInit" in name else 1.0
    e.net_set(0, D.pack(e, [t for _, t in tensors]))
    e.set_inferer(0, K.INF_DUAL)
    e.profile(True)
    assert e.profile(False)["kernel_kind"] == 8
    with pytest.raises(K.AZError) as ei:
        e.infer(0, planes)
    assert ei.value.code == -3 and "activation overflow" in str(ei.value), str(ei.value)
    e.close()
