"""AZ_FLAG_FP16_TOWER: the tensor-core tower with one fp16 per operand and one wgmma pass, against the float64 reference.

Per conv layer l (the depth-l / depth-(l-1) construction of tests/test_tc_layers.py), every element is held to
    |dev - ref| <= C16 * 2^-11 * (mag + |ref|) + 2^-(25 + act_scale_log2),   mag = sum |A'| * (|W| (*) |x|),
a worst-case bound, not a fitted one: fp16 rounding of the filters contributes at most 2^-11 * mag, of the stored
output at most 2^-11 * |ref|, of the encoder planes (layer 0) at most 2^-11 * mag, and fp32 accumulation of 9K terms
9K * 2^-24 * mag; the last term is the fp16 subnormal spacing of the stored activations (x * 2^act_scale_log2).
The ratio reported per case is |dev - ref| / (2^-11 * (mag + |ref|) + 2^-(26 + act_scale_log2)), so the bound is
ratio <= C16."""
import os
import re

import numpy as np
import pytest

from agogo_b200 import _capi as K
from tests import helpers as H
from tests import pyref_dual as D
from tests.test_gpu_engine import _c3_oracle_outputs
from tests.test_tc_layers import (DEFAULT_ACT_SCALE_LOG2, TOWER_CASES, TRAIN_CASES, TOL_POLICY, TOL_VALUE, _desc, _layer_ref,
                                  _planes, tower_layout)
from tests.test_tower_pipeline import LIB, _cuobjdump, _sass_functions

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP16 = K.FLAG_FP16_TOWER
C16 = 2.0
U16 = 2.0 ** -11
# Worst measured ratio over the layers of each case on an H100 SXM (80 GB, 700 W power limit): 0.74-0.90 (always the
# init conv, where the encoder planes are rounded too), 0.21-0.55 on the fused layers; act_scale_log2 in {-5, -2, 5}:
# 0.67-0.69.  The bound leaves more than 2x.
# The flag must be visible: the fused layers' worst error under it, in units of the bound's two terms
# 2^-11 * (mag + |ref|) + 2^-(25 + act_scale_log2), is at least this many times the default path's; a build that ran
# three passes would give a factor near 1.  Measured on an H100 SXM (700 W): fp16 0.293 against 0.0061 on wq13-k64
# (48x), 0.217 against 0.0115 on wq19-k256 (19x; at K = 256 the output rounding's share is small, |ref| << mag).
HONOURED_MIN_FACTOR = 8.0
# C3 end to end against the fp32 oracle: usefulness gate for the tamed nets (per-layer gain 0.9)
USEFUL_POLICY_REL, USEFUL_VALUE = 5e-2, 1e-2
# (policy entry relative, |delta value|) per weight-set kind: 4x the worst measured on an H100 SXM (700 W).  Measured:
# tamed 2.2e-4 / 4.3e-5, reference init (per-layer gain 1.04 over 41 layers) 5.6e-3 / 9.7e-4; argmax agrees on every
# position
C3_TOL = {"tamed": (9e-4, 1.8e-4), "reference": (2.3e-2, 4e-3)}

# the fp16 kernels: k_conv3x3_tc<BN, PAIR, OPS = 1> for the five tower shapes, and the fp16 small net
FP16_CONV = ["k_conv3x3_tcILi%dELb%dELi1EE" % s for s in ((256, 1), (128, 1), (256, 0), (128, 0), (64, 0))]
FP16_SMALL = "k_smallnet_fp16"


def test_fp16_kernels_one_arrive_four_hgmma_no_spills():
    """Every fp16 tower kernel issues each K block as one WARPGROUP.ARRIVE then 4 HGMMAs (one pass x four k16 steps),
    only the last waiting on gsb0, and touches no local memory."""
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built library and cuobjdump")
    funcs = _sass_functions(tool)
    for want in FP16_CONV + [FP16_SMALL]:
        names = [n for n in funcs if want in n]
        assert names, "no %s in the library" % want
        for name in names:
            body = funcs[name]
            assert not any(re.search(r"\b(STL|LDL)\b", ln) for ln in body), (name, "local memory")
            ins = [ln for ln in body if "WARPGROUP.ARRIVE" in ln or "HGMMA" in ln]
            arrives = sum("WARPGROUP.ARRIVE" in ln for ln in ins)
            hgmma = [ln for ln in ins if "HGMMA" in ln]
            assert arrives >= 1 and len(hgmma) == 4 * arrives, (name, arrives, len(hgmma))
            assert sum("gsb0" in ln for ln in hgmma) == arrives, name
            run = []
            for ln in ins:
                if "WARPGROUP.ARRIVE" in ln:
                    assert not run, name
                else:
                    run.append(ln)
                    if "gsb0" in ln:
                        assert len(run) == 4, (name, len(run))
                        run = []


def test_fp16_flag_value_matches_header():
    with open(os.path.join(ROOT, "include", "agogo_b200.h")) as f:
        m = re.search(r"#define AZ_FLAG_FP16_TOWER (\d+)u", f.read())
    assert m and int(m.group(1)) == K.FLAG_FP16_TOWER == 16


# ---------------------------------------------------------------------------------------------------------------------
def _ratio16(dev, ref, mag, act):
    ea = act or DEFAULT_ACT_SCALE_LOG2
    return np.abs(dev.astype(np.float64) - ref) / (U16 * (mag + np.abs(ref)) + 2.0 ** -(26 + ea))


def _layers(engine_lib, monkeypatch, c, flags=FP16, act=0, seed=11):
    """_tower_layers of tests/test_tc_layers.py under `flags`: the device output of every depth 0..L (n descending on each
    engine, rows bit-identical), a fresh engine's bits at n = 1, and per layer (device output, float64 reference, mag).
    Returns (layers, net, planes, the depth-L engine)."""
    for key, val in c.env.items():
        monkeypatch.setenv(key, val)
    L = c.layers
    planes = _planes(c.kind, np.random.default_rng(seed), c.n_big, c.m, c.n)
    X = planes.reshape(c.n_big, -1, c.m, c.n).astype(np.float64)
    deep = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, L, c.n_big, flags=flags, act=act))
    H.tame_gammas([deep], 0, seed, target=0.9)
    src = [t for _, t in D.unpack(deep, 0)]
    net = D.Net(D.unpack(deep, 0), L)
    layers = []
    for l in range(L + 1):
        e = deep if l == L else engine_lib.create(_desc(c.kind, c.m, c.n, c.k, l, c.n_big, flags=flags, act=act))
        if l < L:
            e.net_set(0, D.pack(e, src[:3 * (1 + 2 * l)] + src[-12:]))
        e.set_inferer(0, K.INF_DUAL)
        big = e.infer_tower(0, planes)
        for nn in (c.n_mid, 1):
            small = e.infer_tower(0, planes[:nn])
            assert (small.view(np.uint32) == big[:nn].view(np.uint32)).all(), (c.name, l, nn)
        if l < L:
            e.close()
        assert np.isfinite(big).all(), (c.name, l)
        ref, mag = _layer_ref(net, l, X if l == 0 else layers[-1][0].astype(np.float64))
        layers.append((big, ref, mag))
    fresh = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, L, c.n_big, flags=flags, act=act))
    fresh.net_set(0, deep.net_get(0))
    fresh.set_inferer(0, K.INF_DUAL)
    assert (fresh.infer_tower(0, planes[:1]).view(np.uint32) == deep.infer_tower(0, planes[:1]).view(np.uint32)).all(), c.name
    fresh.close()
    return layers, net, planes, deep


@pytest.mark.gpu
@pytest.mark.parametrize("c", TOWER_CASES, ids=[c.name for c in TOWER_CASES])
def test_fp16_tower_layers_vs_float64(engine_lib, monkeypatch, c):
    """Every conv layer of the fp16 tower within the worst-case fp16 bound, element by element; then the float64 heads on
    the device's fp16 tower output against az_infer (the heads are fp32, so the default path's tolerances hold)."""
    layers, net, planes, deep = _layers(engine_lib, monkeypatch, c)
    worst = [float(_ratio16(dev, ref, mag, 0).max()) for dev, ref, mag in layers]
    p_dev, v_dev = deep.infer(0, planes)
    p_ref, v_ref = net.infer(tower=layers[-1][0].astype(np.float64))
    deep.close()
    rel_p = np.abs(p_dev - p_ref) / p_ref
    dv = np.abs(v_dev - v_ref)
    print("fp16 %s: worst ratio per layer %s ; heads: policy rel %.3g, value abs %.3g" %
          (c.name, " ".join("%.3g" % w for w in worst), rel_p.max(), dv.max()))
    assert max(worst) <= C16, (c.name, worst)
    assert rel_p.max() <= TOL_POLICY and dv.max() <= TOL_VALUE, (c.name, rel_p.max(), dv.max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["wq13-k64", "wq19-k256"])
def test_fp16_flag_is_honoured(engine_lib, monkeypatch, name):
    """Same planes and weights with and without the flag: the fused layers' worst ratio under the flag is many times the
    default path's — a build that quietly ran three passes would fail here."""
    c = next(c for c in TOWER_CASES if c.name == name)
    ea = DEFAULT_ACT_SCALE_LOG2
    worst = {}
    for flags in (FP16, 0):
        layers, _, _, deep = _layers(engine_lib, monkeypatch, c, flags=flags)
        deep.close()
        worst[flags] = max(float((np.abs(dev.astype(np.float64) - ref) / (U16 * (mag + np.abs(ref)) + 2.0 ** -(25 + ea))).max())
                           for dev, ref, mag in layers[1:])
    print("%s fused layers, worst ratio: fp16 %.3g, default %.3g, factor %.3g" %
          (name, worst[FP16], worst[0], worst[FP16] / worst[0]))
    assert worst[FP16] >= HONOURED_MIN_FACTOR * worst[0], worst


def _c2_desc(kind, flags):
    if kind == K.GAME_WQ:  # BASELINE C2: 9x9 wq, 6 blocks x 64
        return K.make_desc(K.GAME_WQ, 9, 9, 0, komi=7.5, sims=2, n_games=40, seed=5, max_moves=4, flags=flags,
                           nn=dict(k=64, shared_layers=6, fc=128, batch_size=2, features=18, action_space=82))
    return K.make_desc(K.GAME_C4, 6, 7, 4, sims=2, n_games=40, seed=5, max_moves=4, flags=flags,
                       nn=dict(k=64, shared_layers=3, fc=32, batch_size=2, features=2, action_space=8))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [K.GAME_WQ, K.GAME_C4], ids=["c2-9x9", "c4-6x7"])
def test_fp16_small_net_equals_per_layer(engine_lib, monkeypatch, kind):
    """The fp16 small-net kernel (kind 7) and the per-layer fp16 kernels (AZ_TC_SMALLNET=0, kind 6) give the same bits:
    same tap order, same epilogue."""
    m, n = (9, 9) if kind == K.GAME_WQ else (6, 7)
    planes = _planes(kind, np.random.default_rng(4), 40, m, n)
    res = {}
    params = None
    for sn in ("1", "0"):
        monkeypatch.setenv("AZ_TC_SMALLNET", sn)
        e = engine_lib.create(_c2_desc(kind, FP16))
        if params is None:
            params = H.tame_gammas([e], 0, 21, target=0.9)
        else:
            e.net_set(0, params)
        e.set_inferer(0, K.INF_DUAL)
        e.profile(True)
        kk = e.profile(False)["kernel_kind"]
        res[sn] = (kk, e.infer_tower(0, planes), *e.infer(0, planes))
        e.close()
    assert res["1"][0] == 7 and res["0"][0] == 6, (res["1"][0], res["0"][0])
    for a, b in zip(res["1"][1:], res["0"][1:]):
        assert np.isfinite(a).all()
        assert (a.view(np.uint32) == b.view(np.uint32)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("act", [-5, -2, 5])
@pytest.mark.parametrize("name", ["wq9-k64-small", "wq13-k64"])
def test_fp16_tower_layers_across_activation_scales(engine_lib, monkeypatch, name, act):
    """act_scale_log2 moves the fp16 window of the stored activations; every layer stays within the bound."""
    c = next(c for c in TOWER_CASES if c.name == name)._replace(n_big=6, n_mid=3)
    layers, *_, deep = _layers(engine_lib, monkeypatch, c, act=act)
    deep.close()
    worst = [float(_ratio16(dev, ref, mag, act).max()) for dev, ref, mag in layers]
    print("fp16 %s act_scale_log2=%d: worst ratio per layer %s" % (name, act, " ".join("%.3g" % w for w in worst)))
    assert max(worst) <= C16, (name, act, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["wq9-k64-small", "wq13-k64"])
def test_fp16_activation_overflow_is_reported(engine_lib, name):
    """Both fp16 kernels (k_smallnet_fp16, the per-layer k_conv3x3_tc) raise the overflow flag past fp16's range."""
    c = next(c for c in TOWER_CASES if c.name == name)
    planes = _planes(c.kind, np.random.default_rng(1), 4, c.m, c.n)
    e = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, 2, 4, flags=FP16, act=20))
    H.tame_gammas([e], 0, 3, target=0.9)
    e.set_inferer(0, K.INF_DUAL)
    e.profile(True)
    assert e.profile(False)["kernel_kind"] == (7 if tower_layout(c.m, c.n, c.k, 2)["small"] else 6)
    with pytest.raises(K.AZError) as ei:
        e.infer(0, planes)
    assert ei.value.code == -3 and "activation overflow" in str(ei.value), str(ei.value)
    e.close()


@pytest.mark.gpu
def test_fp16_c3_end_to_end_vs_oracle(oracle, engine_lib):
    """The headline net (20 blocks x 256, 19x19, FC 512) under the flag against the fp32 oracle on the four weight sets
    of test_tc_tower_full_depth_c3: every policy entry's relative error and |delta value|, and argmax agreement."""
    report, worst_p, worst_v = [], 0.0, 0.0
    for init, seed in [("tamed", 99), ("tamed", 7), ("reference", 5), ("reference", 11)]:
        params, planes, po, vo = _c3_oracle_outputs(oracle, init, seed)
        e = engine_lib.create(K.make_desc(K.GAME_WQ, 19, 19, 0, komi=7.5, sims=2, n_games=4, seed=2, max_moves=4, flags=FP16,
                                          nn=dict(k=256, shared_layers=20, fc=512, batch_size=2, features=18,
                                                  action_space=362)))
        e.net_set(0, params)
        e.set_inferer(0, K.INF_DUAL)
        e.profile(True)
        assert e.profile(False)["kernel_kind"] == 6
        p, v = e.infer(0, planes)
        e.close()
        assert np.isfinite(p).all() and np.isfinite(v).all()
        rel = float((np.abs(p.astype(np.float64) - po) / po).max())
        dv = float(np.abs(v.astype(np.float64) - vo).max())
        agree = int((p.argmax(1) == po.argmax(1)).sum())
        report.append("%s/%d: policy rel %.3g, |dv| %.3g, argmax %d/%d" % (init, seed, rel, dv, agree, len(p)))
        if init == "tamed":
            assert rel <= USEFUL_POLICY_REL and dv <= USEFUL_VALUE, (init, seed, rel, dv)
        worst_p, worst_v = max(worst_p, rel), max(worst_v, dv)
        assert rel <= C3_TOL[init][0] and dv <= C3_TOL[init][1], (init, seed, rel, dv)
    print("fp16 C3 vs oracle: " + "; ".join(report) + " ; worst policy rel %.3g, |dv| %.3g" % (worst_p, worst_v))


def _arena(engine_lib, monkeypatch, desc_fn, n_games, tame, no_graph):
    monkeypatch.setenv("AZ_NO_GRAPH", "1" if no_graph else "0")
    e = engine_lib.create(desc_fn())
    H.tame_gammas([e], 0, tame, target=0.9)
    H.tame_gammas([e], 1, tame + 1, target=0.9)
    e.set_inferer(0, K.INF_DUAL)
    e.set_inferer(1, K.INF_DUAL)
    run = H.play_and_collect(e, n_games)
    e.close()
    for t in (0, 1):  # W and P columns of every tree row
        for ply in run["dumps"]:
            for g in ply:
                assert np.isfinite(g[t][:, 3:5].copy().view(np.float32)).all()
    for x in run["examples"]:
        assert np.isfinite(x).all()
    return run


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["c2-9x9-k64", "19x19-k256"])
def test_fp16_search_in_the_loop(engine_lib, monkeypatch, shape):
    """Arena play with the fp16 tower in the captured wave graph: two engines with the same seed give identical game
    records, examples and trees, and AZ_NO_GRAPH=1 (plain launches) gives the same as graph replay."""
    if shape == "c2-9x9-k64":
        def desc():
            return K.make_desc(K.GAME_WQ, 9, 9, 0, komi=7.5, sims=16, n_games=8, seed=31, max_moves=4, flags=FP16,
                               nn=dict(k=64, shared_layers=6, fc=128, batch_size=2, features=18, action_space=82))
        n_games = 8
    else:
        def desc():
            return K.make_desc(K.GAME_WQ, 19, 19, 0, komi=7.5, sims=8, n_games=4, seed=32, max_moves=2, flags=FP16,
                               nn=dict(k=256, shared_layers=2, fc=64, batch_size=2, features=18, action_space=362))
        n_games = 4
    a = _arena(engine_lib, monkeypatch, desc, n_games, 51, False)
    b = _arena(engine_lib, monkeypatch, desc, n_games, 51, False)
    H.assert_same_run(a, b, shape + " same seed")
    c = _arena(engine_lib, monkeypatch, desc, n_games, 51, True)
    H.assert_same_run(a, c, shape + " AZ_NO_GRAPH=1")


@pytest.mark.gpu
def test_fp16_flag_leaves_training_untouched(engine_lib, monkeypatch):
    """az_train_grads keeps the three-pass GEMMs: the flag changes no bit of the gradients or the cost."""
    c = next(c for c in TRAIN_CASES if c.name == "wq9-k128")
    rng = np.random.default_rng(7)
    A1 = c.m * c.n + 1
    X = _planes(c.kind, rng, c.batch, c.m, c.n)
    Pi = np.zeros((c.batch, A1), np.float32)
    Pi[np.arange(c.batch), rng.integers(0, A1, c.batch)] = 1
    V = rng.choice([-1.0, 0.0, 1.0], c.batch).astype(np.float32)
    res = {}
    for flags in (FP16, 0):
        e = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, c.layers, 2, batch=c.batch, flags=flags))
        H.tame_gammas([e], 1, 17, target=0.05)
        res[flags] = e.train_grads(1, X, Pi, V)
        e.close()
    (g1, c1), (g0, c0) = res[FP16], res[0]
    assert np.isfinite(g1).all()
    assert (g1.view(np.uint32) == g0.view(np.uint32)).all() and np.float32(c1) == np.float32(c0)
