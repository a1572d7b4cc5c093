"""The tensor-core kernels one layer at a time against the float64 restatement of the network (tests/pyref_dual.py).

Tower: a net with SharedLayers = l computes exactly the first l blocks of a deeper net with the same leading weights, so
the output of conv layer l is az_infer_tower of the depth-l engine, and its reference is block l of pyref_dual applied
to the depth-(l-1) engine's device output (errors do not compound; this reaches the middle layers of k_net_small, which
never leave shared memory).  Every element is held to a bound scaled by its own absolute-value computation,
    |dev - ref| <= c * 2^-21 * (sum over branches |A'| * (|W| (*) |x|) + |ref| + 2^-(4 + act_scale_log2)),
(*) the 3x3 convolution of absolute values, not by a global maximum.  The last term is the resolution of the stored
activations: x * 2^act_scale_log2 is kept as fp16 hi + lo, and lo is an fp16 subnormal (spacing 2^-24) once the value
is below 2^-3, so small activations carry an absolute error up to 2^-(25 + act_scale_log2) whatever the arithmetic.
The cases cover every position layout and tile shape tc_tower_alloc and dispatch_conv can pick
(test_dispatch_matrix_is_covered re-derives the choice on the CPU).

Heads: the float64 policy / value heads applied to the device's tower output against az_infer, every policy entry
relative.  Training: every Model() gradient of one az_train_grads step on the tensor-core GEMMs against the float64
gradients, held to a small multiple of the fp32 CUDA-core path's own error on the same tensor."""
import collections

import numpy as np
import pytest

from agogo_b200 import _capi as K
from tests import helpers as H
from tests import pyref_dual as D

BM, SN_R0, SN_MAXL, NUM_SMS = 128, 16, 8, 132  # M tile, k_net_small limits, H100 SXM SM count (tc_gemm_create's split)
ULP = 2.0 ** -21
DEFAULT_ACT_SCALE_LOG2 = -2  # what act_scale_log2 = 0 selects
# The tower bound's constant for K = 64.  A fused layer accumulates 9 * K products in fp32 and their rounding errors add
# like a random walk, so the constant grows as sqrt(K / 64).  Measured on an H100 SXM (80 GB, 700 W): the worst ratio
# |dev - ref| / (2^-21 * (mag + |ref| + 2^-(4 + act_scale_log2))) over every layer and element of a case is the last
# column of TOWER_CASES; 1.68 at K = 64, 2.32 at K = 128, 2.97 at K = 256, so the bound leaves about 4x.
C_TOWER = 6.5
# Dropping the lo(x) * hi(w) pass makes the activations enter as fp16 (2^-12 relative).  On the fused layers of wq13-k64
# the former two-pass diagnostic build measured 128 to 172 on an H100 SXM (80 GB, 700 W), 20x to 26x the bound; the
# float64 restatement of that product in test_bound_catches_a_dropped_pass gives 124 to 173, 19x to 27x.  The test asks
# for 16x.
PASSES2_MIN_EXCESS = 16.0
# heads: relative error of every policy entry, absolute error of the value (measured at most 5.2e-7 and 2.1e-7)
TOL_POLICY, TOL_VALUE = 2e-6, 1e-6
# training: tensor-core error per tensor <= C_TRAIN x the fp32 path's error on that tensor + TRAIN_FLOOR x max |g_ref|.
# Measured: at most 10.8x the fp32 path's error (the block filters' split-K backward-filter at K = 128), at most 4.1e-6
# of the tensor's max; the criterion holds with at least 2.1x to spare.
C_TRAIN, TRAIN_FLOOR = 16.0, 2.0 ** -19


def c_tower(k):
    return C_TOWER * np.sqrt(k / 64)


Case = collections.namedtuple("Case", "name kind m n k layers n_big n_mid env kernels worst")
# kernels: what the layout rule of tc_tower_alloc must pick for the case (checked on the CPU); worst: measured ratio
TOWER_CASES = [
    Case("wq9-k64-small", K.GAME_WQ, 9, 9, 64, 3, 300, 37, {}, "k_net_small", 1.68),
    Case("wq9-k64-layered", K.GAME_WQ, 9, 9, 64, 3, 37, 5, {"AZ_TC_SMALLNET": "0"}, "flat <64,false> <128,true>x1", 1.42),
    Case("c4-6x7-k64-small", K.GAME_C4, 6, 7, 64, 3, 40, 7, {}, "k_net_small", 1.35),
    Case("c4-6x7-k64-layered", K.GAME_C4, 6, 7, 64, 2, 40, 7, {"AZ_TC_SMALLNET": "0"}, "flat <64,false> <128,true>x1", 1.35),
    Case("mnk13x9-k64", K.GAME_MNK, 13, 9, 64, 3, 12, 5, {}, "flat <64,false> <128,true>x1", 1.32),
    Case("mnk9x13-k64", K.GAME_MNK, 9, 13, 64, 3, 12, 5, {}, "per-sample tps=1 <64,false> <128,true>x1", 1.27),
    Case("wq13-k64", K.GAME_WQ, 13, 13, 64, 3, 12, 5, {}, "flat <64,false> <128,true>x1", 1.48),
    Case("wq19-k64", K.GAME_WQ, 19, 19, 64, 3, 6, 3, {}, "per-sample tps=3 <64,false> <128,true>x1", 1.49),
    Case("wq9-k128", K.GAME_WQ, 9, 9, 128, 3, 12, 5, {}, "flat <128,false> <256,true>x1", 1.91),
    Case("wq19-k128", K.GAME_WQ, 19, 19, 128, 2, 6, 3, {}, "per-sample tps=3 <128,false> <256,true>x1", 2.32),
    Case("mnk19x12-k128", K.GAME_MNK, 19, 12, 128, 2, 6, 3, {}, "per-sample tps=2 <128,false> <256,true>x1", 2.07),
    Case("wq13-k256", K.GAME_WQ, 13, 13, 256, 2, 6, 3, {}, "flat <256,false> <256,true>x2", 2.92),
    Case("wq19-k256", K.GAME_WQ, 19, 19, 256, 2, 4, 3, {}, "per-sample tps=3 <256,false> <256,true>x2", 2.97),
]

TrainCase = collections.namedtuple("TrainCase", "name kind m n k layers batch")
TRAIN_CASES = [
    TrainCase("wq9-k128", K.GAME_WQ, 9, 9, 128, 2, 4),
    TrainCase("c4-6x7-k64", K.GAME_C4, 6, 7, 64, 2, 20),
    TrainCase("mnk13x9-k64", K.GAME_MNK, 13, 9, 64, 2, 8),
]


# ---------------------------------------------------------------------------------------------------------------------
# the dispatch rules, restated (tower_tc.cu: tc_tower_alloc / dispatch_conv; train_tc.cu: tc_gemm_create)
def tower_layout(m, n, k, layers, smallnet=True):
    H_, W_ = m, n  # make_desc: height = m, width = n
    s_flat, s_ps = (H_ + 1) * (W_ + 1), H_ * (W_ + 1)
    tps = -(-s_ps // BM)
    per_sample = tps * BM < s_flat
    small = smallnet and k == 64 and not per_sample and s_flat <= BM and W_ + 2 <= SN_R0 and layers + 1 <= SN_MAXL
    if small:
        kernels = "k_net_small"
    else:
        bn_init, bn_pair = min(256, k), min(256, 2 * k)
        kernels = "%s <%d,false> <%d,true>x%d" % ("per-sample tps=%d" % tps if per_sample else "flat", bn_init, bn_pair,
                                                  2 * k // bn_pair)
    return dict(per_sample=per_sample, tps=tps, S=s_ps if per_sample else s_flat, small=small, kernels=kernels)


def tower_cells(c):
    lay = tower_layout(c.m, c.n, c.k, c.layers, c.env.get("AZ_TC_SMALLNET") != "0")
    cells = set()
    if lay["small"]:
        cells.add("k64 small net")
    else:
        cells.add("k%d %s" % (c.k, "per-sample" if lay["per_sample"] else "flat"))
        if not lay["per_sample"] and lay["S"] > BM:
            cells.add("k%d flat, sample > one M tile" % c.k)
    if c.m != c.n:
        cells.add("H != W on tensor cores")
        if lay["per_sample"]:
            cells.add("per-sample H != W tps=%d" % lay["tps"])
    return cells


def train_split(c):
    S = (c.m + 1) * (c.n + 1)
    bn = min(256, c.k)
    tiles = -(-c.k // BM) * (c.k // bn)
    kb_total = -(-(c.batch * S) // 64)
    splits = max(1, min(kb_total, NUM_SMS // (9 * tiles)))
    return dict(BS=c.batch * S, kb_total=kb_total, splits=splits, kb_per_split=-(-kb_total // splits))


def test_dispatch_matrix_is_covered():
    """Every cell of the tensor-core dispatch matrix is hit by a case above, by the layout rule the allocator applies."""
    cells = set()
    for c in TOWER_CASES:
        lay = tower_layout(c.m, c.n, c.k, c.layers, c.env.get("AZ_TC_SMALLNET") != "0")
        assert lay["kernels"] == c.kernels, (c.name, lay)
        cells |= tower_cells(c)
        # the middle n ends inside an M tile, so the tile also holds rows beyond the batch
        assert (c.n_mid * lay["S"]) % BM if not lay["per_sample"] else lay["S"] % BM, c.name
        assert c.n_big > c.n_mid > 1
        if lay["small"] and c.name.startswith("wq9"):
            assert c.n_big > 2 * NUM_SMS  # the persistent sample loop of k_net_small
    for c in TRAIN_CASES:
        sp = train_split(c)
        if c.k == 128:
            cells.add("training K=128")
        if c.m != c.n:
            cells.add("training H != W")
        if sp["BS"] % 64 and sp["kb_total"] % sp["splits"]:
            cells.add("training B*S % 64 != 0, uneven split-K")
    want = {"k64 small net", "k64 flat", "k64 flat, sample > one M tile", "k64 per-sample", "k128 flat", "k128 per-sample",
            "k256 flat", "k256 per-sample", "H != W on tensor cores", "per-sample H != W tps=1", "per-sample H != W tps=2",
            "training K=128", "training H != W", "training B*S % 64 != 0, uneven split-K"}
    assert want <= cells, want - cells


# ---------------------------------------------------------------------------------------------------------------------
def _planes(kind, rng, nb, m, n):
    """Encoder planes of random positions: WQEncoder's 18 (stones +-1 in the history planes, a to-move plane), or the
    two-plane encoder's (+1 black / -1 white / 0.001 empty, then the to-move colour everywhere)."""
    cells = m * n
    if kind == K.GAME_WQ:
        x = np.zeros((nb, 18, cells), np.float32)
        for b in range(nb):
            for q in range(7):
                board = rng.choice([0.0, 1.0, -1.0], size=cells, p=[0.6, 0.2, 0.2])
                x[b, q], x[b, 8 + q] = board, -board
            x[b, 16 if b % 2 == 0 else 17] = 1.0 if b % 2 == 0 else -1.0
    else:
        x = np.zeros((nb, 2, cells), np.float32)
        x[:, 0] = rng.choice([0.001, 1.0, -1.0], size=(nb, cells), p=[0.5, 0.25, 0.25])
        x[:, 1] = rng.choice([1.0, -1.0], size=(nb, 1))
    return x.reshape(nb, -1)


def _desc(kind, m, n, k, layers, n_games, batch=2, flags=0, act=0):
    A = n if kind == K.GAME_C4 else m * n
    feats = 18 if kind == K.GAME_WQ else 2
    win = {K.GAME_WQ: 0, K.GAME_C4: 4, K.GAME_MNK: 5}[kind]
    d = K.make_desc(kind, m, n, win, komi=7.5 if kind == K.GAME_WQ else 0.0, sims=2, n_games=n_games, seed=2, max_moves=4,
                    flags=flags, nn=dict(k=k, shared_layers=layers, fc=32, batch_size=batch, features=feats, action_space=A + 1))
    d.act_scale_log2 = act
    return d


def _layer_ref(net, l, x):
    """Conv layer l of the float64 reference on input x: its output and the absolute-value computation
    sum over branches |A'| * (|W| (*) |x|), A' = gamma / sqrt(eps) (test-mode BatchNorm)."""
    units = [net.units[0]] if l == 0 else [net.units[2 * l - 1], net.units[2 * l]]
    out = sum(u.fwd(x, False) for u in units)
    ax = np.abs(x)
    mag = sum(np.abs(u.gamma[0]) / np.sqrt(D.EPS) * D.conv(ax, np.abs(u.w)) for u in units)
    return out, mag


def _ratio(dev, ref, mag, act):
    """per-element |dev - ref| in units of 2^-21 * (mag + |ref| + 2^-(4 + act_scale_log2))"""
    ea = act or DEFAULT_ACT_SCALE_LOG2
    return np.abs(dev.astype(np.float64) - ref) / (ULP * (mag + np.abs(ref) + 2.0 ** -(4 + ea)))


def _tower_layers(engine_lib, monkeypatch, c, act=0, env=None, seed=11):
    """Device tower output of every depth 0..L (n descending on each engine) and the per-layer ratio against the float64
    reference.  Returns (worst ratio per layer, outputs, the depth-L float64 net, planes, the depth-L engine)."""
    for key, val in dict(c.env, **(env or {})).items():
        monkeypatch.setenv(key, val)
    L = c.layers
    planes = _planes(c.kind, np.random.default_rng(seed), c.n_big, c.m, c.n)
    X = planes.reshape(c.n_big, -1, c.m, c.n).astype(np.float64)
    deep = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, L, c.n_big, act=act))
    H.tame_gammas([deep], 0, seed, target=0.9)
    src = [t for _, t in D.unpack(deep, 0)]
    net = D.Net(D.unpack(deep, 0), L)
    outs, worst = [], []
    for l in range(L + 1):
        e = deep if l == L else engine_lib.create(_desc(c.kind, c.m, c.n, c.k, l, c.n_big, act=act))
        if l < L:
            e.net_set(0, D.pack(e, src[:3 * (1 + 2 * l)] + src[-12:]))
        e.set_inferer(0, K.INF_DUAL)
        big = e.infer_tower(0, planes)
        for nn in (c.n_mid, 1):  # smaller batches after a larger one: rows beyond n are stale, never read
            small = e.infer_tower(0, planes[:nn])
            assert (small.view(np.uint32) == big[:nn].view(np.uint32)).all(), (c.name, l, nn)
        if l < L:
            e.close()
        assert np.isfinite(big).all(), (c.name, l)
        ref, mag = _layer_ref(net, l, X if l == 0 else outs[-1].astype(np.float64))
        r = _ratio(big, ref, mag, act)
        worst.append(float(r.max()))
        outs.append(big)
    fresh = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, L, c.n_big, act=act))
    fresh.net_set(0, deep.net_get(0))
    fresh.set_inferer(0, K.INF_DUAL)
    assert (fresh.infer_tower(0, planes[:1]).view(np.uint32) == deep.infer_tower(0, planes[:1]).view(np.uint32)).all(), c.name
    fresh.close()
    return worst, outs, net, planes, deep


@pytest.mark.gpu
@pytest.mark.parametrize("c", TOWER_CASES, ids=[c.name for c in TOWER_CASES])
def test_tower_layers_vs_float64(engine_lib, monkeypatch, c):
    """Every conv layer of the tensor-core tower against float64, element by element; then the float64 heads on the
    device's tower output against az_infer (k_head_convs_nhwc and heads_tiled on their own)."""
    worst, outs, net, planes, deep = _tower_layers(engine_lib, monkeypatch, c)
    p_dev, v_dev = deep.infer(0, planes)
    p_ref, v_ref = net.infer(tower=outs[-1].astype(np.float64))
    deep.close()
    rel_p = np.abs(p_dev - p_ref) / p_ref
    dv = np.abs(v_dev - v_ref)
    print("%s: worst ratio per layer %s ; heads: policy rel %.3g, value abs %.3g, pmin %.3g, |v| max %.3g" %
          (c.name, " ".join("%.3g" % w for w in worst), rel_p.max(), dv.max(), p_ref.min(), np.abs(v_ref).max()))
    assert max(worst) <= c_tower(c.k), (c.name, worst)
    assert rel_p.max() <= TOL_POLICY and dv.max() <= TOL_VALUE, (c.name, rel_p.max(), dv.max())


def _split_hi_lo(v):
    """The device's operand split of v rounded to fp32: hi = fp16(v), lo = fp16(v - hi), both returned in float64."""
    v = np.asarray(v, np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def test_bound_catches_a_dropped_pass(oracle):
    """The per-layer bound is tight enough to see a real precision loss: the fused layers of wq13-k64 without the
    lo(x) * hi(w) pass, restated in float64, must exceed it many times over.  Each layer's input is stored as the device
    stores it (x * 2^act_scale_log2 as fp16 hi + lo), its filters are taken at their per-layer power-of-two scale and
    split the same way (tc_tower_prepare), and hi(x) * (hi(w) + lo(w)) goes through the layer's affine, ReLU and branch
    add; the reference is the exact layer on the same stored input."""
    c = next(c for c in TOWER_CASES if c.name == "wq13-k64")
    e = oracle.create(_desc(c.kind, c.m, c.n, c.k, c.layers, c.n_big))
    H.tame_gammas([e], 0, 11, target=0.9)
    net = D.Net(D.unpack(e, 0), c.layers)
    e.close()
    x = _planes(c.kind, np.random.default_rng(11), c.n_big, c.m, c.n).reshape(c.n_big, -1, c.m, c.n).astype(np.float64)
    x = _layer_ref(net, 0, x)[0]
    scale = 2.0 ** DEFAULT_ACT_SCALE_LOG2
    worst = []
    for l in range(1, c.layers + 1):
        x_hi, x_lo = _split_hi_lo(x * scale)
        ref, mag = _layer_ref(net, l, (x_hi + x_lo) / scale)
        units = [net.units[2 * l - 1], net.units[2 * l]]
        ew = 7 - int(np.frexp(max(np.abs(u.w).max() for u in units))[1])  # max |w| * 2^ew in [64, 128)
        out = 0.0
        for u in units:
            w_hi, w_lo = _split_hi_lo(np.ldexp(u.w, ew))
            z = D.conv(x_hi / scale, np.ldexp(w_hi + w_lo, -ew))
            out = out + np.maximum(u.gamma[0] / np.sqrt(D.EPS) * z + u.beta[0], 0)
        worst.append(float(_ratio(out, ref, mag, 0).max()))
        x = ref
    print("%s without lo(x) * hi(w): worst ratio per fused layer %s" % (c.name, " ".join("%.3g" % w for w in worst)))
    assert min(worst) >= PASSES2_MIN_EXCESS * c_tower(c.k), worst


@pytest.mark.gpu
@pytest.mark.parametrize("act", [-5, -2, 5])
@pytest.mark.parametrize("name", ["wq9-k64-small", "wq13-k64"])
def test_tower_layers_across_activation_scales(engine_lib, monkeypatch, name, act):
    """act_scale_log2 only moves the fp16 hi/lo window of the stored activations: across -5..5 every layer stays within
    the same bound."""
    c = next(c for c in TOWER_CASES if c.name == name)._replace(n_big=6, n_mid=3)
    worst, *_, deep = _tower_layers(engine_lib, monkeypatch, c, act=act)
    deep.close()
    print("%s act_scale_log2=%d: worst ratio per layer %s" % (name, act, " ".join("%.3g" % w for w in worst)))
    assert max(worst) <= c_tower(c.k), (name, act, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["wq9-k64-small", "wq13-k64"])
def test_activation_overflow_is_reported(engine_lib, monkeypatch, name):
    """An activation scale beyond fp16's range makes the tower kernel (k_net_small, or the per-layer k_conv3x3_tc) raise
    its overflow flag: az_infer returns AZ_ERR_PANIC "activation overflow"; a fresh engine at the default scale works."""
    c = next(c for c in TOWER_CASES if c.name == name)
    planes = _planes(c.kind, np.random.default_rng(1), 4, c.m, c.n)
    for act, ok in ((20, False), (0, True)):
        e = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, 2, 4, act=act))
        H.tame_gammas([e], 0, 3, target=0.9)
        e.set_inferer(0, K.INF_DUAL)
        if ok:
            p, v = e.infer(0, planes)
            assert np.isfinite(p).all() and np.isfinite(v).all()
        else:
            with pytest.raises(K.AZError) as ei:
                e.infer(0, planes)
            assert ei.value.code == -3 and "activation overflow" in str(ei.value), str(ei.value)
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
def _train_errors(engine_lib, monkeypatch, c, scale=1.0):
    """One az_train_grads step on the tensor-core ("1") and the fp32 ("0") training path, and the float64 cost and
    gradients (Model() order) of the same step"""
    rng = np.random.default_rng(7)
    A1 = (c.n if c.kind == K.GAME_C4 else c.m * c.n) + 1
    X = (_planes(c.kind, rng, c.batch, c.m, c.n) * np.float32(scale)).astype(np.float32)
    Pi = np.zeros((c.batch, A1), np.float32)
    Pi[np.arange(c.batch), rng.integers(0, A1, c.batch)] = 1
    V = rng.choice([-1.0, 0.0, 1.0], c.batch).astype(np.float32)
    res = {}
    for tc in ("1", "0"):
        monkeypatch.setenv("AZ_TRAIN_TC", tc)
        e = engine_lib.create(_desc(c.kind, c.m, c.n, c.k, c.layers, 2, batch=c.batch, flags=K.FLAG_FP32_TOWER))
        H.tame_gammas([e], 1, 17, target=0.05)
        if tc == "1":
            net = D.Net(D.unpack(e, 1), c.layers)
            cost, grads = net.loss_grads(X.astype(np.float64).reshape(c.batch, -1, c.m, c.n), Pi.astype(np.float64),
                                         V.astype(np.float64))
            names = [e.param_desc(i)[0] for i in range(e.param_count()[0])]
        res[tc] = e.train_grads(1, X, Pi, V)
        e.close()
    return res, cost, grads, names


def _check_train(engine_lib, monkeypatch, c, scale):
    res, cost, grads, names = _train_errors(engine_lib, monkeypatch, c, scale)
    (g1, c1), (g0, c0) = res["1"], res["0"]
    assert np.isfinite(g1).all() and np.isfinite(c1), (c.name, "non-finite tensor-core gradients")
    off, bad, report = 0, [], []
    for name, g in zip(names, grads):
        sl = slice(off, off + g.size)
        off += g.size
        ref = g.ravel()
        e_tc, e_32, gmax = np.abs(g1[sl] - ref).max(), np.abs(g0[sl] - ref).max(), np.abs(ref).max()
        report.append("%s tc %.3g fp32 %.3g max %.3g" % (name, e_tc, e_32, gmax))
        if not e_tc <= C_TRAIN * e_32 + TRAIN_FLOOR * gmax:
            bad.append(name)
    assert off == g1.size
    e_tc, e_32 = abs(c1 - cost), abs(c0 - cost)
    report.append("cost tc %.3g fp32 %.3g value %.6g" % (e_tc, e_32, cost))
    print("%s x%g:\n  %s" % (c.name, scale, "\n  ".join(report)))
    assert e_tc <= C_TRAIN * e_32 + TRAIN_FLOOR * abs(cost), (c.name, e_tc, e_32)
    assert not bad, (c.name, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("c", TRAIN_CASES, ids=[c.name for c in TRAIN_CASES])
def test_train_grads_per_tensor_vs_float64(engine_lib, monkeypatch, c):
    """One training step on the wgmma GEMMs (forward, backward-data, split-K backward-filter): every Model() gradient
    within a small multiple of the fp32 CUDA-core path's own error on that tensor."""
    _check_train(engine_lib, monkeypatch, c, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("c", TRAIN_CASES, ids=[c.name for c in TRAIN_CASES])
def test_train_grads_tiny_inputs(engine_lib, monkeypatch, c):
    """Planes scaled by 2^-120: the operand exponent of a tensor that small must still give a finite power-of-two scale
    (2^133 is not a float: every zero would pack as 0 * inf = NaN), and the de-scale of the products must not flush to
    zero; the gradients stay finite and within the same criterion as at scale 1."""
    _check_train(engine_lib, monkeypatch, c, 2.0 ** -120)
