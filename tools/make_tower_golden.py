#!/usr/bin/env python
"""Regenerates tests/golden/tower_c3_bits.npz: the exact bits the tensor-core kernels produce at the headline width.

  * inference: the 20 x 256 tower on 19x19 (seeded net, BN scales with the spread of the bench nets) through the heads,
    for n in {1, 3, 64, 512} positions per launch (odd and even M-tile counts, one to many tiles per CTA);
  * training: the parameters after one dual.Train step (K = 256, 19x19, batch 4), which runs the conv kernel in its raw
    (fp32 output) mode for the forward and backward-data passes and the backward-filter kernel.

Every array is stored as the sha256 of its bytes; the outputs for n <= 3 are also stored in full so that a mismatch can
be read.  Changes to the kernels' pipelining must leave all of these bits as they are (the per-accumulator sequence of
MMAs is the same).  Needs a GPU; --lib selects the library to run (default: the in-tree build)."""
import argparse
import hashlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from agogo_b200 import _capi as K  # noqa: E402
from tests import helpers as H  # noqa: E402

SIZES = (1, 3, 64, 512)
FULL_UP_TO = 3


def _sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def _planes(rng, n):
    x = np.zeros((n, 18, 361), np.float32)
    for b in range(n):
        for q in range(7):
            board = rng.choice([0.0, 1.0, -1.0], size=361, p=[0.6, 0.2, 0.2]).astype(np.float32)
            x[b, q] = board
            x[b, 8 + q] = -board
        x[b, 16 + (b & 1)] = 1.0
    return x.reshape(n, -1)


def compute(lib):
    out = {}
    d = K.make_desc(K.GAME_WQ, 19, 19, 0, komi=7.5, sims=2, n_games=max(SIZES), seed=2, max_moves=4,
                    nn=dict(k=256, shared_layers=20, fc=512, batch_size=2, features=18, action_space=362))
    e = lib.create(d)
    H.tame_gammas([e], 0, 5, target=1.0396)
    e.set_inferer(0, K.INF_DUAL)
    planes = _planes(np.random.default_rng(8), max(SIZES))
    for n in SIZES:
        p, v = e.infer(0, planes[:n])
        out["infer%d_policy_sha" % n] = _sha(p)
        out["infer%d_value_sha" % n] = _sha(v)
        if n <= FULL_UP_TO:
            out["infer%d_policy" % n] = p
            out["infer%d_value" % n] = v
    e.close()

    nn = dict(k=256, shared_layers=2, fc=64, batch_size=4, features=18, action_space=362)
    d = K.make_desc(K.GAME_WQ, 19, 19, 0, komi=7.5, sims=2, n_games=2, seed=1, nn=nn, max_moves=4, flags=K.FLAG_FP32_TOWER)
    e = lib.create(d)
    H.tame_gammas([e], 1, 23, target=0.05)
    rng = np.random.default_rng(5)
    X = rng.choice([0.001, 1.0, -1.0], size=(4, 18 * 361)).astype(np.float32)
    Pi = np.zeros((4, 362), np.float32)
    Pi[np.arange(4), rng.integers(0, 362, 4)] = 1
    V = rng.choice([-1.0, 0.0, 1.0], 4).astype(np.float32)
    costs = e.train(1, X, Pi, V, 1, 1, lr=0.1, shuffle_seed=0)
    out["train_cost"] = costs
    out["train_params_sha"] = _sha(e.net_get(1))
    e.close()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="libagogo_b200.so to run (default: the in-tree build)")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "tower_c3_bits.npz"))
    args = ap.parse_args()
    res = compute(K.load(args.lib) if args.lib else K.load())
    np.savez_compressed(args.out, **res)
    print({k: (v.shape, v.dtype.str) for k, v in res.items()})
