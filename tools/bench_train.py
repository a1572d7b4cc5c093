#!/usr/bin/env python
"""dual.Train step (K7) timing: forward (BN train mode) + loss + backward + SGD on one batch.  3x3 layers with
K in {64,128,256} run forward / backward-data / backward-filter on the wgmma kernels (AZ_TRAIN_TC=0 forces the fp32
CUDA-core kernels of train.cu, which every other layer uses).  Prints one JSON line per shape with the algorithmic FLOPs (3 x forward) and the achieved rate."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from agogo_b200 import _capi as K  # noqa: E402

SHAPES = [
    ("C1 tic-tac-toe (K=3, 3 blocks, batch 100)", K.GAME_MNK, 3, 3, 3, dict(k=3, shared_layers=3, fc=8, batch_size=100, features=2, action_space=10)),
    ("C4 connect-4 (K=16, 6 blocks, batch 256)", K.GAME_C4, 6, 7, 4, dict(k=16, shared_layers=6, fc=32, batch_size=256, features=2, action_space=8)),
    ("C2 9x9 Go (K=64, 6 blocks, batch 256)", K.GAME_WQ, 9, 9, 0, dict(k=64, shared_layers=6, fc=128, batch_size=256, features=18, action_space=82)),
    ("C3/C5 19x19 Go (K=256, 20 blocks, batch 32)", K.GAME_WQ, 19, 19, 0, dict(k=256, shared_layers=20, fc=512, batch_size=32, features=18, action_space=362)),
    ("C5 19x19 Go at DefaultConf batch (K=256, 20 blocks, batch 256)", K.GAME_WQ, 19, 19, 0, dict(k=256, shared_layers=20, fc=512, batch_size=256, features=18, action_space=362)),
]
lib = K.load()
ONLY = sys.argv[1] if len(sys.argv) > 1 else ""   # substring filter on the shape name (e.g. C3)
for name, kind, m, n, k, nn in SHAPES:
    if ONLY not in name:
        continue
    d = K.make_desc(kind, m, n, k, komi=7.5, sims=2, n_games=2, seed=1, nn=nn, max_moves=4, flags=K.FLAG_FP32_TOWER)
    e = lib.create(d)
    e.net_init(1, 3)
    B, hw, F, A1, Kc, L, FC = nn["batch_size"], m * n, nn["features"], nn["action_space"], nn["k"], nn["shared_layers"], nn["fc"]
    rng = np.random.default_rng(0)
    X = rng.choice([0.0, 1.0, -1.0], size=(B, F * hw)).astype(np.float32)
    Pi = np.zeros((B, A1), np.float32); Pi[np.arange(B), rng.integers(0, A1, B)] = 1
    V = rng.choice([-1.0, 1.0], B).astype(np.float32)
    fwd = B * (2 * L * 2 * 9 * Kc * Kc * hw + 2 * 9 * F * Kc * hw + 2 * Kc * 3 * hw + 2 * 2 * hw * A1 + 2 * hw * FC + 2 * FC)
    e.train(1, X.copy(), Pi.copy(), V.copy(), 1, 1)  # warm-up (allocations)
    iters = 3
    t0 = time.perf_counter()
    costs = e.train(1, X.copy(), Pi.copy(), V.copy(), 1, iters)
    dt = (time.perf_counter() - t0) / iters
    print(json.dumps({"shape": name, "ms_per_step": dt * 1e3, "algorithmic_gflop_per_step": 3 * fwd / 1e9,
                      "tflops": 3 * fwd / dt / 1e12, "cost": float(costs[-1]),
                      "train_tc": os.environ.get("AZ_TRAIN_TC", "1")}), flush=True)
    e.close()
