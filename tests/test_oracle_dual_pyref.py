"""oracle/dual.hpp (fp32) against the independent numpy float64 restatement of the dual network (tests/pyref_dual.py):
inference outputs (BatchNorm in test mode, batch row 0 of the batch-shaped parameters, softmax / tanh) and one training
step's cost and every Model() gradient (BatchNorm in train mode with batch-shaped affine, cross-entropy on the raw
logits, MSE on the pre-tanh value).  Parity with gorgonia itself stays unpinned (DESIGN.md §2); this pins the oracle to
the four stated assumptions."""
import numpy as np
import pytest

from agogo_b200 import _capi as K
from tests import helpers as H
from tests import pyref_dual as D

# one training step of the fp32 oracle against float64: every tensor (every batch row of a batch-shaped one) within
# TOL_GRAD of its own largest gradient, the cost within TOL_COST relative.  Measured at most 1.4e-6 and 6.2e-7.
TOL_GRAD, TOL_COST = 6e-6, 2.5e-6

@pytest.mark.parametrize("kind,m,n,k,nn", [
    (K.GAME_MNK, 3, 3, 3, dict(k=3, shared_layers=3, fc=8, batch_size=6, features=2, action_space=10)),
    (K.GAME_C4, 6, 7, 4, dict(k=5, shared_layers=2, fc=12, batch_size=4, features=2, action_space=8)),
    (K.GAME_WQ, 5, 5, 0, dict(k=4, shared_layers=1, fc=6, batch_size=3, features=18, action_space=26)),
])
def test_dual_forward_and_gradients_vs_numpy(oracle, kind, m, n, k, nn):
    e = oracle.create(K.make_desc(kind, m, n, k, sims=2, n_games=2, seed=1, nn=nn))
    H.tame_gammas([e], 1, 17, target=0.05)
    rng = np.random.default_rng(3)
    B, F, A1 = nn["batch_size"], nn["features"], nn["action_space"]
    net = D.Net(D.unpack(e, 1), nn["shared_layers"])
    # ---- training step: cost and gradients
    X = rng.choice([0.001, 1.0, -1.0], size=(B, F, m, n))
    Pi = np.zeros((B, A1)); Pi[np.arange(B), rng.integers(0, A1, B)] = 1
    V = rng.choice([-1.0, 0.0, 1.0], B)
    go, co = e.train_grads(1, X.astype(np.float32).reshape(B, -1), Pi.astype(np.float32), V.astype(np.float32))
    cost, grads = net.loss_grads(X, Pi, V)
    assert abs(co - cost) <= TOL_COST * abs(cost), (co, cost)
    # every tensor on its own scale, the batch-shaped ones (BatchNorm scale / bias, the linear biases) per batch row
    worst = []
    for i, g in enumerate(grads):
        name, shape, off, size = e.param_desc(i)
        d = np.abs(go[off:off + size].reshape(g.shape) - g)
        rows = B if shape[0] == B and (name.endswith(("_γ", "_β")) or name.endswith("_b")) else 1
        dm, gm = d.reshape(rows, -1).max(1), np.abs(g).reshape(rows, -1).max(1)
        # a row whose reference is all zero (every unit of the sample rectified away) must be exactly zero
        r = np.where(gm > 0, dm / np.where(gm > 0, gm, 1.0), np.where(dm > 0, np.inf, 0.0))
        worst.append((float(r.max()), name))
    print("worst per-tensor gradient ratio %.3g (%s), cost %.3g" % (*max(worst), abs(co - cost) / abs(cost)))
    assert max(worst)[0] <= TOL_GRAD, sorted(worst)[-3:]
    # ---- inference (test-mode BatchNorm needs gains that keep 316x per layer finite: tame to ~1)
    H.tame_gammas([e], 0, 19, target=0.9)
    e.set_inferer(0, K.INF_DUAL)
    net0 = D.Net(D.unpack(e, 0), nn["shared_layers"])
    Xi = rng.choice([0.0, 1.0, -1.0], size=(5, F, m, n))
    po, vo = e.infer(0, Xi.astype(np.float32).reshape(5, -1))
    pn, vn = net0.infer(Xi)
    assert np.abs(po - pn).max() < 2e-5 and np.abs(vo - vn).max() < 2e-5, (np.abs(po - pn).max(), np.abs(vo - vn).max())
    # ---- the tower output (az_infer_tower): NCHW [n,K,H,W], the activations the heads read
    to = e.infer_tower(0, Xi.astype(np.float32).reshape(5, -1))
    tn = net0.tower
    assert to.shape == tn.shape == (5, nn["k"], m, n), (to.shape, tn.shape)
    assert np.abs(to - tn).max() <= 1e-6 * np.abs(tn).max(), (np.abs(to - tn).max(), np.abs(tn).max())
