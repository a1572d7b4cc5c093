#!/usr/bin/env python
"""Two (or more) ranks, a small c4 net, a few data-parallel az_train steps through the fused peer-memory all-reduce + SGD
kernel:
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/k8_small.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from agogo_b200 import _capi as K  # noqa: E402

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
lib = K.load()
d = K.make_desc(K.GAME_C4, 6, 7, 4, sims=4, n_games=2, seed=1, device=lr, flags=K.FLAG_FP32_TOWER,
                nn=dict(k=16, shared_layers=2, fc=32, batch_size=16, features=2, action_space=8))
e = lib.create(d)
e.net_init(1, 7)
uid = K.comm_unique_id(lib)
t = torch.tensor(list(uid), dtype=torch.uint8).cuda()
dist.broadcast(t, 0)
e.comm_init(rank, world, bytes(t.cpu().tolist()))
rng = np.random.default_rng(3 + rank)
X = rng.choice([0.001, 1.0, -1.0], size=(32, 2 * 42)).astype(np.float32)
Pi = np.zeros((32, 8), np.float32); Pi[np.arange(32), rng.integers(0, 8, 32)] = 1
V = rng.choice([-1.0, 1.0], 32).astype(np.float32)
costs = e.train(1, X, Pi, V, 2, 2)
p = torch.from_numpy(e.net_get(1)).cuda()
ref = p.clone()
dist.broadcast(ref, 0)
assert torch.equal(p, ref), "replicas diverged"
if rank == 0:
    print("k8_small ok: world %d, costs %s" % (world, np.round(costs, 5).tolist()))
dist.barrier()
e.close()
dist.destroy_process_group()
