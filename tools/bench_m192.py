"""The fused layers on 192-row tiles (default, kernel_kind 8) against the 128-row kernel (AZ_TC_M192=0, kind 0), in one
process.

For each workload the two settings run alternately, `--pairs` pairs each, on bench.py's device-timed wave region
(az_profile with per-launch events over `--steps` MCTS waves after `--warmup`).  One JSON line per run: sims/s, ms per
fused-layer launch, kernel_kind, whether the probe outputs of the pair are bit-identical, and the card's name, power
limit and SM clock read in the same call."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from agogo_b200 import _capi as K  # noqa: E402
from bench import WORKLOADS, probe_planes  # noqa: E402
from bench_fp16_tower import card, run  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C3")
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    lib = K.load()
    for wl in args.workloads.split(","):
        probe = probe_planes(WORKLOADS[wl], 16)
        for pair in range(args.pairs):
            outs, lines = {}, []
            for flag in ("0", "1"):
                os.environ["AZ_TC_M192"] = flag  # read when the engine allocates its tower
                res, outs[flag] = run(lib, wl, 0, args.steps, args.warmup, probe)
                res.update(card(), pair=pair, AZ_TC_M192=flag)
                res.pop("mode")
                lines.append(res)
            same = all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(outs["0"], outs["1"]))
            for res in lines:
                print(json.dumps(dict(res, probe_bits_equal=same)), flush=True)


if __name__ == "__main__":
    main()
