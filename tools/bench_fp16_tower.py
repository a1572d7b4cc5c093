"""Default (three-pass hi/lo) against AZ_FLAG_FP16_TOWER (one fp16 pass) on the bench workloads, in one process.

For C3 and C2, the two modes run alternately, `--pairs` pairs each, on the device-timed wave region of bench.py
(az_profile region time over `--steps` MCTS waves after `--warmup`).  C2's small net is launch bound, so it is timed as
bench.py times kind 5 — enable=2, the captured wave graph replayed with no events inside — and here that applies to
kinds 5 and 7; C3 is timed with per-launch events, which also give the fused-layer launch time.  One JSON line per run:
sims/s, ms per fused-layer launch (C3), kernel_kind, the probe outputs' max policy relative difference and |delta value|
between the two modes, and the card's name, power limit and SM clock read in the same call."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from agogo_b200 import _capi as K  # noqa: E402
from bench import WORKLOADS, make_desc, probe_planes, setup_nets  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], check=True,
                         capture_output=True, text=True).stdout.splitlines()[0]
    name, power, clock = [s.strip() for s in out.split(",")]
    return dict(gpu=name, power_limit=power, sm_clock=clock)


def run(lib, wl, flags, steps, warmup, probe):
    w = dict(WORKLOADS[wl])
    e = lib.create(make_desc(w, w["n_games"], 0, 1000, flags=flags))
    setup_nets(e, 1000)
    e.arena_begin(w["n_games"], False)
    state = {"in": False, "left": 0}

    def step():
        if not state["in"]:
            e.search_begin()
            state["in"], state["left"] = True, w["sims"]
            return
        e.search_run(1)
        state["left"] -= 1
        if state["left"] == 0:
            e.search_end()
            state["in"] = False

    for _ in range(warmup):
        step()
    e.profile(True)
    kind = e.profile(False)["kernel_kind"]
    e.counters_reset()
    e.counters()  # synchronises the engine's stream
    e.profile(2 if kind in (5, 7) else 1)
    for _ in range(steps):
        step()
    prof = e.profile(False)
    cnt = e.counters()
    if state["in"]:
        e.search_run(state["left"])
        e.search_end()
    e.arena_finish()
    p, v = e.infer(0, probe)
    e.close()
    res = dict(workload=wl, mode="fp16" if flags & K.FLAG_FP16_TOWER else "default", kernel_kind=kind,
               sims_per_s=cnt["sims"] / (prof["region_ms"] / 1e3), region_ms=prof["region_ms"], steps=steps)
    if prof["conv_launches"]:
        res["ms_per_fused_launch"] = prof["conv_ms"] / prof["conv_launches"]
    return res, (p, v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C3,C2")
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    lib = K.load()
    for wl in args.workloads.split(","):
        probe = probe_planes(WORKLOADS[wl], 16)
        for pair in range(args.pairs):
            outs = {}
            lines = []
            for flags in (0, K.FLAG_FP16_TOWER):
                res, outs[flags] = run(lib, wl, flags, args.steps, args.warmup, probe)
                res.update(card(), pair=pair)
                lines.append(res)
            (p0, v0), (p1, v1) = outs[0], outs[K.FLAG_FP16_TOWER]
            on = p0 > 0  # an untrained net can give exact zeros; those entries have no relative difference
            diff = dict(probe_policy_max_rel=float((np.abs(p1.astype(np.float64) - p0)[on] / p0[on]).max()),
                        probe_policy_max_abs=float(np.abs(p1.astype(np.float64) - p0).max()),
                        probe_value_max_abs=float(np.abs(v1.astype(np.float64) - v0).max()))
            for res in lines:
                print(json.dumps(dict(res, **diff)), flush=True)


if __name__ == "__main__":
    main()
