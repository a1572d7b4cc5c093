"""bench.py's reference arm (`--impl reference`: the CPU oracle on the host cores) end to end on the small workload, and
the arithmetic of its roofline helper: the keys the driver parses are there, the faithful rate (every evaluation padded
to ActionSpace samples, meta.go:125-135) sits below the useful-work rate, rank > 0 prints nothing."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True, env=e, timeout=300)


def test_reference_arm_json_line():
    r = _run(["--impl", "reference", "--workload", "C2", "--steps", "3", "--warmup", "3"])
    assert r.returncode == 0, r.stderr[-500:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["metric"] == "mcts_sims_per_sec" and d["unit"] == "sims/s"
    assert d["higher_is_better"] is True and d["value"] > 0 and d["e2e"]["value"] == d["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["value"] == d["value"] and cb["cores"] >= 1 and cb["nproc"] >= cb["cores"]
    assert 0 < d["faithful_sims_per_sec"] < d["value"]           # 81 samples per evaluation instead of 1
    assert "workload" in d["config"] and "model" not in d["config"]


def test_reference_arm_other_ranks_are_silent():
    r = _run(["--impl", "reference", "--workload", "C2", "--steps", "2", "--warmup", "3", "--gpus", "2"],
             env={"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"})
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_roofline_arithmetic():
    sys.path.insert(0, ROOT)
    import bench
    w = bench.WORKLOADS["C3"]
    assert bench.flops_per_eval(w) == 17065507816      # SURVEY section 8d: 17.07 GFLOP per 19x19 20x256 evaluation
    arm = dict(prof=dict(conv_ms=800.0, conv_launches=1000.0, kernel_kind=0), cnt=dict(evals=25600), dt=1.0, workload="C3")
    r = bench.roofline_of(arm, w, {"bf16_tflops_sustained": 1465.8}, "measured")
    per_launch = 2 * 9 * 256 * 512 * 361 * 25600 * 20 / 1000.0
    assert abs(r["algorithmic_flops_per_launch"] - per_launch) < 1 and abs(r["achieved"] - per_launch * 1000 / 0.8 / 1e12) < 1e-6
    assert abs(r["frac"] - r["achieved"] / 1465.8) < 1e-12 and r["tensor_passes_per_mac"] == 3.0
    assert "wgmma" in r["kernel"] and "<BN,true>" in r["kernel"] and r["bound"] == "tensor" and r["unit"] == "TFLOP/s"
