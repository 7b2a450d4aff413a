"""CPU: the reference arm of bench.py runs here (it is the CPU port) and prints the contract's
JSON line; the GPU arm's helpers are importable."""
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def test_reference_arm_prints_contract_line():
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--workload", "cfg0",
                        "--steps", "2", "--warmup", "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step",
              "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in line, k
    assert line["impl"] == "reference" and line["unit"] == "frames/s" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["e2e"]["value"] == line["value"]
    assert line["config"]["workload"].startswith("cfg0")


def test_reference_arm_stays_bounded_at_many_steps():
    """At large step counts (the no-flag default is 100) a step becomes a plane subset of one frame, the
    metric stays per frame and the run stays within its budget."""
    import os
    env = dict(os.environ, SRCV_REF_BUDGET_S="0.02", SRCV_CPU_THREADS="2")
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--workload", "cfg0",
                        "--steps", "12", "--warmup", "3"], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    cb = line["cpu_baseline"]
    assert "planes of one frame per step" in cb["sample"] and 0 < cb["frames_per_step_timed"] < 1
    assert line["steps"] == 12 and line["value"] > 0 and line["config"]["workload"].startswith("cfg0")


def test_algorithmic_bytes_match_survey():
    sys.path.insert(0, str(ROOT))
    import bench
    from simplerecon_b200.synthetic import CONFIGS
    # SURVEY.md §8(d): cfgA 14.82 MB (dot) / 14.84 MB (hero) per frame
    assert abs(bench.algorithmic_bytes_per_frame(CONFIGS[1], False, True) - 14.82e6) < 0.02e6
    assert abs(bench.algorithmic_bytes_per_frame(CONFIGS[2], True, True) - 14.84e6) < 0.02e6
    assert abs(bench.algorithmic_bytes_per_frame(CONFIGS[3], True, True) - 17.30e6) < 0.03e6


def test_mlp_flops_match_survey_and_configs_agree_between_arms():
    sys.path.insert(0, str(ROOT))
    import bench
    from simplerecon_b200.synthetic import CONFIGS
    # SURVEY.md §8(d): 104.1 GFLOP (MLP) per frame at cfgA, 156.2 at cfgB
    assert abs(bench.mlp_flops_per_frame(CONFIGS[2], False) - 104.1e9) < 0.1e9
    assert abs(bench.mlp_flops_per_frame(CONFIGS[3], False) - 156.2e9) < 0.15e9
    # what the wgmma kernel issues: 3 MMAs per product, layer-1 K = 192 (pose measures as a bias)
    assert bench.mlp_flops_per_frame(CONFIGS[2], True) > 3 * 0.95 * bench.mlp_flops_per_frame(CONFIGS[2], False)
    # the default workload is the hero configuration at 8 frames per GPU: N = 1 is BASELINE configs[2],
    # N = 8 is configs[4]; both arms print the same `config`
    assert bench.DEFAULT_WORKLOAD == "cfg2" and bench.PER_GPU["cfg2"] == 8
    w = next(c for c in CONFIGS if c.name.startswith(bench.DEFAULT_WORKLOAD))
    c1, _ = bench.workload_config(w, bench.PER_GPU["cfg2"], 8)
    assert c1["global_batch"] == 64 and c1["matching"] == "mlp" and c1["planes"] == 64
