"""CPU-side checks of bench.py's launch contract (the timed arms themselves need an H100 / minutes of
host time; their JSON lines are kept under tests/golden/bench_lines/)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None, timeout=120):
    e = dict(os.environ)
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True,
                          text=True, env=e, timeout=timeout, cwd=ROOT)


def test_reference_arm_other_ranks_exit_silently():
    """Under torchrun only rank 0 runs and prints the CPU arm; the other ranks exit 0 without work."""
    r = _run(["--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1"],
             env={"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"})
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_b200_arm_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    r = _run(["--steps", "1", "--warmup", "1"])
    assert r.returncode != 0
    assert "no CPU fallback" in (r.stderr + r.stdout)


@pytest.mark.parametrize("name", ["h100_bench_c3.json", "bench_reference_arm_c3.json"])
def test_committed_bench_lines_follow_the_contract(name):
    """Recorded bench.py lines (one H100 run of the GPU arm, one run of the CPU reference arm) carry
    every key a consumer of the result line reads."""
    path = os.path.join(ROOT, "tests", "golden", "bench_lines", name)
    line = json.loads(open(path).read().strip().splitlines()[-1])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step",
              "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "e2e"):
        assert k in line, k
    assert line["unit"] == "images/sec" and line["higher_is_better"] is True
    assert "workload" in line["config"] and line["scaling"] == "weak"
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in line["e2e"], k
    if line.get("impl") == "reference":
        assert line["cpu_baseline"]["kind"] in ("port", "reference") and line["e2e"]["h2d_bytes_per_step"] == 0
    else:
        assert line["gpu_launches"] > 0 and line["e2e"]["h2d_bytes_per_step"] > 0
        rf = line["roofline"]
        for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
            assert k in rf, k
        assert abs(rf["frac"] - rf["achieved"] / rf["peak"]) < 1e-9
        assert set(line["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}
        if line["n_gpus"] == 1:
            cb = line["cpu_baseline"]
            assert cb and cb["cores"] >= 1 and cb["kind"] in ("port", "reference") and cb["sample"]
