"""bench.py --dump-outputs: two runs with the same arguments write identical files.  The default
arm is the production one -- bf16, CUDA graph, deterministic left at its default, so wgrad and the
SK / SE GEMMs run split-K with ordered reductions -- and every dumped buffer must match bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bench_dump_outputs_identical_across_runs(tmp_path):
    dirs = []
    for run in range(2):
        d = tmp_path / ("run%d" % run)
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps",
                            "2", "--warmup", "1", "--batch", "32", "--no-cpu-baseline",
                            "--dump-outputs", str(d)],
                           cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-4000:])
        dirs.append(d)
    names = sorted(os.listdir(dirs[0]))
    assert "loss.npy" in names and "grads_sample.npy" in names, names
    assert names == sorted(os.listdir(dirs[1]))
    for n in names:
        a, b = np.load(dirs[0] / n), np.load(dirs[1] / n)
        assert a.shape == b.shape and np.array_equal(a, b), n
