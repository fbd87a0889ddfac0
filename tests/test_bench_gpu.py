"""GPU: the GPU arm of bench.py prints one line that satisfies the contract validator, for the default workload (shrunk) and the two
secondary configs (shrunk); e2e crosses host buffers; --dump-outputs writes the same arrays on every run with the same arguments."""
import json
import os
import subprocess
import sys

import pytest

from tests.test_bench_contract import validate_line

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("cfg,extra", [("idqn", ["--envs", "256", "--batch", "64", "--buffer", "1024"]), ("vdn15", ["--envs", "128", "--batch", "32", "--buffer", "512"]),
                                       ("ia2c", ["--envs", "512"])])
def test_b200_arm_line(cfg, extra):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--config", cfg, "--steps", "2", "--warmup", "3", "--no-cpu-baseline"] + extra,
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, out.stdout
    d = json.loads(lines[0])
    validate_line(d)
    assert d["n_gpus"] == 1 and d["env_steps_timed"] > 0
    assert 0.2 * d["value"] < d["e2e"]["value"] <= 1.1 * d["value"]


@pytest.mark.parametrize("cfg,extra", [("idqn", ["--envs", "256", "--batch", "64", "--buffer", "1024"]), ("ia2c", ["--envs", "512"])])
def test_dump_outputs_repeat_exactly(cfg, extra, tmp_path):
    import numpy as np

    dumps = []
    for run in range(2):
        d = tmp_path / f"run{run}"
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--config", cfg, "--steps", "2", "--warmup", "3", "--no-cpu-baseline", "--no-e2e",
                              "--dump-outputs", str(d)] + extra, capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr[-3000:]
        dumps.append({f.stem: np.load(f) for f in sorted(d.glob("*.npy"))})
    assert "theta" in dumps[0] and "metrics" in dumps[0] and "episode_length" in dumps[0]
    assert sum(a.nbytes for a in dumps[0].values()) <= 64 << 20
    assert dumps[0].keys() == dumps[1].keys()
    for name, a in dumps[0].items():
        assert a.dtype == np.float32 and np.array_equal(a, dumps[1][name]), name
