"""CPU: bench.py's contract, exercised on CODE (not on a committed artefact): the reference arm runs here end to end (it needs no GPU) and must
print exactly one JSON line with every contract key and consistent timing arithmetic; the workload table matches BASELINE.json's configs; under
a multi-rank launch only rank 0 speaks.  The GPU arm's line is checked by the same validator in the `-m gpu` suite (tests/test_bench_gpu.py)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches")


def validate_line(d, reference=False):
    for k in BASE_KEYS + (("impl", "cpu_baseline") if reference else ("clocks", "roofline")):
        assert k in d, k
    assert d["metric"] == "env-steps/sec" and d["unit"] == "env-steps/s" and d["higher_is_better"] is True and d["scaling"] == "weak"
    assert d["vs_baseline"] is None and d["data"] == "synthetic" and d["dtype"] == "f32"
    assert "workload" in d["config"] and "model" not in d["config"] and "BASELINE.json configs[" in d["config"]["workload"]
    e = d["e2e"]
    assert e["unit"] == d["unit"] and e["value"] > 0
    if reference:
        assert d["impl"] == "reference" and e["h2d_bytes_per_step"] == 0 and e["d2h_bytes_per_step"] == 0 and e["value"] == d["value"] and d["gpu_launches"] == 0
        b = d["cpu_baseline"]
        assert b["kind"] in ("reference", "port") and b["cores"] >= 1 and b["value"] == d["value"] and b["sample"] and "plan_a" in b
    else:
        assert d["warmup"] >= 3 and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and d["gpu_launches"] > 0
        r = d["roofline"]
        assert r["bound"] in ("hbm", "tensor", "fp32-fma") and r["unit"] in ("GB/s", "TFLOP/s")
        assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
        assert abs(r["achieved"] - r["flop_per_launch"] / (r["launch_us"] * 1e-6) / 1e12) < 1e-6 * r["achieved"]
        assert set(d["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}


def _run(extra, env=None):
    t0 = time.perf_counter()
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + extra, capture_output=True, text=True, timeout=900, env={**os.environ, **(env or {})})
    return out, time.perf_counter() - t0


def test_reference_arm_prints_one_contract_line_whose_clock_fits_the_run():
    out, wall = _run(["--impl", "reference", "--steps", "2", "--warmup", "1", "--batch", "32"])
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, out.stdout
    d = json.loads(lines[0])
    validate_line(d, reference=True)
    assert d["steps"] == 2 and d["warmup"] == 1
    # the timed steps are wall clock of the whole pool: they must fit inside the caller's own clock around the run (VERDICT r1 weak #3)
    assert d["ms_per_step"] * d["steps"] / 1e3 <= wall
    assert d["cpu_baseline"]["cores"] == len(os.sched_getaffinity(0))
    # every copy stepped real episodes: 3 iterations x <= 25 steps per copy and step
    per_step = d["value"] * d["ms_per_step"] / 1e3
    assert 0 < per_step <= d["cpu_baseline"]["cores"] * 3 * 25


def test_reference_arm_other_ranks_stay_silent():
    out, _ = _run(["--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "0"], env={"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"})
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_workload_table_matches_baseline_configs():
    sys.path.insert(0, ROOT)
    import bench

    cfgs = json.load(open(os.path.join(ROOT, "BASELINE.json")))["configs"]
    for name, wl in bench.WORKLOADS.items():
        text = cfgs[wl["baseline_config"]]
        assert wl["env"].split(":")[1].rsplit("-v", 1)[0] in text, (name, text)
        assert f"{wl['envs']} " in text and wl["algo"].upper()[:4] in text.upper()
    assert bench.WORKLOADS["idqn"]["batch"] == 1024 and "batch_size=1024" in cfgs[1]
    assert bench.dims(bench.WORKLOADS["idqn"]) == (2, 15, 6) and bench.dims(bench.WORKLOADS["vdn15"]) == (4, 27, 6)
    assert bench.fwd_flop_per_row(15, 6) == 38144    # SURVEY section 8d


def test_bench_cli_parses():
    out, _ = _run(["--help"])
    assert out.returncode == 0 and "--impl" in out.stdout and "--collective" in out.stdout and "--config" in out.stdout
