"""CPU tests of bench.py's contract pieces that do not need a GPU: the reference (CPU) arm prints ONE
JSON line with the keys the driver reads, the clock sampler degrades gracefully without NVML / a GPU,
and the engine arm refuses to run without CUDA instead of falling back."""

import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def _run(*args, timeout=300):
    return subprocess.run([sys.executable, str(ROOT / "bench.py"), *args], capture_output=True, text=True, timeout=timeout, cwd=ROOT)


def test_reference_arm_prints_one_json_line():
    r = _run("--impl", "reference", "--gpus", "1", "--steps", "1", "--warmup", "1", "--cpu-rows", "2048")
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "nsf_log_prob_samples_per_sec" and d["unit"] == "samples/s"
    assert d["higher_is_better"] is True and d["n_gpus"] == 1 and d["steps"] == 1
    assert d["value"] > 0 and d["ms_per_step"] > 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and "model" not in d["config"]


def test_engine_arm_refuses_without_cuda():
    import torch

    if torch.cuda.is_available():
        import pytest

        pytest.skip("this check is for the CPU-only build container")
    r = _run("--steps", "1")
    assert r.returncode != 0 and "no CUDA device" in (r.stderr + r.stdout)


def test_clock_sampler_without_gpu_is_harmless():
    sys.path.insert(0, str(ROOT))
    import bench

    clk = bench.ClockSampler(0).prepare()
    with clk:
        pass
    s = clk.summary()
    assert set(s) >= {"sm_mhz", "sm_max_mhz", "reasons", "samples"} and isinstance(s["reasons"], list)


def test_tensor_roofline_denominator_follows_the_clock():
    """bench.tensor_peak: the cuBLAS burst figure when the run held >= 98 % of the maximum SM clock, else that figure
    scaled to the clock actually held (a power-capped run is measured against the pipe's capacity at its clock, not
    against a 'sustained' number taken at some other clock) — never a fraction that the kind string does not explain."""
    sys.path.insert(0, str(ROOT))
    import bench

    peaks = {"bf16_tflops": 989.0, "bf16_tflops_sustained": 900.0}
    assert bench.tensor_peak(peaks, {"sm_mhz": 1980.0, "sm_max_mhz": 1980.0, "reasons": []}) == (989.0, "burst")
    assert bench.tensor_peak(peaks, {"sm_mhz": 1950.0, "sm_max_mhz": 1980.0, "reasons": ["sw_power_cap"]}) == (989.0, "burst")
    peak, kind = bench.tensor_peak(peaks, {"sm_mhz": 1680.0, "sm_max_mhz": 1980.0, "reasons": ["sw_power_cap"]})
    assert abs(peak - 989.0 * 1680.0 / 1980.0) < 1e-9 and "1680" in kind and "burst" in kind
    assert bench.tensor_peak(peaks, {}) == (989.0, "burst")  # no NVML: nothing to scale by
