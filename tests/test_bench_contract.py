"""The committed bench lines (profiles/r0*_bench_*.json, produced by bench.py on an H100) carry every key the
measurement contract asks for.  Guards the JSON shape; the numbers themselves are measured, not tested.  The
sharded (N > 1) line is produced in the test itself, on N GPUs of the machine that runs it."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROFILES = os.path.join(ROOT, "profiles")
BASE = {"metric": str, "value": float, "unit": str, "n_gpus": int, "steps": int, "warmup": int, "ms_per_step": float,
        "higher_is_better": bool, "scaling": str, "dtype": str, "data": str, "config": dict, "e2e": dict,
        "gpu_launches": int}


def load(name):
    with open(os.path.join(PROFILES, name)) as f:
        return json.load(f)


@pytest.mark.parametrize("name", ["r01_bench_n1.json"])
def test_cuda_arm_line(name):
    d = load(name)
    for k, ty in BASE.items():
        assert isinstance(d[k], ty), k
    assert "vs_baseline" in d and d["vs_baseline"] is None          # BASELINE.md publishes no number for this metric
    assert d["unit"] == "Mvoxels/s" and d["dtype"] == "f32" and d["data"] == "synthetic" and d["higher_is_better"]
    assert "prospero" in d["config"]["workload"] and "4096" in d["config"]["workload"]
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"])
    assert d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["value"] < d["value"]
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(d["clocks"])
    assert not {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} & set(d["clocks"]["reasons"])
    r = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(r) and r["bound"] == "hbm" and r["unit"] == "GB/s"
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert d["gpu_launches"] > 0
    assert d["value"] == pytest.approx(d["config"].get("frames", 1) * (d["n_gpus"] if d["scaling"] == "weak" else 1)
                                       * 4096 * 4096 / (d["ms_per_step"] * 1e-3) / 1e6, rel=1e-6)


def test_n1_line_has_the_cpu_baseline():
    d = load("r01_bench_n1.json")
    c = d["cpu_baseline"]
    assert {"value", "unit", "cores", "kind", "sample"} <= set(c) and c["kind"] == "port" and c["cores"] >= 1
    assert d["n_gpus"] == 1 and d["scaling"] == "weak"


def test_reference_arm_line():
    d = load("r01_bench_reference_arm.json")
    assert d["impl"] == "reference" and d["unit"] == "Mvoxels/s" and d["gpu_launches"] == 0
    assert d["e2e"] == {"value": d["value"], "unit": "Mvoxels/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["cpu_baseline"]["value"] == d["value"] and d["cpu_baseline"]["kind"] == "port"


# ---- round 2 lines: N = 1 is the 2D headline (+ the strong-scaling base), N > 1 is the sharded 4096^3 volume ----
def _last_line(text):
    return json.loads([l for l in text.splitlines() if l.startswith("{")][-1])


def _r02(name):
    with open(os.path.join(PROFILES, name)) as f:
        return _last_line(f.read())


def _sharded_bench_line(n):
    """Runs bench.py --gpus n (one process per GPU, NCCL) and returns rank 0's line."""
    import torch
    if torch.cuda.device_count() < n:
        pytest.skip(f"the sharded bench needs {n} GPUs; this machine has {torch.cuda.device_count()}")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc-per-node={n}",
                          os.path.join(ROOT, "bench.py"), "--gpus", str(n), "--steps", "10", "--warmup", "3"],
                         cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stderr[-4000:]
    return _last_line(out.stdout)


def _common(d):
    for k, ty in BASE.items():
        assert isinstance(d[k], ty), k
    assert d["vs_baseline"] is None and d["unit"] == "Mvoxels/s" and d["dtype"] == "f32" and d["higher_is_better"]
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"]) and d["e2e"]["value"] < d["value"]
    assert not {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} & set(d["clocks"]["reasons"])
    r = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(r) and r["bound"] == "hbm"
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert d["gpu_launches"] > 0


def test_r02_n1_line():
    d = _r02("r02_bench_n1.json")
    _common(d)
    assert d["n_gpus"] == 1 and "2D render 4096x4096" in d["config"]["workload"]
    assert d["value"] == pytest.approx(4096 * 4096 / (d["ms_per_step"] * 1e-3) / 1e6, rel=1e-6)
    r = d["roofline"]
    # SURVEY 8(d): the headline fraction is the frame's written bytes over the whole step
    assert r["algorithmic_bytes"] == 4096 * 4096 * 4
    assert r["achieved"] == pytest.approx(r["algorithmic_bytes"] / (d["ms_per_step"] * 1e-3) / 1e9, rel=1e-6)
    assert sum(k["frame_bytes_written"] for k in r["kernels"].values()) == r["algorithmic_bytes"]
    assert {"mask_u8", "bitmap_1bit", "rgba8"} <= set(d["e2e"]["other_output_formats"])
    b = d["strong_scaling_base"]
    assert "4096^3" in b["workload"] and b["value"] == pytest.approx(4096 ** 3 / (b["ms_per_step"] * 1e-3) / 1e6, rel=1e-6)
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 4, 8])
def test_sharded_bench_line_on_n_gpus(n):
    """bench.py --gpus n, run here: the sharded 4096^3 line carries the contract's keys and a strong-scaling speed-up."""
    d = _sharded_bench_line(n)
    _common(d)
    assert d["n_gpus"] == n and d["scaling"] == "strong" and "3D render 4096^3" in d["config"]["workload"]
    assert "all-gather" in d["config"]["collective"].lower() or "allgather" in d["config"]["collective"].lower()
    assert "byte for byte" in d["config"]["identity_check"]
    assert d["value"] == pytest.approx(4096 ** 3 / (d["ms_per_step"] * 1e-3) / 1e6, rel=1e-6)
    b = d["strong_scaling_base"]
    speedup = d["value"] / b["value"]
    assert 1.0 < speedup <= n * 1.02        # a fixed workload over n ranks
