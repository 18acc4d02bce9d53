"""bench.py pieces that run without a GPU: the reference arm's JSON line (the contract the driver parses), the
roofline helpers and the clock-sample reduction.  The GPU arm itself needs the device."""
import json
import os
import subprocess
import sys
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    env = dict(os.environ, BENCH_CPU_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                        "--ref-frames", "2"], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "images/sec" and d["unit"] == "images/s"
    assert d["higher_is_better"] is True and d["vs_baseline"] is None and d["data"] == "synthetic"
    assert d["value"] > 0 and d["ms_per_step"] > 0 and d["steps"] == 1
    assert d["config"]["workload"] == "posenet_bs64"
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "frame" in cb["sample"]
    assert d["e2e"] == {"value": d["value"], "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


def test_b200_arm_refuses_to_run_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1"], capture_output=True, text=True,
                       timeout=600, cwd=ROOT)
    assert r.returncode != 0 and "no CPU fallback" in (r.stderr + r.stdout)


def test_roofline_helpers_and_clock_reduction():
    sys.path.insert(0, ROOT)
    import bench
    p = bench._peaks()
    assert p["tc_sustained"] > 100 and p["hbm"] > 1000 and p["src"] in ("measured", "datasheet")
    t = bench._ncu_traffic()
    assert t is None or (t["dram_bytes_per_launch"] > 0 and t["kernel"].startswith("k_tc_"))
    assert bench.usable_cores() >= 1
    assert bench.frames(bench.WORKLOADS["mapnetpp_n16t10"]) == 160 and bench.frames(bench.WORKLOADS["mapnet_n32t3"]) == 96
    s = bench.ClockSampler(0)
    now = time.time()
    s.rows = [(now + 0.1 * i, ["1965", "1965", "700.0", "Not Active", "Not Active", "Not Active",
                               "Active" if i == 2 else "Not Active"]) for i in range(5)]
    s.rows.append((now + 100.0, ["210", "1965", "90.0", "Active", "Not Active", "Not Active", "Not Active"]))   # outside the window
    out = s.summary(now, now + 0.5)
    assert out["sm_mhz"] == 1965.0 and out["sm_max_mhz"] == 1965.0 and out["reasons"] == ["sw_power_cap"] and out["samples"] == 5


def test_ncu_summary_tool_on_a_sample_report(tmp_path):
    """tools/ncu_summary.py (turns an `ncu --set full` report into profiles/<tag>_ncu_full_summary.csv and the
    roofline.traffic source) against one of the reports Nsight Compute ships as samples."""
    import glob
    reps = sorted(glob.glob("/opt/nvidia/nsight-compute/*/extras/samples/instructionMix/sobelFloat.ncu-rep"))
    import shutil
    if not reps or shutil.which("ncu") is None:
        pytest.skip("no Nsight Compute sample report / ncu on this machine")
    env = dict(os.environ, NCU_SUMMARY_OUT=str(tmp_path), NCU_SUMMARY_PREFIX="Sobel")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_summary.py"), reps[0], "t"], capture_output=True,
                       text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stderr[-1500:]
    lines = open(tmp_path / "t_ncu_full_summary.csv").read().splitlines()
    assert lines[0].startswith("#") and lines[1].startswith("kernel,dur_ns,")
    cols = lines[1].split(",")
    row = dict(zip(cols, lines[2].split(",")))
    assert float(row["dur_ns"]) > 1000 and float(row["dram_read_bytes"]) > 1e5 and "tensor_pipe_pct_active" in cols
    t = json.load(open(tmp_path / "ncu_traffic.json"))
    assert t["dram_bytes_per_launch"] > 1e5 and t["launches_captured"] >= 1


def test_ncu_stall_summary_tool_on_a_sample_report(tmp_path):
    import glob
    import shutil
    reps = sorted(glob.glob("/opt/nvidia/nsight-compute/*/extras/samples/instructionMix/sobelFloat.ncu-rep"))
    if not reps or shutil.which("ncu") is None:
        pytest.skip("no Nsight Compute sample report / ncu on this machine")
    src = subprocess.run(["ncu", "-i", reps[0], "--page", "source", "--csv"], capture_output=True, text=True, timeout=300)
    assert src.returncode == 0
    (tmp_path / "s.csv").write_text(src.stdout)
    env = dict(os.environ, NCU_SUMMARY_OUT=str(tmp_path))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_stalls.py"), str(tmp_path / "s.csv"), "t", "top=5"],
                       capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0, r.stderr[-1500:]
    txt = open(tmp_path / "t_ncu_stalls.txt").read()
    assert "Sobel" in txt and "long_sb" in txt and txt.count("%") > 10
