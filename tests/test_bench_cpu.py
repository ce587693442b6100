"""CPU: the host-side arithmetic of bench.py (no GPU, no library call): algorithmic FLOP per ray of SURVEY.md 8(d), the roofline object
assembled from per-launch timings, the per-workload DRAM-traffic entry, the JSON-line contract of the reference arm's workloads."""
import ctypes as C
import json
import os
import sys

from conftest import ROOT

sys.path.insert(0, ROOT)
import bench  # noqa: E402


def test_algorithmic_flop_per_ray_matches_the_survey():
    w = bench.WORKLOADS
    assert abs(bench.flop_per_ray(w["C2"]) / 1e9 - 4.66) < 0.01          # SURVEY.md 8(d): 4.66 GFLOP per ray at C2
    assert abs(bench.flop_per_ray(w["C2"]) * 8192 / 1e12 - 38.2) < 0.05   # 38.2 TFLOP per 8192-ray step
    assert abs(bench.flop_per_ray(w["C3"]) / 1e9 - 4.99) < 0.01
    assert abs(bench.flop_per_ray(w["C1"]) / 1e9 - 2.93) < 0.01
    assert bench.F_SDF_VALUE == 4195328 - 2 * 512 * 512


def test_roofline_object_from_launch_timings():
    out5 = (C.c_double * 5)(200.0, 80e12, 160e12, 1000.0, 600e9)          # 2 steps: ms, flop, MMA flop, launches, bytes
    r = bench.roofline_from_timing(None, out5, 2, 110.0, 38.2e12, 1409.5, "test")
    assert r["bound"] == "tensor" and r["unit"] == "TFLOP/s" and r["peak"] == 1409.5
    assert abs(r["kernel_ms_per_step"] - 100.0) < 1e-9 and abs(r["achieved"] - 400.0) < 1e-6
    assert abs(r["frac"] - 400.0 / 1409.5) < 1e-9 and abs(r["share_of_step"] - 100.0 / 110.0) < 1e-9
    assert abs(r["mma_tflops_incl_split_products"] - 800.0) < 1e-6 and r["launches_per_step"] == 500.0
    assert abs(r["algorithmic_hbm_gbs_in_kernel"] - 3000.0) < 1e-6
    assert abs(r["step_level"]["frac"] - 38.2e12 / 0.110 / 1e12 / 1409.5) < 1e-9
    r5 = bench.roofline_from_timing(None, out5, 2, 110.0, 38.2e12, 1409.5, "test", workload="C5")
    assert "sdf_fused_kernel" in r5["kernel"]


def test_roofline_traffic_entry_per_workload(tmp_path, monkeypatch):
    """a DRAM-traffic capture file, when present, is read per workload (top level = the training workloads)"""
    out5 = (C.c_double * 5)(200.0, 80e12, 160e12, 1000.0, 600e9)
    monkeypatch.setattr(bench, "NCU_TRAFFIC", str(tmp_path / "absent.json"))
    assert bench.roofline_from_timing(None, out5, 2, 110.0, 38.2e12, 989.0, "test")["traffic"] is None
    t = {"dram_bytes_per_launch": 1000, "source": "s2", "kernel": "k2", "C5": {"dram_bytes_per_launch": 50, "source": "s5", "kernel": "k5"}}
    p = tmp_path / "gemm_traffic.json"
    p.write_text(json.dumps(t))
    monkeypatch.setattr(bench, "NCU_TRAFFIC", str(p))
    r = bench.roofline_from_timing(None, out5, 2, 110.0, 38.2e12, 989.0, "test")
    assert (r["traffic"], r["traffic_source"], r["traffic_kernel"]) == (1000, "s2", "k2")
    r5 = bench.roofline_from_timing(None, out5, 2, 110.0, 38.2e12, 989.0, "test", workload="C5")
    assert (r5["traffic"], r5["traffic_source"], r5["traffic_kernel"]) == (50, "s5", "k5")


def test_workload_table_names_the_baseline_configs():
    assert set(bench.WORKLOADS) == {"C1", "C2", "C3", "C5"}
    assert bench.WORKLOADS["C2"]["rays"] == 8192 and "8192 rays x 128 samples" in bench.WORKLOADS["C2"]["name"]
    assert bench.WORKLOADS["C5"]["dim"] == 512
    assert bench.DEFAULT_PRECISION in bench.DTYPES
