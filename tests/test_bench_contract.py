"""bench.py contract checks that need no GPU: the reference arm's JSON line and the byte model."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--workload", "cfg3"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "edge-feature-op/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0
    assert d["gpu_launches"] == 0


def test_reference_arm_other_ranks_stay_silent():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2"],
                         capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_gather_model_bytes():
    sys.path.insert(0, ROOT)
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    # SURVEY.md §8d: nnz*(4+s) + (N+1)*8 + nnz*C*s + N*C*s ; headline: 32M nnz, 1M nodes, 64 fp32 columns ~ 8.7 GB
    b = bench.hop_algorithmic_bytes(32_000_000, 1_000_000, 64)
    assert b == 32_000_000 * 8 + 1_000_001 * 8 + 32_000_000 * 256 + 1_000_000 * 256
    assert abs(b / (32_000_000 * 64) - 4.25) < 0.02           # 4.25 bytes per edge-feature op
    assert bench.hop_algorithmic_bytes(10, 5, 3, 8) == 10 * 12 + 6 * 8 + 10 * 24 + 5 * 24
    assert bench.WORKLOADS["er1m"]["N"] == 1_000_000 and bench.WORKLOADS["cfg2"]["B"] == 32
    # the roofline block of one hop kernel, from launch times (no GPU needed for the arithmetic)
    import types
    ctx = types.SimpleNamespace(es=4, peak=6566.7, peak_src="test", args=types.SimpleNamespace(dtype="f32"))
    rf = bench.hop_roofline(ctx, [1.0, 1.1, 0.9], 5.0 * 1, 32_000_000, 1_000_000, 64, "k")
    assert rf["bytes_per_launch"] == b and rf["launches_timed"] == 3 and abs(rf["ms_per_launch"] - 1.0) < 1e-12
    assert abs(rf["achieved"] - b / 1e-3 / 1e9) < 1e-6 and abs(rf["frac"] - rf["achieved"] / 6566.7) < 1e-12
    assert abs(rf["kernel_share_of_step"] - 0.6) < 1e-12 and rf["traffic"] is None and "dram_frac" not in rf
    assert rf["compulsory_bytes"] == 2 * 1_000_000 * 64 * 4 + 32_000_000 * 8              # 0.77 GB at the headline
    assert abs(rf["compulsory_frac"] - rf["compulsory_bytes"] / 1e-3 / 1e9 / 6566.7) < 1e-12
    # measured DRAM bytes per launch, when a capture of the workload is on file, give the DRAM fraction
    bench.load_ncu_traffic = lambda workload, dtype: 6287089304 if workload == "er1m" else None
    rf = bench.hop_roofline(ctx, [1.0], 2.0, 32_000_000, 1_000_000, 64, "k", workload="er1m")
    assert rf["traffic"] == 6287089304 and abs(rf["dram_frac"] - 6287089304 / 1e-3 / 1e9 / 6566.7) < 1e-12
    assert bench.hop_roofline(ctx, [], 1.0, 1, 1, 1, "k") is None
