"""bench.py contract pieces that run without a GPU: the reference arm's JSON line and the clock sampler's parsing."""
import datetime
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_reference_arm_prints_the_contract_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "ngp_lego_train_rays_per_s" and line["unit"] == "rays/s"
    assert line["higher_is_better"] is True and line["steps"] == 1 and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1 and line["cpu_baseline"]["value"] == line["value"]
    assert line["e2e"] == {"value": line["value"], "unit": "rays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert line["gpu_launches"] == 0


def test_reference_arm_other_ranks_exit_quietly():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1"],
                       capture_output=True, text=True, timeout=120, env=dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1"))
    assert r.returncode == 0 and r.stdout.strip() == ""


def test_clock_sampler_selects_the_timed_window():
    import bench
    cs = bench.ClockSampler(0)
    cs.proc = type("P", (), {"terminate": lambda self: None})()
    cs.t = type("T", (), {"join": lambda self, timeout=None: None})()
    t0 = datetime.datetime(2026, 1, 2, 3, 4, 5).timestamp()

    def row(dt, sm, cap="Not Active"):
        ts = datetime.datetime.fromtimestamp(t0 + dt).strftime("%Y/%m/%d %H:%M:%S.%f")[:-3]
        return f"{ts}, {sm}, 1965, 700.0, 0x0, Not Active, Not Active, Not Active, {cap}\n"

    cs.lines = [row(-1.0, 300), row(-0.5, 1200)] + [row(0.01 * k, 1950 + k) for k in range(1, 8)] + [row(2.0, 400, "Active")]
    out = cs.stop(t0, t0 + 0.1)
    assert out["window"] == "timed region" and out["samples"] == 7 and out["sm_mhz"] == 1954 and out["sm_max_mhz"] == 1965 and out["reasons"] == []
    cs.lines = [row(-1.0, 1900, "Active"), row(5.0, 1910)]
    out = cs.stop(t0, t0 + 0.1)                                  # too few samples inside: falls back to everything under load
    assert out["window"] != "timed region" and out["samples"] == 2 and out["reasons"] == ["sw_power_cap"]


class _FakeEvent:
    def __init__(self, enable_timing=True):
        pass

    def record(self, *a, **k):
        pass

    def elapsed_time(self, other):
        return 1.0


def _run_ours_on_cpu(monkeypatch, capsys, argv):
    """bench.run_ours end to end with the operator layer swapped for the oracle (tests/cpu_backend.py): the control flow, the
    argument handling and every key of the JSON line -- numbers are meaningless (fake CUDA events)."""
    import argparse
    import torch
    import cpu_backend
    import bench
    cpu_backend.install(monkeypatch)
    from jnerf_b200 import runner as R
    from jnerf_b200.plugin.sampler import DensityGridSampler
    for name in ("lego_cfg", "fox_cfg"):                                  # 32 rays per batch: the scalar oracle marches them in milliseconds
        orig = getattr(R, name)
        monkeypatch.setattr(R, name, lambda _o=orig, **k: _o(**dict(k, n_rays_per_batch=32)))
    monkeypatch.setattr(DensityGridSampler, "update_density_grid", lambda self: self.update_density_grid_nerf(0.95, 20000, 0))
    monkeypatch.setattr(torch.cuda, "set_device", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "Event", _FakeEvent)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    st = bench.stage_times
    monkeypatch.setattr(bench, "stage_times", lambda r, n: st(r, 2))
    monkeypatch.setattr(sys, "argv", ["bench.py"] + argv)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    monkeypatch.delenv("RANK", raising=False)
    bench.main()
    return json.loads(capsys.readouterr().out.strip().splitlines()[-1])


def test_our_arm_control_flow_and_json_keys(monkeypatch, capsys):
    line = _run_ours_on_cpu(monkeypatch, capsys, ["--steps", "2", "--warmup", "1", "--pretrain", "1", "--images", "3", "--res", "24", "--target-batch", "16384",
                                                  "--no-cpu-baseline"])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config",
              "e2e", "gpu_launches", "clocks", "roofline", "iters_per_s", "samples_per_s"):
        assert k in line, k
    assert line["metric"] == "ngp_lego_train_rays_per_s" and line["unit"] == "rays/s" and line["n_gpus"] == 1 and line["steps"] == 2
    assert line["scaling"] == "weak" and line["dtype"] == "f16" and line["data"] == "synthetic" and line["vs_baseline"] is None
    assert line["config"]["target_batch_size"] == 16384 and "lego" in line["config"]["workload"] and "3 synthetic 24x24 views" in line["config"]["workload"]
    assert line["config"]["parallelism"] == "dp1"
    assert set(line["e2e"]) >= {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} and line["e2e"]["h2d_bytes_per_step"] > 0
    roof = line["roofline"]
    assert roof["bound"] == "hbm" and roof["unit"] == "GB/s" and roof["kernel"] in ("network_fwd", "network_bwd") and roof["peak"] > 0
    assert set(roof["stage_ms"]) == {"prepare_batch", "march", "network_fwd", "composite_loss_bwd", "network_bwd", "adam_ema"}
    assert roof["algorithmic_bytes_per_sample"] in (624, 1124) and "tensor" in roof


def test_our_arm_fox_workload(monkeypatch, capsys):
    line = _run_ours_on_cpu(monkeypatch, capsys, ["--steps", "1", "--warmup", "1", "--pretrain", "1", "--images", "3", "--res", "18", "--workload", "fox",
                                                  "--target-batch", "16384", "--no-cpu-baseline"])
    assert line["metric"] == "ngp_fox_train_rays_per_s" and "ngp_fox.py" in line["config"]["workload"] and "18x32 views" in line["config"]["workload"]


def test_sweep_summary_from_a_committed_bench_line():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sweep
    line = json.load(open(os.path.join(ROOT, "tests", "golden", "bench_line_h100.json")))    # bench.py --gpus 1 --steps 1000, H100, this build
    row = sweep.summarise(18, 1, line)
    assert row["log2_target"] == 18 and row["gpus"] == 1 and abs(row["iters_per_s"] - line["iters_per_s"]) < 1e-9
    n = line["roofline"]["samples_per_launch"]
    assert abs(row["bwd_gbs"] - n * 1124 / (line["roofline"]["stage_ms"]["network_bwd"] * 1e-3) / 1e9) < 1e-6
    assert abs(row["fwd_gbs"] - n * 624 / (line["roofline"]["stage_ms"]["network_fwd"] * 1e-3) / 1e9) < 1e-6
    dom = {"network_fwd": "fwd_gbs", "network_bwd": "bwd_gbs"}[line["roofline"]["kernel"]]
    assert abs(row[dom] - line["roofline"]["achieved"]) < 1e-3 * line["roofline"]["achieved"]      # the same number bench.py reports
    assert sweep.summarise(16, 2, {"error": "x" * 1000, "returncode": 1})["error"] == "x" * 300
