"""bench.py's host-side helpers (no GPU): the synthetic Cartesian mask has the RandomMaskGenerator structure the workload names,
the clock sampler picks the samples inside the timed window (or the replay window when the timed region is too short), and the
JSON contract keys the driver reads are spelled as in the task statement."""
import datetime
import importlib.util
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent


def _bench():
    spec = importlib.util.spec_from_file_location("bench_module", ROOT / "bench.py")
    mod = importlib.util.module_from_spec(spec)
    argv, sys.argv = sys.argv, ["bench.py"]
    try:
        spec.loader.exec_module(mod)
    finally:
        sys.argv = argv
    return mod


def test_cartesian_mask_structure():
    b = _bench()
    m = b.cartesian_mask(5, 256, 256, 4, seed=0)
    assert m.shape == (5, 2, 256, 256) and set(m.unique().tolist()) <= {0.0, 1.0}
    cols = m[:, 0, 0]
    assert torch.equal(m, cols[:, None, None, :].expand_as(m))                 # lines: constant along H, same on both planes
    assert torch.all(cols.sum(-1) == 64)                                        # 256 / 4 columns per sample
    lo = (256 - round(256 * 0.08)) // 2
    assert torch.all(cols[:, lo: lo + round(256 * 0.08)] == 1)                   # fully sampled centre band (8 % at 4x)
    assert not torch.equal(cols[0], cols[1])                                    # per-sample masks


def test_clock_sampler_selects_the_window():
    b = _bench()
    cs = b.ClockSampler(0)

    class Done:
        def terminate(self):
            pass

        def wait(self, timeout=None):
            pass

    cs.p = Done()
    t0 = datetime.datetime.now()
    for i in range(12):
        t = t0 + datetime.timedelta(milliseconds=20 * i)
        cap = "Active" if i >= 6 else "Not Active"
        cs.f.write(f"{t.strftime('%Y/%m/%d %H:%M:%S.%f')[:-3]}, {1500 + i}, 1965, {400 + i}.5, 0x4, Not Active, Not Active, Not Active, {cap}\n")
    cs.f.flush()
    ms = lambda k: t0 + datetime.timedelta(milliseconds=k)
    short, probe = ("timed region", ms(50), ms(70)), ("replay", ms(110), ms(230))
    out = cs.stop([short, probe])
    assert out["window"] == "replay" and out["samples"] == 6 and out["reasons"] == ["sw_power_cap"] and out["sm_max_mhz"] == 1965.0
    assert 1506 <= out["sm_mhz"] <= 1511


def test_bench_line_contract_of_the_committed_profile():
    """the bench line measured on the H100 (profiles/) carries every key of the contract"""
    line = json.loads((ROOT / "profiles" / "bench_h100.json").read_text())
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"):
        assert k in line, k
    assert set(("bound", "achieved", "peak", "unit", "frac", "traffic")) <= set(line["roofline"])
    assert set(("value", "unit", "cores", "kind", "sample")) <= set(line["cpu_baseline"])
    assert set(("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step")) <= set(line["e2e"])
    assert line["clocks"]["samples"] >= 3 and line["clocks"]["window"] == "timed region" and "workload" in line["config"]


def test_binding_roofline_picks_the_algorithmic_bound():
    """the roofline object counts ALGORITHMIC work against the roofline that binds it; the executed-MMA view is a sub-object.
    Numbers: the round-1 bf16 kernel as the judge recomputed it (0.72 of HBM, 0.53 of the tensor peak) and the split-operand kernel"""
    import bench

    r = bench.binding_roofline("k", 0.341, 309.237645312, 1610686464, 6569.0, 1695.9, 1.58e9, "src")
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - 0.719) < 2e-3 and abs(r["frac_tensor_algorithmic"] - 0.535) < 2e-3
    assert "tensor_pipe" not in r
    r = bench.binding_roofline("k", 0.8589, 309.237645312, 3221389312, 6569.0, 1695.9, 3197100000, "src", executed_factor=3.0)
    assert r["bound"] == "hbm" and abs(r["frac"] - 0.571) < 2e-3 and abs(r["tensor_pipe"]["frac_of_peak"] - 0.637) < 2e-3
    assert abs(r["achieved"] - 3221389312 / 1e6 / 0.8589) < 1e-6 and r["traffic"] == 3197100000
    r = bench.binding_roofline("k", 1.0, 1000.0, 1e9, 6569.0, 1695.9, None, "src")     # flop-heavy: the tensor roofline binds
    assert r["bound"] == "tensor" and r["unit"] == "TFLOP/s" and abs(r["frac"] - 1000.0 / 1695.9) < 1e-9
    for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
        assert k in r


def test_gpu_session_scripts_parse():
    """the shell drivers of the GPU sessions (tools/*.sh) need a GPU machine: at least their syntax is checked here"""
    import subprocess

    for sh in sorted((ROOT / "tools").glob("*.sh")):
        r = subprocess.run(["bash", "-n", str(sh)], capture_output=True, text=True)
        assert r.returncode == 0, (sh.name, r.stderr)


def test_bench_config_names_the_split_under_strong_scaling():
    import bench

    weak = bench.bench_config("cfg2", 4, "weak")
    strong = bench.bench_config("cfg2", 4, "strong")
    assert weak["global_batch"] == 256 and "batch=64 per GPU" in weak["workload"]
    assert strong["global_batch"] == 64 and "16 per GPU" in strong["workload"] and "per GPU" in strong["workload"]
    assert bench.bench_config("cfg2", 1, "strong") == bench.bench_config("cfg2", 1, "weak")
