"""The committed bench lines (profiles/h100_bench_n1.json = `python bench.py`, h100_bench_reference_arm.json =
`python bench.py --impl reference`) carry every key of the bench contract and are internally consistent."""
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
  with open(os.path.join(ROOT, "profiles", name)) as fh:
    return json.loads(fh.read().strip().splitlines()[-1])


def test_committed_bench_line_follows_the_contract():
  d = _load("h100_bench_n1.json")
  for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline", "outputs_match_oracle"):
    assert key in d, key
  assert d["n_gpus"] == 1 and d["higher_is_better"] is True and d["vs_baseline"] is None and d["data"] == "synthetic"
  assert "workload" in d["config"] and "model" not in d["config"]
  assert d["outputs_match_oracle"] is True and d["gpu_launches"] > 0 and d["warmup"] >= 3
  # value = Q * steps / time
  assert abs(d["value"] - 4096 / (d["ms_per_step"] * 1e-3)) <= 1e-6 * d["value"]
  r = d["roofline"]
  assert r["bound"] == "tensor" and r["unit"] == "TFLOP/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
  assert abs(r["achieved"] - 2.0 * 4096 * 1e6 * 64 / (r["stage_ms_per_call"]["filter_pass"] * 1e-3) / 1e12) <= 1e-6 * r["achieved"]
  assert r["traffic"] and r["traffic"] >= 132e6          # never below the algorithmic bytes (the fp16 image + queries + results)
  e = d["e2e"]
  assert e["h2d_bytes_per_step"] == 4096 * 64 * 4 and e["d2h_bytes_per_step"] == 4096 * 100 * 8 and e["value"] < d["value"] * 1.02
  c = d["cpu_baseline"]
  assert c["kind"] in ("port", "reference") and c["cores"] >= 1 and c["value"] > 0 and "sample" in c
  clk = d["clocks"]
  assert clk["samples"] > 0 and not set(clk["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
  assert d["gather"]["cfg5_uniform"]["frac_of_hbm_peak"] >= 0.70      # the north-star target for the gather


def test_committed_reference_arm_line():
  r = _load("h100_bench_reference_arm.json")
  assert r["impl"] == "reference" and r["gpu_launches"] == 0
  assert r["e2e"]["h2d_bytes_per_step"] == 0 and r["e2e"]["d2h_bytes_per_step"] == 0 and r["e2e"]["value"] == r["value"]
  assert r["cpu_baseline"]["value"] == r["value"] and r["cpu_baseline"]["cores"] >= 1
  ours = _load("h100_bench_n1.json")
  assert r["metric"] == ours["metric"] and r["unit"] == ours["unit"] and r["config"]["workload"] == ours["config"]["workload"]
