"""The committed bench line (profiles/h100_bench_fp16.json, written by `python bench.py` on one H100 80GB HBM3) carries every
key of the measurement contract, and the CPU-runnable parts of bench.py (argument surface, algorithmic constants) agree
with SURVEY.md section 8d."""
import importlib.util
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench():
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


BENCH_LINE = os.path.join(ROOT, "profiles", "h100_bench_fp16.json")


def test_committed_bench_line_has_the_contract_keys():
    d = json.load(open(BENCH_LINE))
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"):
        assert k in d, k
    assert d["unit"] == "audio-s/s" and d["higher_is_better"] is True and d["scaling"] == "weak" and d["data"] == "synthetic"
    assert d["n_gpus"] == 1 and d["warmup"] >= 3 and d["value"] > 0 and d["gpu_launches"] > 0
    assert "workload" in d["config"] and "model" not in d["config"]
    e = d["e2e"]
    assert e["unit"] == d["unit"] and 0 < e["value"] <= d["value"] * 1.02 and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and "traffic" in r
    c = d["cpu_baseline"]
    assert c["kind"] in ("port", "reference") and c["cores"] >= 1 and c["value"] > 0 and c["sample"]
    k = d["clocks"]
    assert k["sm_mhz"] > 0.9 * k["sm_max_mhz"] and not set(k["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    # consistency: value = audio seconds per step / step time
    assert abs(d["value"] - d["config"]["audio_seconds_per_utterance"] * d["config"]["global_batch"] / (d["ms_per_step"] * 1e-3)) / d["value"] < 1e-6


def test_bench_line_has_the_named_workloads():
    """The default `python bench.py` line also carries the named extra workloads, each with a positive rate."""
    d = json.load(open(BENCH_LINE))
    for k in ("stage_ms", "config3_batched", "config5_generator", "flow_wn", "config2_length_scale_1"):
        assert k in d, k
    e = d["e2e"]
    assert e["workspace_regrowths_in_timed_loops"] == 0
    c = d["cpu_baseline"]
    assert "T=256" in c["sample"]  # same utterance as the GPU arm
    assert len(d["config5_generator"]["sweep"]) >= 6 and d["config3_batched"]["value"] > 0 and d["flow_wn"]["value"] > 0


def test_algorithmic_constants_match_the_survey():
    b = _bench()
    # SURVEY.md section 8d: Generator layer-boundary bytes and FLOPs per 512-sample frame
    assert b.GEN_BYTES_PER_FRAME == 6_830_852 and b.GEN_FLOP_PER_FRAME == 651_608_576
    assert b.HOP == 512 and b.SR == 44100
