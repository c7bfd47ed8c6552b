"""The bench.py output contract, checked on stored bench lines (tests/golden/bench/, each measured on one H100 SXM 80 GB:
the *_w3 / *_w5 lines at a 700 W power limit, the others at 400 W): every key a consumer of the line reads must be there
with the right type."""
import glob
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH = os.path.join(ROOT, "tests", "golden", "bench")
LINES = sorted(glob.glob(os.path.join(BENCH, "h100_bench_110m_*.json")) + glob.glob(os.path.join(BENCH, "h100_bench_600m_*.json")))


def _line(path):
    return json.loads(open(path).read().strip().splitlines()[-1])


@pytest.mark.parametrize("path", LINES, ids=[os.path.basename(p) for p in LINES])
def test_bench_line_has_the_contract_keys(path):
    d = _line(path)
    for k, t in (("metric", str), ("value", float), ("unit", str), ("n_gpus", int), ("steps", int), ("warmup", int),
                 ("ms_per_step", float), ("higher_is_better", bool), ("scaling", str), ("dtype", str), ("data", str),
                 ("config", dict), ("e2e", dict), ("gpu_launches", int), ("clocks", dict), ("roofline", dict)):
        assert isinstance(d[k], t), (k, type(d[k]))
    assert "vs_baseline" in d and d["vs_baseline"] is None          # BASELINE.md has no published number for H100
    assert d["warmup"] >= 3 and d["scaling"] == "weak" and d["higher_is_better"] is True
    assert "workload" in d["config"] and "l2" in d["config"]
    e = d["e2e"]
    assert e["value"] > 0 and e["h2d_bytes_per_step"] in (64 * 160000 * 4, 16 * 480000 * 4) and e["d2h_bytes_per_step"] > 0
    assert e["value"] <= d["value"] * 1.02                           # end to end cannot beat the device-resident number
    assert e["sync_call"]["value"] <= e["value"] * 1.02
    r = d["roofline"]
    assert r["bound"] in ("hbm", "tensor") and r["unit"] in ("GB/s", "TFLOP/s")
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and 0 < r["frac"] < 1
    assert r["traffic"] is None or r["traffic"] > 0
    c = d["clocks"]
    # a power-limited card (400 W here) runs below its maximum SM clock under sustained load: the line records it
    assert 0 < c["sm_mhz"] <= c["sm_max_mhz"] and c["samples"] > 0 and not any("slowdown" in x for x in c["reasons"])
    if "job_clips" in d["config"]:           # the timed region is a job of distinct clips with one all-gather
        assert d["config"]["job_clips"] == d["steps"] * d["config"]["clips_per_gpu_per_step"] * d["n_gpus"]
        assert d["config"]["distinct_hypotheses_in_job"] >= 0.9 * d["config"]["job_clips"]
    assert d["gpu_launches"] > 0
    if d["n_gpus"] == 1:
        b = d["cpu_baseline"]
        assert b["kind"] in ("reference", "port") and b["cores"] >= 1 and b["value"] > 0 and b["sample"]
        assert b.get("tokens_match_gpu", True) is True


def test_streaming_bench_lines():
    paths = glob.glob(os.path.join(BENCH, "h100_bench_eou_stream_*.json"))
    assert paths
    for p in paths:
        d = _line(p)
        assert d["metric"].startswith("audio-seconds/sec (RTFx) eou-120m streaming") and d["value"] > 0 and d["higher_is_better"] is True
        assert d["config"]["streams"] >= 1 and d["config"]["chunk_samples"] == 2560 and d["gpu_launches"] > 0
        assert d["latency"]["ms_per_chunk_single_stream"] < d["latency"]["real_time_budget_ms"]
        r = d["roofline"]
        assert r["bound"] == "hbm" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9


@pytest.mark.parametrize("config", ["110m", "600m"])
def test_reference_arm_line(config):
    d = _line(os.path.join(BENCH, f"h100_bench_reference_arm_{config}.json"))
    assert d["impl"] == "reference" and d["value"] > 0 and d["e2e"]["value"] == d["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["cpu_baseline"]["kind"] == "reference"
    ours = _line(sorted(glob.glob(os.path.join(BENCH, f"h100_bench_{config}_*.json")))[0])
    assert d["metric"] == ours["metric"] and d["unit"] == ours["unit"]
