"""The bench line contract (driver-facing): the committed record lines under profiles/ carry every key the
contract names, with consistent values; `bench.py` parses its flags without a GPU."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _line(name):
    with open(os.path.join(ROOT, "profiles", name)) as f:
        return json.loads(f.read().strip().splitlines()[-1])


@pytest.mark.parametrize("n", [1])
def test_record_line_has_the_contract_keys(n):
    d = _line(f"h100_bench_n{n}.json")
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                "dtype", "data", "config", "roofline", "e2e", "gpu_launches", "clocks", "parity"):
        assert key in d, key
    assert d["n_gpus"] == n and d["higher_is_better"] is True and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["metric"] == "mash.Sketch Gbases/s" and d["unit"] == "Gbases/s" and d["data"] == "synthetic" and d["dtype"] == "u32"
    assert "workload" in d["config"] and "model" not in d["config"]
    assert d["warmup"] >= 3 and d["gpu_launches"] >= d["steps"] > 0
    # value is the whole-job aggregate: units of all ranks / max-over-ranks time
    reads = d["config"]["reads_per_gpu"] * d["config"]["read_len"] * n
    assert abs(d["value"] - reads / d["ms_per_step"] / 1e6) / d["value"] < 1e-6
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert r["traffic"] is None or r["traffic"] > 0
    e = d["e2e"]
    assert e["unit"] == "Gbases/s" and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and 0 < e["value"] < d["value"]
    c = d["clocks"]
    assert not set(c["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert all(d["parity"].values())
    if n == 1:
        cb = d["cpu_baseline"]
        assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] > 0 and cb["sample"]
        assert all(s["parity_vs_oracle"] for s in d["secondary"])
    else:
        assert d["pipeline"]["parity_all_green"] is True


@pytest.mark.parametrize("n", [1, 2, 4, 8])
def test_reference_arm_line(n):
    d = _line(f"h100_bench_ref_n{n}.json")
    assert d["impl"] == "reference" and d["metric"] == "mash.Sketch Gbases/s" and d["unit"] == "Gbases/s"
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["value"] == d["value"]


def test_bench_cli_parses_without_a_gpu():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--help"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0
    for flag in ("--gpus", "--steps", "--warmup", "--impl", "--dump-outputs"):
        assert flag in out.stdout


def test_documented_numbers_trace_to_the_record_lines():
    """The H100 tables of README.md / DESIGN.md quote the committed bench line (within rounding)."""
    import re

    d1 = _line("h100_bench_n1.json")
    sec = {s["name"]: s for s in d1["secondary"]}
    readme = open(os.path.join(ROOT, "README.md")).read()
    design = open(os.path.join(ROOT, "DESIGN.md")).read()

    def quoted(text, pattern):
        m = re.search(pattern, text)
        assert m, pattern
        return float(m.group(1))

    ms, gb = quoted(readme, r"\*\*([\d.]+) ms / pass"), quoted(readme, r"ms / pass = (\d+) Gbases/s\*\*")
    assert abs(ms - d1["ms_per_step"]) < 0.01 and abs(gb - d1["value"]) / d1["value"] < 0.01
    assert abs(quoted(readme, r"cfg3 \(100 k × 10 kbp, k=31, s=2000\) \| \*\*([\d.]+) ms") - sec["cfg3 sketch (K2)"]["ms"]) < 0.03
    sw = sec["cfg5 Smith-Waterman score (K4)"]
    assert abs(quoted(readme, r"\*\*([\d.]+) ms = [\d.]+ TCUPS\*\*") - sw["ms"]) < 0.2
    assert abs(quoted(readme, r"\*\*[\d.]+ ms = ([\d.]+) TCUPS\*\*") - sw["value"]) < 0.01
    frac = quoted(design, r"([\d.]+) of the H100 data-sheet HBM bandwidth")
    assert abs(frac - d1["roofline"]["frac"]) < 0.01
    assert abs(quoted(design, r"of the H100 data-sheet HBM bandwidth; [\d.]+ ms, (\d+) Gbases/s") - d1["value"]) / d1["value"] < 0.01
