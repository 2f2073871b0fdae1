"""CPU: the JSON line bench.py prints is a contract with whoever reads it.  The files kept under profiles/ hold real
outputs of bench.py on one H100 (N = 1 and the reference arm), the last line of each being bench.py's line and the
first the device it ran on; this checks that every key the contract names is there with the right type, that the
internal arithmetic is consistent (value = rows x N / time, roofline.frac = achieved / peak, achieved = algorithmic
bytes / kernel time) and that the two arms describe the same metric."""
import json
import os

import pytest

from conftest import ROOT

PROFILES = os.path.join(ROOT, "profiles")
REQUIRED = {"metric": str, "value": float, "unit": str, "n_gpus": int, "steps": int, "warmup": int,
            "ms_per_step": float, "higher_is_better": bool, "scaling": str, "dtype": str, "data": str,
            "config": dict, "e2e": dict, "gpu_launches": int}


def _line(name):
    path = os.path.join(PROFILES, name)
    if not os.path.exists(path):
        pytest.skip(name + " not kept")
    return json.loads(open(path).read().strip().splitlines()[-1])


@pytest.mark.parametrize("name", ["h100_bench_n1.jsonl"])
def test_gpu_arm_line_has_the_contract_keys_and_adds_up(name):
    d = _line(name)
    for key, typ in REQUIRED.items():
        assert key in d and isinstance(d[key], typ), key
    assert "vs_baseline" in d and d["vs_baseline"] is None  # BASELINE.md holds no published number
    assert d["higher_is_better"] is True and d["scaling"] == "weak" and d["data"] == "synthetic"
    assert "workload" in d["config"] and "model" not in d["config"]
    rows = d["config"]["rows_per_gpu"]
    assert d["value"] == pytest.approx(d["n_gpus"] * rows / (d["ms_per_step"] * 1e-3), rel=1e-9)
    for k in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert k in d["e2e"]
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
    assert d["e2e"]["value"] < d["value"]  # host buffers cross PCIe inside the timed region
    assert d["gpu_launches"] >= d["steps"]  # at least the epoch kernel per step
    rf = d["roofline"]
    assert rf["bound"] == "hbm" and rf["unit"] == "GB/s"
    assert rf["frac"] == pytest.approx(rf["achieved"] / rf["peak"], rel=1e-9)
    assert rf["achieved"] == pytest.approx(rows * rf["algorithmic_bytes_per_example"] / (d["ms_per_step"] * 1e-3) / 1e9,
                                           rel=1e-9)
    assert rf["algorithmic_bytes_per_example"] == 2 * 8 * 2 * 4  # 2 k nnz 4 (SURVEY.md section 8d)
    assert 0 < rf["frac"] < 1
    ck = d["clocks"]
    assert ck["sm_mhz"] and ck["sm_max_mhz"] and not ({"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"} &
                                                      set(ck["reasons"]))
    if d["n_gpus"] == 1:
        cpu = d["cpu_baseline"]
        assert cpu["kind"] in ("reference", "port") and cpu["cores"] == 1 and cpu["value"] > 0
        tol = d["tolerance_mode"]
        assert tol["parity"]["max_abs_gap"] <= tol["parity"]["tolerance_north_star"] == 1e-5
        assert tol["value"] > cpu["value"]  # the mode inside the gate beats the reference's own loop
        for key in ("c2_zipf", "c3", "c4"):
            assert key in d["extra"] and d["extra"][key]["roofline"]["frac"] > 0
    else:
        pm = d["parity_multi_gpu"]  # (None when the line was produced with --no-parity)
        if pm is not None:
            assert len(pm["heldout_rmse_gpu"]) == len(pm["heldout_rmse_one_sequential_stream"]) == pm["epochs"]
    if d["n_gpus"] == 8:
        c5 = d["extra"]["c5"]
        assert c5["rows_per_gpu"] * 8 == 100_000_000 and c5["k"] == 128 and "error" not in c5
        assert c5["roofline"]["frac"] > 0.5


def test_reference_arm_line():
    d = _line("h100_bench_ref.jsonl")
    ours = _line("h100_bench_n1.jsonl")
    assert d["impl"] == "reference" and d["metric"] == ours["metric"] and d["unit"] == ours["unit"]
    assert d["higher_is_better"] is True and d["gpu_launches"] == 0
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["value"] == d["value"]
    assert d["config"]["workload"] == ours["config"]["workload"]
