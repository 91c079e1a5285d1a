"""CPU-only: the JSON lines bench.py printed on an H100 (committed under profiles/) carry every key of the benchmark's result format, and
the derived fields are consistent with each other (value <-> ms_per_step, roofline.frac = achieved / peak, e2e bytes declared)."""
import glob
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LINES = sorted(glob.glob(os.path.join(ROOT, "profiles", "r02_bench_*.json")))

BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline", "dtype", "data", "config", "e2e",
             "gpu_launches", "roofline", "cpu_baseline", "clocks"}


@pytest.mark.parametrize("path", LINES, ids=[os.path.basename(p) for p in LINES])
def test_committed_bench_lines_follow_the_contract(path):
    with open(path) as fh:
        d = json.loads(fh.read().strip().splitlines()[-1])
    assert BASE_KEYS <= set(d), BASE_KEYS - set(d)
    assert d["unit"] == "rays/s" and d["higher_is_better"] is True and d["scaling"] == "weak" and d["data"] == "synthetic" and d["vs_baseline"] is None
    assert d["warmup"] >= 3 and d["steps"] >= 1 and d["gpu_launches"] > 0
    assert "workload" in d["config"] and "l2" in d["config"] and "model" not in d["config"]
    e = d["e2e"]
    assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(e) and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0
    assert e["value"] != d["value"]                                   # measured separately, not a copy of the device-timed value
    r = d["roofline"]
    assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(r) and r["bound"] in ("hbm", "tensor")
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    rays = d["config"]["rays_per_gpu"] * d["n_gpus"]
    assert abs(d["value"] - rays / (d["ms_per_step"] * 1e-3)) <= 1e-6 * d["value"]
    c = d["clocks"]
    assert c["sm_mhz"] >= 0.9 * c["sm_max_mhz"] and not [x for x in c["reasons"] if "slowdown" in x]
    if d["cpu_baseline"] is not None:
        assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"]) and d["cpu_baseline"]["kind"] in ("port", "reference")
    if "training_step" in d:
        t = d["training_step"]
        assert t["workload"] == "angelo-train-8192" and ("error" in t or (t["value"] > 0 and t["n_gpus"] == d["n_gpus"]))


def test_there_are_lines_for_every_baseline_config():
    names = " ".join(os.path.basename(p) for p in LINES)
    for wl in ("neus-facto-dtu65-4096x128", "volsdf-errorbounded-4096", "angelo-train-8192", "bakedsdf-render-65536"):
        assert wl in names, wl
