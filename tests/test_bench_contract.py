"""bench.py keeps the driver's contract: one JSON line with the agreed keys, for both arms."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "cpu_baseline"}


def _run(args, timeout):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True,
                         timeout=timeout, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, out.stdout
    return json.loads(lines[0])


def test_reference_arm_line():
    d = _run(["--impl", "reference", "--steps", "1", "--warmup", "0"], 300)
    assert d["impl"] == "reference" and BASE_KEYS <= set(d)
    assert d["steps"] == 1                                   # --steps sets the number of timed steps exactly
    assert d["metric"] == "candidate schedules/sec" and d["unit"] == "candidates/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["gpu_launches"] == 0
    assert "workload" in d["config"] and "model" not in d["config"]
    # both arms print the same `config` object for the headline run
    sys.path.insert(0, ROOT)
    import bench
    assert d["config"] == bench.static_config(True)
    assert d["cpu_baseline"]["cores"] <= (os.cpu_count() or 1) and "physical cores" in d["run"]["cores_how"]


def _load_dump(d):
    import numpy as np
    return {f[:-4]: np.load(os.path.join(d, f)) for f in sorted(os.listdir(d))}


def test_dump_outputs_layout_and_size_cap(tmp_path):
    """--dump-outputs writes float32 / float64 arrays only, stays under 64 MB for any batch (a seeded sample plus
    its indices above DUMP_LIMIT makespans), and writes the same files for the same outputs."""
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    import bench
    key = torch.tensor([(int(np.float32(3.5).view(np.uint32)) << 32) | 12345], dtype=torch.int64)
    for n in (1000, 9_000_000):
        out = torch.arange(n, dtype=torch.float32)
        runs = []
        for r in ("a", "b"):
            d = tmp_path / ("%d_%s" % (n, r))
            bench.dump_outputs(str(d), out, key)
            assert sum(f.stat().st_size for f in d.iterdir()) <= 64 * 10 ** 6
            runs.append(_load_dump(str(d)))
        a, b = runs
        assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)
        assert all(v.dtype in (np.float32, np.float64) for v in a.values())
        assert a["best_makespan"][0] == np.float32(3.5) and a["best_candidate"][0] == 12345
        if n <= bench.DUMP_LIMIT:
            assert set(a) == {"makespans", "best_makespan", "best_candidate"}
            assert np.array_equal(a["makespans"], out.numpy())
        else:
            idx = a["makespans_index"].astype(np.int64)
            assert len(idx) == bench.DUMP_LIMIT and np.all(np.diff(idx) > 0)
            assert np.array_equal(a["makespans"], out.numpy()[idx])


@pytest.mark.gpu
def test_dump_outputs_reproduce_the_timed_path(tmp_path):
    """Two runs with the same arguments dump identical outputs, and the dumped key is the arg-min of the dumped
    makespans (first index of the minimum)."""
    import numpy as np
    args = ["--steps", "2", "--warmup", "3", "--batch", str(132 * 16 * 32), "--no-cpu", "--no-e2e"]
    dumps = []
    for r in ("a", "b"):
        d = _run(args + ["--dump-outputs", str(tmp_path / r)], 600)
        assert d["steps"] == 2 and d["gpu_launches"] == 2
        dumps.append(_load_dump(str(tmp_path / r)))
    a, b = dumps
    assert set(a) == {"makespans", "best_makespan", "best_candidate"}
    assert all(np.array_equal(a[k], b[k]) for k in a)
    mk = a["makespans"]
    assert mk.dtype == np.float32 and mk.shape == (132 * 16 * 32,)
    assert a["best_makespan"][0] == mk.min() and int(a["best_candidate"][0]) == int(np.argmin(mk))


@pytest.mark.gpu
def test_our_arm_line():
    d = _run(["--steps", "4", "--warmup", "3", "--batch", str(132 * 16 * 32 * 2), "--no-cpu"], 600)
    assert BASE_KEYS <= set(d) and {"roofline", "clocks"} <= set(d)
    assert d["metric"] == "candidate schedules/sec" and d["n_gpus"] == 1 and d["steps"] == 4 and d["warmup"] >= 3
    assert d["scaling"] == "weak" and d["vs_baseline"] is None and d["dtype"] == "f32" and d["data"] == "synthetic"
    r = d["roofline"]
    assert r["bound"] == "hbm" and r["unit"] == "GB/s" and 0 < r["frac"] < 1.2 and r["peak"] > 1000
    assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["value"] > 0
    assert d["gpu_launches"] == 4 and d["value"] > 1e8
    assert set(d["clocks"]) >= {"sm_mhz", "sm_max_mhz", "reasons"}
    sys.path.insert(0, ROOT)
    import bench
    assert d["config"] == bench.static_config(True)
    assert d["e2e"]["candidates_per_gpu_per_step"] == d["run"]["candidates_per_gpu_per_step"]   # same batch as `value`
