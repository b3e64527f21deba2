"""The driver's contract for bench.py that can be checked without a GPU: the reference arm prints exactly one JSON line on
stdout with the agreed keys, whatever libraries print elsewhere."""
import json
import os
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def test_reference_arm_prints_one_json_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", "--rows", "300"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, r.stdout
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "windows/s" and d["higher_is_better"] is True and d["value"] > 0
    assert d["steps"] == 1 and d["n_gpus"] == 1 and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "windows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and "model" not in d["config"]


def test_gpu_arm_fails_loudly_without_a_gpu():
    import torch

    if torch.cuda.is_available():
        return  # with a GPU the arm runs for real
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode != 0 and r.stdout.strip() == ""  # no CPU fallback, no fake number


def test_dump_outputs_writes_a_fixed_float32_row_sample(tmp_path):
    """--dump-outputs: one float32 .npy per output array, the same seeded rows in every file and in every run."""
    import numpy as np
    import torch

    import bench

    n = bench.DUMP_ROWS + 3000
    rows = torch.arange(n, dtype=torch.float64)
    out = {"model-output": rows[:, None].repeat(1, 4).float(), "total-anomaly-scaled": rows * 0.5}
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), out, n)
    assert sorted(p.name for p in (tmp_path / "a").iterdir()) == ["model-output.npy", "total-anomaly-scaled.npy"]
    model, total = np.load(tmp_path / "a" / "model-output.npy"), np.load(tmp_path / "a" / "total-anomaly-scaled.npy")
    assert model.dtype == np.float32 and total.dtype == np.float32
    assert model.shape == (bench.DUMP_ROWS, 4) and total.shape == (bench.DUMP_ROWS,)
    picked = model[:, 0]
    assert np.all(np.diff(picked) > 0) and picked[-1] < n  # distinct rows of the output, in row order
    np.testing.assert_array_equal(total, picked * 0.5)  # the same rows in every array
    for name in ("model-output.npy", "total-anomaly-scaled.npy"):
        np.testing.assert_array_equal(np.load(tmp_path / "a" / name), np.load(tmp_path / "b" / name))
    small = {"model-output": torch.ones((10, 4))}
    bench.dump_outputs(str(tmp_path / "c"), small, 10)
    assert np.load(tmp_path / "c" / "model-output.npy").shape == (10, 4)  # fewer rows than the sample: all of them
