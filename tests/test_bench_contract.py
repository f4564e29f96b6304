"""bench.py's reference arm runs on the host cores only, so its JSON contract can be checked without a GPU; --dump-outputs is
checked on the host (sampling, format) and on the GPU (the timed path's results)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_json_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1]
    d = json.loads(line)
    assert d["impl"] == "reference" and d["unit"] == "windows/s" and d["higher_is_better"] is True
    assert d["metric"].startswith("BA windows/s") and d["dtype"] == "f64" and d["scaling"] == "weak"
    assert d["value"] > 0 and d["steps"] == 1 and d["warmup"] == 1
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "windows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "config 2" in d["config"]["workload"]


def test_b200_arm_refuses_to_run_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        return
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "0"], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and "no CPU fallback" in (r.stderr + r.stdout)


def test_dump_outputs_sample_is_fixed_and_bounded(tmp_path, monkeypatch):
    """--dump-outputs keeps every window while the batch fits the size limit, else the same seeded sample of windows on every
    run; arrays are float32 / float64 and concatenated in batch order"""
    import types
    import numpy as np
    import bench
    wins = [types.SimpleNamespace(n_kf=3, n_lm=5 + i % 3) for i in range(40)]
    res = []
    for i, w in enumerate(wins):
        c = types.SimpleNamespace(initial_cost=2.0 * i, final_cost=float(i), status=0)
        res.append(types.SimpleNamespace(kf_pose=np.full((w.n_kf, 7), float(i)), kf_plane=np.zeros((w.n_kf, 4)),
                                         lm_pos=np.full((w.n_lm + 1, 3), float(i)), lm_rejected=np.ones(w.n_lm + 1, np.uint8),
                                         c=c, solves=[types.SimpleNamespace(num_iterations=i)]))
    bench.dump_outputs(str(tmp_path / "all"), wins, res)
    idx = np.load(tmp_path / "all" / "window_index.npy")
    assert np.array_equal(idx, np.arange(40))
    assert np.load(tmp_path / "all" / "lm_pos.npy").shape == (sum(w.n_lm for w in wins), 3)
    monkeypatch.setattr(bench, "DUMP_LIMIT_BYTES", 4000)
    for run in ("a", "b"):
        bench.dump_outputs(str(tmp_path / run), wins, res)
    total = 0
    for f in sorted(os.listdir(tmp_path / "a")):
        a, b = np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)
        assert a.dtype in (np.float32, np.float64) and np.array_equal(a, b), f
        total += a.nbytes
    assert total <= 4000
    idx = np.load(tmp_path / "a" / "window_index.npy").astype(int)
    assert 0 < len(idx) < 40 and np.all(np.diff(idx) > 0)
    assert np.array_equal(np.load(tmp_path / "a" / "final_cost.npy"), idx.astype(float))
    assert np.array_equal(np.load(tmp_path / "a" / "kf_pose.npy")[::3, 0], idx.astype(float))


@pytest.mark.gpu
def test_dump_outputs_of_the_timed_path(tmp_path):
    """bench.py --dump-outputs on the GPU: --steps is the number of timed steps, and two runs with the same arguments write
    identical arrays (seeded inputs, deterministic solver)"""
    import numpy as np
    args = ["--steps", "2", "--warmup", "1", "--batch", "6", "--distinct", "3", "--no-sub", "--cpu-sample", "0", "--in-flight", "1"]
    for run in ("a", "b"):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args + ["--dump-outputs", str(tmp_path / run)],
                           cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        d = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
        assert d["steps"] == 2 and d["config"]["batch_windows_per_gpu"] == 6
    names = sorted(os.listdir(tmp_path / "a"))
    assert {"kf_pose.npy", "lm_pos.npy", "final_cost.npy", "window_index.npy"} <= set(names)
    for f in names:
        a, b = np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)
        assert a.dtype in (np.float32, np.float64) and np.array_equal(a, b), f
    assert np.array_equal(np.load(tmp_path / "a" / "window_index.npy"), np.arange(6))
    assert np.all(np.load(tmp_path / "a" / "status.npy") == 0)
    assert np.load(tmp_path / "a" / "kf_pose.npy").shape == (6 * 30, 7)
