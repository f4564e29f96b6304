"""Landmark selection per solve(): the host select() against the store computing the chain's quantities.

Device: kba_track_select_landmarks on synthetic stores (every landmark measured by 6 consecutive keyframes, one camera, limo's
mono-lidar voxel parameters), wall time of the call as solve() pays it (upload, kernels, download, synchronisation).
Host and end to end: tests/cpp/test_facade_select in its timing mode -- a drive through the facade with limo's chain, the host
select() of a standalone selector on the same state, and solve() with device and with host selection.
Prints one JSON line per measurement: median and p90 in ms.  Usage: python scripts/select_bench.py [--repeats 50]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def device_store(h, n_kf, n_lm, seed=0):
    from limo_b200 import capi
    rng = np.random.default_rng(seed)
    per_kf = 6 * n_lm // n_kf + 1
    t = capi.Track(h, [[700.0, 600.0, 190.0]], [[0.5, 0.5, -0.5, 0.5, 0.0, 0.0, 0.0]], max_keyframes=n_kf, max_landmarks=n_lm,
                   max_measurements=n_kf * per_kf, win_keyframes=8, win_landmarks=64, win_observations=64)
    pos = np.column_stack([rng.uniform(-5, 80, n_lm), rng.uniform(-30, 30, n_lm), rng.uniform(-2, 6, n_lm)])
    t.set_landmarks(np.arange(n_lm, dtype=np.int32), pos=pos)
    first = rng.integers(0, n_kf - 5, n_lm)               # seen by keyframes first .. first + 5
    for k in range(n_kf):
        lm = np.nonzero((first <= k) & (k < first + 6))[0].astype(np.int32)
        pose = [1.0, 0.0, 0.0, 0.0, -1.5 * k, 0.0, 0.0]
        t.push_keyframe(k, pose, lm, rng.uniform(0, 1200, len(lm)), rng.uniform(0, 380, len(lm)), np.full(len(lm), -1.0))
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=50)
    args = ap.parse_args()
    import torch
    from limo_b200 import capi
    h = capi.Handle(0)
    for n_kf, n_lm in ((12, 1100), (20, 8000), (20, 20000)):
        t = device_store(h, n_kf, n_lm)
        kf, lm = np.arange(n_kf, dtype=np.int32), np.arange(n_lm, dtype=np.int32)
        prm = dict(voxel_size=(0.5, 0.5, 0.3), roi_far=40.0, roi_middle=15.0)
        for _ in range(5):
            out = t.select_landmarks(kf, lm, **prm)
        ts = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            t.select_landmarks(kf, lm, **prm)
            ts.append(1e3 * (time.perf_counter() - t0))
        print(json.dumps(dict(what="device_select", keyframes=n_kf, landmarks=n_lm, near=len(out["near_order"]),
                              median_ms=round(float(np.median(ts)), 3), p90_ms=round(float(np.percentile(ts, 90)), 3),
                              gpu=torch.cuda.get_device_name(0))), flush=True)
        t.close()
    h.close()
    exe = os.path.join(ROOT, "tests", "cpp", "test_facade_select")
    for window, n_scene in ((12, 900), (20, 6400), (20, 16000)):
        r = subprocess.run([exe, str(window), str(n_scene), "33"], capture_output=True, text=True, check=True)
        line = json.loads(r.stdout.strip().splitlines()[-1])
        line["what"] = "facade_drive"
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
