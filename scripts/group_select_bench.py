"""Landmark selection for a group of tracks: one kba_track_select_landmarks per track against one
kba_track_group_select_landmarks.

Stores from scripts/select_bench.py's device_store (12 keyframes / 1.1k landmarks and 20 / 8k, one camera, limo's mono-lidar
voxel parameters), G = 1, 32 and 132 tracks.  Wall time per call of the whole group, ending in a synchronisation (median and
p90), and in a run of its own under torch.profiler the summed device time of the k_sel_* kernels per call.  Prints one JSON
line per measurement with the GPU name, its power limit and its max SM clock.
Usage: python scripts/group_select_bench.py [--repeats 30] [--groups 1,32,132]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def card():
    """name, power limit (W) and max SM clock (MHz) of GPU 0 as nvidia-smi reports them"""
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        return dict(gpu="unknown", power_limit_w=None, max_sm_clock_mhz=None)
    name, pl, clk = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit_w=float(pl), max_sm_clock_mhz=int(float(clk)))


def timed(fn, repeats, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), float(np.percentile(ts, 90))


def kernel_ms(fn, calls):
    """summed CUDA time of the k_sel_* kernels per call, from torch.profiler (None if it recorded none)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(calls):
            fn()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_sel_" in e.key)
    return round(us / 1e3 / calls, 3) if us > 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--groups", default="1,32,132")
    args = ap.parse_args()
    import torch
    from limo_b200 import capi
    from select_bench import device_store
    info = card()
    h = capi.Handle(0)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]):  # CUPTI's set-up, outside every measured session
        torch.cuda.synchronize()
    prm = dict(voxel_size=(0.5, 0.5, 0.3), roi_far=40.0, roi_middle=15.0)
    for n_kf, n_lm in ((12, 1100), (20, 8000)):
        G_max = max(int(g) for g in args.groups.split(","))
        tracks = [device_store(h, n_kf, n_lm, seed=s) for s in range(G_max)]
        req = dict(kf_slots=np.arange(n_kf, dtype=np.int32), lm_slots=np.arange(n_lm, dtype=np.int32), **prm)
        for G in (int(g) for g in args.groups.split(",")):
            ts = tracks[:G]
            grp = capi.TrackGroup(h, ts)
            reqs = [req] * G
            singles = lambda: [t.select_landmarks(**req) for t in ts]  # noqa: E731
            group = lambda: grp.select_landmarks(reqs)  # noqa: E731
            a, b = singles(), group()
            for x, y in zip(a, b):  # the same quantities either way
                assert all(np.array_equal(x[k], y[k], equal_nan=k == "flow") for k in x)
            for what, fn in (("per_track_calls", singles), ("group_call", group)):
                med, p90 = timed(fn, args.repeats)
                line = dict(what=what, tracks=G, keyframes=n_kf, landmarks=n_lm, median_ms=round(med, 3), p90_ms=round(p90, 3),
                            k_sel_device_ms=kernel_ms(fn, 10), **info)
                print(json.dumps(line), flush=True)
            grp.close()
        for t in tracks:
            t.close()
    h.close()


if __name__ == "__main__":
    main()
