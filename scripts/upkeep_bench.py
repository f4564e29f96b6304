"""Window upkeep on the store: kba_track_deactivate_keyframes / kba_track_depth_costs, their group forms and the facade's host
deactivateKeyframes() and AddDepth getSelection().

Drives from tests/upkeep_drive.py (one camera, 300 new landmarks per push, ground labels) with windows of 12 and 20 keyframes.
Every track of a group holds the same drive; the timed requests are the last step's (tests/test_track_upkeep.drive_steps): the
deactivation of its active keyframes and landmarks, and the costs of its eligible landmarks over the keyframes that stay.  Wall
time per call ending in a synchronisation (median and p90) of the single calls and of the group calls at G = 1, 32 and 132, and
the facade's two host steps on the same drive (tests/cpp/test_facade_upkeep, bench mode).  With --profile it measures instead,
under torch.profiler, the summed device time of the k_up_* kernels per call.  One JSON line per measurement, with the GPU name,
its power limit and its max SM clock.
Usage: python scripts/upkeep_bench.py [--repeats 30] [--groups 1,32,132] [--profile]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from group_select_bench import card, timed  # noqa: E402


def kernel_ms(fn, calls):
    """summed CUDA time of the k_up_* kernels per call, from torch.profiler (None if it recorded none)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(calls):
            fn()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_up_" in e.key)
    return round(us / 1e3 / calls, 4) if us > 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--groups", default="1,32,132")
    ap.add_argument("--profile", action="store_true", help="k_up_* device time under torch.profiler instead of wall time")
    args = ap.parse_args()
    import torch
    from limo_b200 import capi
    from tests.test_track_upkeep import _push, _track, drive_steps
    from tests.upkeep_drive import UpkeepDrive
    info = card()
    h = capi.Handle(0)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]):  # CUPTI's set-up, outside every measured session
            torch.cuda.synchronize()
    groups = [int(g) for g in args.groups.split(",")]
    exe = os.path.join(ROOT, "tests", "cpp", "test_facade_upkeep")
    for window in (12, 20):
        dr = UpkeepDrive(7, n_push=window + 10, window=window, rig=False, new_per_push=300)
        st = list(drive_steps(dr))[-1]
        S = window + 2
        i32 = lambda x: np.asarray(x, np.int32)  # noqa: E731  (a caller keeps its lists as arrays: no conversion inside the timing)
        dreq = dict(kf_slots=i32([a % S for a in st["kf"]]), lm_slots=i32(st["lm"]), min_connecting=3, min_window=4, max_window=window)
        creq = dict(kf_slots=i32([a % S for a in st["active"]]), lm_slots=i32(st["elig"]))
        tracks = []
        for _ in range(max(groups)):
            t, done = _track(h, dr), set()
            for k in range(dr.n_push):
                _push(t, dr, k, st["pos"], done)
            tracks.append(t)
        base = dict(keyframes=len(st["kf"]), active_landmarks=len(st["lm"]), eligible=len(st["elig"]), pairs=int(st["off"][-1]), **info)
        calls = dict(deactivate=(lambda: tracks[0].deactivate_keyframes(**dreq)), depth_costs=(lambda: tracks[0].depth_costs(**creq)))
        d0, c0 = calls["deactivate"](), calls["depth_costs"]()
        assert np.array_equal(d0[1], st["common"]) and np.array_equal(c0[2].view(np.int64), st["cost"].view(np.int64))
        for what, fn in calls.items():
            if args.profile:
                print(json.dumps(dict(what=what + "_single", tracks=1, k_up_device_ms=kernel_ms(fn, 10), **base)), flush=True)
            else:
                med, p90 = timed(fn, args.repeats)
                print(json.dumps(dict(what=what + "_single", tracks=1, median_ms=round(med, 4), p90_ms=round(p90, 4), **base)), flush=True)
        for G in groups:
            grp = capi.TrackGroup(h, tracks[:G])
            gcalls = dict(deactivate=(lambda: grp.deactivate_keyframes([dreq] * G)), depth_costs=(lambda: grp.depth_costs([creq] * G)))
            for d, c in zip(gcalls["deactivate"](), gcalls["depth_costs"]()):  # every track gives the single call's outputs
                assert all(np.array_equal(a, b) for a, b in zip(d, d0)) and np.array_equal(c[2].view(np.int64), c0[2].view(np.int64))
            for what, fn in gcalls.items():
                if args.profile:
                    print(json.dumps(dict(what=what + "_group", tracks=G, k_up_device_ms=kernel_ms(fn, 10), **base)), flush=True)
                else:
                    med, p90 = timed(fn, args.repeats)
                    print(json.dumps(dict(what=what + "_group", tracks=G, median_ms=round(med, 4), p90_ms=round(p90, 4), **base)), flush=True)
            grp.close()
        for t in tracks:
            t.close()
        if not args.profile:
            with tempfile.TemporaryDirectory() as tmp:  # the facade's host steps on the same drive, every step
                path = os.path.join(tmp, "drive.txt")
                dr.write(path)
                r = subprocess.run([exe, "bench", path], capture_output=True, text=True, check=True)
                line = json.loads(r.stdout.strip().splitlines()[-1])
                for what in ("facade_deactivate_ms", "facade_add_depth_ms"):
                    print(json.dumps(dict(what=what[:-3], median_ms=line[what][0], p90_ms=line[what][1], steps=line["steps"], **base)), flush=True)
    h.close()


if __name__ == "__main__":
    main()
