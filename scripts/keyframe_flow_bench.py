"""The flow scheme of keyframe selection on the store: kba_track_frame_flow, its group form and the facade's host
KeyframeSelector::select().

Drives from tests/keyframe_drive.py at limo's sizes (one camera, 2500 features per frame) with windows of 12 and 20 keyframes.
Every track of a group holds the same drive; the timed request is the last frame's (its measurements that have slots, against the
newest keyframe).  Wall time per call ending in a synchronisation (median and p90) of the single call and of the group calls at
G = 1, 32 and 132, and the facade's select() and its flow walk alone on the same drive, every frame (tests/cpp/test_facade_keyframe,
bench mode).  With --profile it measures instead, under torch.profiler, the summed device time of the k_kf_* kernels per call.
One JSON line per measurement, with the GPU name, its power limit and its max SM clock.
Usage: python scripts/keyframe_flow_bench.py [--repeats 30] [--groups 1,32,132] [--profile]"""
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
    """summed CUDA time of the k_kf_* kernels per call, from torch.profiler (None if it recorded none)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(calls):
            fn()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_kf_" in e.key)
    return round(us / 1e3 / calls, 4) if us > 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--groups", default="1,32,132")
    ap.add_argument("--profile", action="store_true", help="k_kf_* device time under torch.profiler instead of wall time")
    args = ap.parse_args()
    import torch
    from limo_b200 import capi
    from tests.keyframe_drive import KeyframeDrive
    from tests.test_track_keyframe import _push, _request, _track, replay
    info = card()
    h = capi.Handle(0)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]):  # CUPTI's set-up, outside every measured session
            torch.cuda.synchronize()
    groups = [int(g) for g in args.groups.split(",")]
    exe = os.path.join(ROOT, "tests", "cpp", "test_facade_keyframe")
    for window in (12, 20):
        dr = KeyframeDrive(7, n_frames=40, window=window, rig=False, n_feat=2500)
        steps = list(replay(dr))
        st = steps[-1]
        req = _request(dr, st)
        req = dict(req, lm_slot=np.asarray(req["lm_slot"], np.int32), cam=np.asarray(req["cam"], np.int32))
        tracks = []
        for _ in range(max(groups)):
            t, n_kf = _track(h, dr), 0
            for s in steps[:-1]:
                if s["sel"]:
                    _push(t, dr, s["k"], n_kf)
                    n_kf += 1
            tracks.append(t)
        base = dict(window=window, frame_features=len(st["lm"]), matched=st["flow"][0], **info)
        fn = lambda: tracks[0].frame_flow(**req)  # noqa: E731
        r0 = fn()
        assert r0["n_matched"] == st["flow"][0] and np.float64(r0["flow_sum"]).view(np.int64) == np.float64(st["flow"][1]).view(np.int64)
        if args.profile:
            print(json.dumps(dict(what="frame_flow_single", tracks=1, k_kf_device_ms=kernel_ms(fn, 10), **base)), flush=True)
        else:
            med, p90 = timed(fn, args.repeats)
            print(json.dumps(dict(what="frame_flow_single", tracks=1, median_ms=round(med, 4), p90_ms=round(p90, 4), **base)), flush=True)
        for G in groups:
            grp = capi.TrackGroup(h, tracks[:G])
            gfn = lambda: grp.frame_flow([req] * G)  # noqa: E731, B023
            for r in gfn():  # every track gives the single call's outputs
                assert r["n_matched"] == r0["n_matched"] and np.array_equal(r["match"], r0["match"])
            if args.profile:
                print(json.dumps(dict(what="frame_flow_group", tracks=G, k_kf_device_ms=kernel_ms(gfn, 10), **base)), flush=True)
            else:
                med, p90 = timed(gfn, args.repeats)
                print(json.dumps(dict(what="frame_flow_group", tracks=G, median_ms=round(med, 4), p90_ms=round(p90, 4), **base)), flush=True)
            grp.close()
        for t in tracks:
            t.close()
        if not args.profile:
            with tempfile.TemporaryDirectory() as tmp:  # the facade's host selector on the same drive, every frame
                path = os.path.join(tmp, "drive.txt")
                dr.write(path)
                r = subprocess.run([exe, "bench", path], capture_output=True, text=True, check=True)
                line = json.loads(r.stdout.strip().splitlines()[-1])
                for what in ("facade_select_ms", "facade_flow_ms"):
                    print(json.dumps(dict(what=what[:-3], median_ms=line[what][0], p90_ms=line[what][1], frames=line["frames"], **base)), flush=True)
    h.close()


if __name__ == "__main__":
    main()
