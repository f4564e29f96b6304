"""Free landmark slots of the store: kba_track_reclaim_landmarks, its group form, and the facade past its landmark capacity.

Stores sized like the facade's (256 keyframe slots, 131072 landmark slots): 256 live keyframes of 500 measurements each on random
slots.  Wall time per call ending in a synchronisation (median and p90) of the single call over the range [0, 131072), without
and with the eviction outputs, and of the group call at G = 1, 32 and 132 (every track of a group holds the same store).  With
--profile it measures instead, under torch.profiler, the summed device time of the k_rc_* kernels per call.  Then the facade on
the drive of tests/cpp/test_facade_reclaim (bench mode): solve() and adjustPoseOnly() with a 4096-slot store that reclaims, and
on the rebuild path (set_persistent_window(false)) that the store fell back to once its slots ran out.  One JSON line per
measurement, with the GPU name, its power limit and its max SM clock.
Usage: python scripts/reclaim_bench.py [--repeats 30] [--groups 1,32,132] [--profile] [--frames 130]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from group_select_bench import card, timed  # noqa: E402

KF, LM, MEAS = 256, 1 << 17, 500


def kernel_ms(fn, calls):
    """summed CUDA time of the k_rc_* kernels per call, from torch.profiler (None if it recorded none)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(calls):
            fn()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_rc_" in e.key)
    return round(us / 1e3 / calls, 4) if us > 0 else None


def store(h, rng):
    from limo_b200 import capi
    t = capi.Track(h, [[700.0, 600.0, 190.0]], [[1.0, 0, 0, 0, 0, 0, 0]], max_keyframes=KF, max_landmarks=LM, max_measurements=1 << 21,
                   win_keyframes=30, win_landmarks=1024, win_observations=8192)
    f = np.zeros(MEAS, np.float32)
    for k in range(KF):
        t.push_keyframe(k, [1.0, 0, 0, 0, 0, 0, 0], np.sort(rng.choice(LM, MEAS, replace=False)), f, f, f)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--groups", default="1,32,132")
    ap.add_argument("--profile", action="store_true", help="k_rc_* device time under torch.profiler instead of wall time")
    ap.add_argument("--frames", type=int, default=130, help="frames of the facade drive (0: skip the facade)")
    args = ap.parse_args()
    import torch
    from limo_b200 import capi
    info = card()
    h = capi.Handle(0)
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]):  # CUPTI's set-up, outside every measured session
            torch.cuda.synchronize()
    rng = np.random.default_rng(0)
    t = store(h, rng)
    free = len(t.reclaim_landmarks(0, LM))
    for evict in (False, True):
        fn = lambda: t.reclaim_landmarks(0, LM, evict=evict)  # noqa: E731
        rec = dict(info, what="single", keyframes=KF, range=LM, free=free, evict=evict)
        if args.profile:
            rec["kernel_ms"] = kernel_ms(fn, args.repeats)
        else:
            rec["median_ms"], rec["p90_ms"] = timed(fn, args.repeats)
        print(json.dumps(rec), flush=True)
    tracks = [t]
    for G in [int(g) for g in args.groups.split(",")]:
        while len(tracks) < G:
            tracks.append(store(h, np.random.default_rng(0)))
        g = capi.TrackGroup(h, tracks[:G])
        reqs = [dict(lo=0, hi=LM)] * G
        fn = lambda: g.reclaim_landmarks(reqs)  # noqa: E731
        rec = dict(info, what="group", G=G, keyframes=KF, range=LM)
        if args.profile:
            rec["kernel_ms"] = kernel_ms(fn, args.repeats)
        else:
            rec["median_ms"], rec["p90_ms"] = timed(fn, args.repeats)
        print(json.dumps(rec), flush=True)
        g.close()
    for x in tracks:
        x.close()
    h.close()
    if args.frames and not args.profile:
        exe = os.path.join(ROOT, "tests", "cpp", "test_facade_reclaim")
        out = subprocess.run([exe, str(args.frames), "bench"], capture_output=True, text=True, check=True)
        print(json.dumps(dict(info, what="facade", **json.loads(out.stdout.strip().splitlines()[-1]))), flush=True)


if __name__ == "__main__":
    main()
