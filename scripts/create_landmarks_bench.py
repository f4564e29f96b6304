"""push()'s landmark creation on the store: kba_track_create_landmarks, kba_track_group_create_landmarks and the facade's host push().

Drives from tests/create_drive.py (one camera, 300 new landmarks per push, with and without lidar depths) in windows of 12 and 20
keyframes.  Every track of a group holds the same drive; the timed request is the last push's: its active keyframes and the
landmarks it has to create.  Wall time per call ending in a synchronisation (median and p90) of the single call and of the group
call at G = 1, 32 and 132, in a run of its own under torch.profiler the summed device time of the k_cr_* kernels per call, and the
facade's push() on the host for the same drive (tests/cpp/test_facade_create, bench mode).  One JSON line per measurement, with
the GPU name, its power limit and its max SM clock.
Usage: python scripts/create_landmarks_bench.py [--repeats 30] [--groups 1,32,132]"""
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
    """summed CUDA time of the k_cr_* kernels per call, from torch.profiler (None if it recorded none)"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(calls):
            fn()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_cr_" in e.key)
    return round(us / 1e3 / calls, 4) if us > 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--groups", default="1,32,132")
    args = ap.parse_args()
    import torch
    from limo_b200 import capi
    from tests.create_drive import Drive
    from tests.test_track_create import _push, _track, drive_requests
    info = card()
    h = capi.Handle(0)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]):  # CUPTI's set-up, outside every measured session
        torch.cuda.synchronize()
    groups = [int(g) for g in args.groups.split(",")]
    exe = os.path.join(ROOT, "tests", "cpp", "test_facade_create")
    for window in (12, 20):
        for depth in (True, False):
            dr = Drive(7, n_push=window + 6, window=window, rig=False, new_per_push=300, depth=depth)
            last = dr.n_push - 1
            created = set()  # the landmarks created before the last push (the facade's rule: at least two rays, or a depth)
            for k, active, ids, res in drive_requests(dr):
                if k == last:
                    break
                created |= {lid for lid, (fl, _) in zip(ids, res) if fl & 1}
            active = list(range(last - window, last + 1))
            lm_new = sorted(lid for lid in dr.meas[last] if lid not in created)
            store_lm = len({lid for k in active for lid in dr.meas[k]})
            S = window + 2
            req = dict(kf_slots=[a % S for a in active], kf_new=len(active) - 1, lm_slots=lm_new)
            tracks = []
            for _ in range(max(groups)):
                t = _track(h, dr, solves=False)
                for k in range(dr.n_push):
                    _push(t, dr, k)
                tracks.append(t)
            base = dict(keyframes=window + 1, store_landmarks=store_lm, new_landmarks=len(lm_new), depth=depth, **info)
            single = lambda: tracks[0].create_landmarks(**req)  # noqa: E731
            med, p90 = timed(single, args.repeats)
            print(json.dumps(dict(what="single_call", tracks=1, median_ms=round(med, 4), p90_ms=round(p90, 4),
                                  k_cr_device_ms=kernel_ms(single, 10), **base)), flush=True)
            ref = single()
            for G in groups:
                grp = capi.TrackGroup(h, tracks[:G])
                reqs = [req] * G
                group = lambda: grp.create_landmarks(reqs)  # noqa: E731
                for pos, flags in group():  # the same positions as the single call, in every track
                    assert np.array_equal(flags, ref[1]) and np.array_equal(pos, ref[0], equal_nan=True)
                med, p90 = timed(group, args.repeats)
                print(json.dumps(dict(what="group_call", tracks=G, median_ms=round(med, 4), p90_ms=round(p90, 4),
                                      k_cr_device_ms=kernel_ms(group, 10), **base)), flush=True)
                grp.close()
            for t in tracks:
                t.close()
            with tempfile.TemporaryDirectory() as tmp:  # the facade's host push() of the same drive, all pushes
                path = os.path.join(tmp, "drive.txt")
                dr.write(path)
                r = subprocess.run([exe, "bench", path], capture_output=True, text=True, check=True)
                line = json.loads(r.stdout.strip().splitlines()[-1])
                print(json.dumps(dict(what="facade_host_push", median_ms=line["facade_push_ms"][0], p90_ms=line["facade_push_ms"][1],
                                      **base)), flush=True)
    h.close()


if __name__ == "__main__":
    main()
