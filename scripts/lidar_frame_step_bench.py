"""limo's mono-lidar frame step with the frame's depths from its lidar cloud as one store call (kba_track_frame_step_lidar and
its group form) against the chain it replaces, for one track and for groups of tracks.

Stores, frames and the per-step undo are those of scripts/frame_step_bench.py (one camera; every frame selected by the time
scheme, its keyframe dropped again outside the timing).  Every track's frame comes with its own KITTI-sized cloud (64 rings x
1875 azimuths, 4 floats per point, synth.make_lidar_scene; 8 scenes used in turn) seen through the KITTI camera <- velodyne pose.
  chain:      Handle.lidar_depth_batch with one view per track (the depths come back to the host), then frame_step /
              TrackGroup.frame_step with those depths;
  one:        frame_step / TrackGroup.frame_step with the cloud (depths not downloaded);
  one_c_call: the C call of `one` alone, on request records built once before the timing.
Per path: wall time per step (median and p90 of --repeats after warm-up, the paths alternating, each step ending in its calls'
synchronisation) and bytes up and down per step: transfer_bytes of the frame step, plus for the chain the clouds, 8 bytes of
(u, v) up and 4 bytes of depth down per feature of the batch call (its 152-byte view records not counted).  Before the timing,
the one call's depths are checked against the batch's, bit for bit.  Then, in a separate run under torch.profiler, the kernels'
device time per step of each path.  One JSON line per measurement, with the GPU name, its power limit and its max SM clock.
Usage: python scripts/lidar_frame_step_bench.py [--repeats 30] [--groups 1,32,132] [--stores 12:4000,20:8000] [--profile-steps 5]"""
import argparse
import ctypes as C
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

N_SCENES = 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--groups", default="1,32,132")
    ap.add_argument("--stores", default="12:4000,20:8000")
    ap.add_argument("--profile-steps", type=int, default=5)
    args = ap.parse_args()
    from frame_step_bench import INTR, store
    from group_select_bench import card
    from limo_b200 import capi, synth
    info = card()
    h = capi.Handle(0)
    opt = capi.default_options()
    scenes = [synth.make_lidar_scene(seed=0xBA5E0004 + s) for s in range(N_SCENES)]
    T = scenes[0][1]
    groups = [int(g) for g in args.groups.split(",")]
    for spec in args.stores.split(","):
        n_kf, n_lm = (int(x) for x in spec.split(":"))
        made = [store(h, n_kf, n_lm, seed=s) for s in range(max(groups))]
        for G in groups:
            tracks = [m[0] for m in made[:G]]
            clouds = [scenes[i % N_SCENES][0] for i in range(G)]
            base = [{k: x for k, x in m[1].items() if k != "d"} for m in made[:G]]
            lid = [dict(r, cloud=c, T_cam_lidar=T) for r, c in zip(base, clouds)]
            grp = capi.TrackGroup(h, tracks) if G > 1 else None

            def undo():  # the pushed keyframe out again, outside the timing
                if grp is None:
                    tracks[0].drop_keyframe(n_kf)
                else:
                    grp.drop_keyframes([n_kf] * G)

            def step(reqs):
                if grp is None:
                    out = [tracks[0].frame_step(opt=opt, **reqs[0])]
                    return out, tracks[0].transfer_bytes()[:2]
                return grp.frame_step(reqs, opt=opt), grp.transfer_bytes()

            def chain():
                views = [(i, T, INTR[0], np.stack([r["u"], r["v"]], axis=1)) for i, r in enumerate(base)]
                depths, _ = h.lidar_depth_batch(clouds, views)
                _, (up, down) = step([dict(r, d=d) for r, d in zip(base, depths)])
                n = sum(len(r["u"]) for r in base)
                return up + sum(c.nbytes for c in clouds) + 8 * n, down + 4 * n

            def one():
                return step(lid)[1]

            fn = capi.lib().kba_track_frame_step_lidar if grp is None else capi.lib().kba_track_group_frame_step_lidar
            req, out, ress, _keep, _result, recs = capi._frame_step_records(fn, lid, 256, True)
            c_args = (tracks[0]._p if grp is None else grp._p, req.ctypes.data_as(C.POINTER(capi.KbaFrameStepRequest)),
                      recs.ctypes.data_as(C.POINTER(capi.KbaFrameLidar)), C.byref(opt), out.ctypes.data_as(C.POINTER(capi.KbaFrameStepOut)),
                      ress)

            def one_c():
                capi._check(fn(*c_args))
                return tracks[0].transfer_bytes()[:2] if grp is None else grp.transfer_bytes()

            # the one call's depths against the batch's, bit for bit
            views = [(i, T, INTR[0], np.stack([r["u"], r["v"]], axis=1)) for i, r in enumerate(base)]
            ref, _ = h.lidar_depth_batch(clouds, views)
            got, _ = step([dict(r, depths=True) for r in lid])
            undo()
            assert all(np.array_equal(o["depth"].view(np.uint32), d.view(np.uint32)) for o, d in zip(got, ref))
            hits = sum(int((d > 0).sum()) for d in ref)
            paths = (("chain", chain), ("one", one), ("one_c_call", one_c))
            ts = {what: [] for what, _ in paths}
            moved = {}
            for what, f in paths:
                moved[what] = f()
                undo()
            for rep in range(3 + args.repeats):  # the paths alternate, so that all see the same host and GPU load
                for what, f in paths:
                    t0 = time.perf_counter()
                    f()
                    if rep >= 3:
                        ts[what].append(1e3 * (time.perf_counter() - t0))
                    undo()
            for what, _ in paths:
                up, down = moved[what]
                print(json.dumps(dict(what=what, tracks=G, keyframes=n_kf, landmarks=n_lm, features=sum(len(r["u"]) for r in base),
                                      depths_found=hits, median_ms=round(float(np.median(ts[what])), 3),
                                      p90_ms=round(float(np.percentile(ts[what], 90)), 3), h2d_bytes=int(up), d2h_bytes=int(down), **info)),
                      flush=True)
            if args.profile_steps > 0:
                profile(n_kf, G, paths, undo, args.profile_steps, info)
            if grp is not None:
                grp.close()
        for t, _ in made:
            t.close()
    h.close()


def profile(n_kf, G, paths, undo, steps, info):
    """the kernels' device time per step of each path, from torch.profiler in a run of its own"""
    import torch
    from torch.profiler import ProfilerActivity
    for what, f in paths:
        if what == "one_c_call":
            continue
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                f()
                torch.cuda.synchronize()
                undo()
        per = {}
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if us > 0 and not e.key.startswith("Memcpy") and not e.key.startswith("Memset"):
                m = re.search(r"\b(k_\w+)", e.key)
                name = m.group(1) if m else e.key[:60]
                per[name] = per.get(name, 0.0) + us / steps
        lidar = sum(v for k, v in per.items() if k.startswith("k_lidar"))
        print(json.dumps(dict(what=what + "_kernels", tracks=G, keyframes=n_kf, device_us_per_step=round(sum(per.values()), 1),
                              lidar_kernels_us=round(lidar, 1), kernels={k: round(v, 1) for k, v in sorted(per.items(), key=lambda x: -x[1])},
                              **info)), flush=True)


if __name__ == "__main__":
    main()
