"""limo's frame step -- adjustPoseOnly, keyframe selection, push() with its new landmarks -- as one store call against the chain of
calls it replaces, for one track and for groups of tracks.

Stores of n_kf keyframes and n_lm landmarks, one camera, every landmark measured by 6 consecutive keyframes; one spare keyframe
slot.  Each step's frame measures the newest keyframe's landmarks (90% of its runs in the last selection) and 200 new ones, a
third of them with a depth, and is selected (the time scheme); the new keyframe is dropped again outside the timing, so that
every step is the same work and the arena compacts now and then, as it does on a drive.
  chain: adjust_pose, frame_flow, the selector's verdict on the host, push_keyframe, create_landmarks -- or their group forms;
  one:   frame_step (G = 1) or TrackGroup.frame_step;
  one_c_call: the C call of `one` alone, on request records built once before the timing;
  one_rejected: `one` on a frame the time and pose schemes turn down (the call ends after its first download).
Per path: wall time per step (median and p90 of --repeats after warm-up, the paths alternating, each step ending in its calls'
synchronisation) and bytes up and down per step (transfer_bytes summed over the calls).  One JSON line per measurement, with the
GPU name, its power limit and its max SM clock.
Usage: python scripts/frame_step_bench.py [--repeats 30] [--groups 1,32,132] [--stores 12:4000,20:8000]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

INTR, CAM = [[700.0, 600.0, 190.0]], [[0.5, 0.5, -0.5, 0.5, 0.0, 0.0, 0.0]]
N_NEW = 200


def store(h, n_kf, n_lm, seed):
    """a track of n_kf keyframes in slots 0 .. n_kf - 1, landmarks 0 .. n_lm - 1, room for one more keyframe and N_NEW landmarks"""
    from limo_b200 import capi
    rng = np.random.default_rng(seed)
    per_kf = 6 * n_lm // n_kf + 1
    first = rng.integers(0, n_kf - 5, n_lm)
    t = capi.Track(h, INTR, CAM, max_keyframes=n_kf + 1, max_landmarks=n_lm + N_NEW, max_measurements=(n_kf + 2) * (per_kf + N_NEW),
                   win_keyframes=n_kf + 1, win_landmarks=n_lm + N_NEW, win_observations=n_kf * per_kf + N_NEW)
    pos = np.column_stack([rng.uniform(5, 80, n_lm), rng.uniform(-30, 30, n_lm), rng.uniform(-2, 6, n_lm)])
    t.set_landmarks(np.arange(n_lm, dtype=np.int32), pos=pos, weight=np.ones(n_lm))
    last = None
    for k in range(n_kf):
        lm = np.nonzero((first <= k) & (k < first + 6))[0].astype(np.int32)
        pose = [1.0, 0.0, 0.0, 0.0, -1.5 * k, 0.0, 0.0]
        u, v = rng.uniform(0, 1200, len(lm)).astype(np.float32), rng.uniform(0, 380, len(lm)).astype(np.float32)
        t.push_keyframe(k, pose, lm, u, v, np.full(len(lm), -1.0))
        last = (lm, u, v, pose)
    lm, u, v, pose = last
    new = np.arange(n_lm, n_lm + N_NEW, dtype=np.int32)
    lm_f = np.r_[lm, new]
    uf = np.r_[u + rng.normal(0, 20, len(u)), rng.uniform(0, 1200, N_NEW)].astype(np.float32)
    vf = np.r_[v + rng.normal(0, 20, len(v)), rng.uniform(0, 380, N_NEW)].astype(np.float32)
    d = np.where(rng.random(len(lm_f)) < 1 / 3, rng.uniform(5, 40, len(lm_f)), -1.0).astype(np.float32)
    run_sel = np.r_[rng.random(len(lm)) < 0.9, np.zeros(N_NEW, bool)]
    req = dict(kf_slots=np.arange(n_kf, dtype=np.int32), lm_slot=lm_f, u=uf, v=vf, d=d, run_sel=run_sel, kf_new=n_kf, new_slots=new,
               pose7=[1.0, 0.0, 0.0, 0.0, -1.5 * n_kf, 0.0, 0.0], stamp=10**9, stamp_last=0, critical_quaternion_diff=0.03,
               time_difference_ns=4 * 10**8, min_median_flow=5.0)
    return t, req


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--groups", default="1,32,132")
    ap.add_argument("--stores", default="12:4000,20:8000")
    args = ap.parse_args()
    from group_select_bench import card
    from limo_b200 import capi
    from limo_b200.keyframe_selector import calcQuaternionDiff
    info = card()
    h = capi.Handle(0)
    opt = capi.default_options()
    groups = [int(g) for g in args.groups.split(",")]
    for spec in args.stores.split(","):
        n_kf, n_lm = (int(x) for x in spec.split(":"))
        made = [store(h, n_kf, n_lm, seed=s) for s in range(max(groups))]
        for G in groups:
            tracks, rs = [m[0] for m in made[:G]], [m[1] for m in made[:G]]
            rejected = [dict(r, stamp=r["stamp_last"], critical_quaternion_diff=10.0) for r in rs]
            grp = capi.TrackGroup(h, tracks) if G > 1 else None
            last_pose = [1.0, 0.0, 0.0, 0.0, -1.5 * (n_kf - 1), 0.0, 0.0]

            def undo():  # the pushed keyframe out again, outside the timing
                if grp is None:
                    tracks[0].drop_keyframe(n_kf)
                else:
                    grp.drop_keyframes([n_kf] * G)

            def chain():
                up = down = 0

                def add(tb):
                    nonlocal up, down
                    up, down = up + tb[0], down + tb[1]
                sel = [r["run_sel"][np.r_[0, np.cumsum(r["lm_slot"][1:] != r["lm_slot"][:-1])]] for r in rs]
                adj = [dict(pose7=r["pose7"], lm_slot=r["lm_slot"][m], u=r["u"][m], v=r["v"][m], d=r["d"][m]) for r, m in zip(rs, sel)]
                flow = [dict(kf_last=n_kf - 1, lm_slot=r["lm_slot"], u=r["u"], v=r["v"], min_median_flow=5.0) for r in rs]
                if grp is None:
                    t = tracks[0]
                    res = [t.adjust_pose(opt=opt, **adj[0])]
                    add(t.transfer_bytes())
                    fl = [t.frame_flow(**flow[0])]
                    add(t.transfer_bytes())
                else:
                    res = grp.adjust_pose(adj, opt=opt)
                    add(grp.transfer_bytes())
                    fl = grp.frame_flow(flow)
                    add(grp.transfer_bytes())
                pushes = []
                for r, x, f in zip(rs, res, fl):
                    pose = x.kf_pose[0]
                    picked = f["usable"] and (calcQuaternionDiff(list(pose), last_pose) > r["critical_quaternion_diff"] or
                                              r["stamp"] - r["stamp_last"] > r["time_difference_ns"])
                    pushes.append(dict(slot=n_kf, pose7=pose, lm_slot=r["lm_slot"], u=r["u"], v=r["v"], d=r["d"]) if picked else None)
                creates = [None if p is None else dict(kf_slots=list(range(n_kf + 1)), kf_new=n_kf, lm_slots=r["new_slots"])
                           for p, r in zip(pushes, rs)]
                if grp is None:
                    if pushes[0]:
                        p = pushes[0]
                        tracks[0].push_keyframe(p["slot"], p["pose7"], p["lm_slot"], p["u"], p["v"], p["d"])
                        add(tracks[0].transfer_bytes())
                        tracks[0].create_landmarks(**creates[0])
                        add(tracks[0].transfer_bytes())
                else:
                    grp.push_keyframes(pushes)
                    add(grp.transfer_bytes())
                    grp.create_landmarks(creates)
                    add(grp.transfer_bytes())
                return up, down

            def one(reqs=rs):
                if grp is None:
                    tracks[0].frame_step(opt=opt, **reqs[0])
                    return tracks[0].transfer_bytes()[:2]
                grp.frame_step(reqs, opt=opt)
                return grp.transfer_bytes()

            fn = capi.lib().kba_track_frame_step if grp is None else capi.lib().kba_track_group_frame_step
            req, out, ress, _keep, _result = capi._frame_step_records(fn, rs, 256)
            c_args = (fn, tracks[0]._p if grp is None else grp._p, req.ctypes.data_as(C.POINTER(capi.KbaFrameStepRequest)), C.byref(opt),
                      out.ctypes.data_as(C.POINTER(capi.KbaFrameStepOut)), ress)

            def one_c():
                capi._check(c_args[0](*c_args[1:]))
                return tracks[0].transfer_bytes()[:2] if grp is None else grp.transfer_bytes()

            paths = (("chain", chain, True), ("one", one, True), ("one_c_call", one_c, True),
                     ("one_rejected", lambda: one(rejected), False))
            ts = {what: [] for what, _, _ in paths}
            moved = {}
            for what, f, pushes in paths:
                moved[what] = f()
                if pushes:
                    undo()
            for rep in range(3 + args.repeats):  # the paths alternate, so that all see the same host and GPU load
                for what, f, pushes in paths:
                    t0 = time.perf_counter()
                    f()
                    if rep >= 3:
                        ts[what].append(1e3 * (time.perf_counter() - t0))
                    if pushes:
                        undo()
            for what, _, _ in paths:
                up, down = moved[what]
                print(json.dumps(dict(what=what, tracks=G, keyframes=n_kf, landmarks=n_lm, median_ms=round(float(np.median(ts[what])), 3),
                                      p90_ms=round(float(np.percentile(ts[what], 90)), 3), h2d_bytes=int(up), d2h_bytes=int(down), **info)),
                      flush=True)
            if grp is not None:
                grp.close()
        for t, _ in made:
            t.close()
    h.close()


if __name__ == "__main__":
    main()
