"""limo's camera callback as one store call (kba_track_camera_step and its group form) against the chain it replaces, for one
track and for groups of tracks, with and without lidar clouds.

Stores and frames are those of scripts/frame_step_bench.py (12 keyframes, 4000 landmarks, one camera; every frame selected by
the time scheme); with lidar, each track's frame comes with a KITTI-sized cloud (synth.make_lidar_scene, 8 scenes in turn).
  chain: frame_step / TrackGroup.frame_step, the post-push landmark lists built on the host from the creation's flags, then
         keyframe_solve / TrackGroup.keyframe_solve when the frame solves;
  one:   camera_step / TrackGroup.camera_step.
A solving frame (solve = "always") and a non-solving one (solve = "never") are timed separately.  Every step starts from fresh
clones of the same stores (made outside the timing), the paths alternate in one process, and the first step's outputs and
snapshots of both paths are checked equal.  Per path: wall time per step (median and p90 of --repeats after warm-up), one JSON
line per measurement with the GPU name and its power limit.
Usage: python scripts/camera_step_bench.py [--repeats 10] [--groups 1,32,132]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

N_KF, N_LM, N_SCENES = 12, 4000, 8


def solve_kw(req, solve):
    new = [int(x) for x in req["new_slots"]]
    cand = list(range(N_LM)) + new
    tags = [-2] * N_LM + list(range(len(new)))
    return dict(solve=solve, cand_slots=cand, cand_tags=tags, max_window=N_KF + 1, draws=np.arange(len(cand) + 1),
                voxel_size=(0.5, 0.5, 0.3), scale_weight=-1.0, scale_value=1.5)


def chain(tracks, grp, reqs, opt):
    """the frame step, the host's lists, the solve block"""
    from limo_b200 import capi
    fs = [{k: v for k, v in r.items() if k in capi._STEP_KEYS} for r in reqs]
    steps = [tracks[0].frame_step(opt=opt, **fs[0])] if grp is None else grp.frame_step(fs, opt=opt)
    kfs = []
    for r, s in zip(reqs, steps):
        if r["solve"] == "never":
            kfs.append(None)
            continue
        keep = [t == -2 or (s["selected"] and (t == -1 or (t >= 0 and s["flags"][t] & 1))) for t in r["cand_tags"]]
        kw = {k: v for k, v in r.items() if k in ("max_window", "draws", "voxel_size", "scale_weight", "scale_value")}
        kfs.append(dict(kf_slots=list(r["kf_slots"]) + ([r["kf_new"]] if s["selected"] else []),
                        lm_slots=[c for c, f in zip(r["cand_slots"], keep) if f], **kw))
    if any(k is not None for k in kfs):
        sol = [tracks[0].keyframe_solve(opt=opt, **kfs[0])] if grp is None else grp.keyframe_solve(kfs, opt=opt)
    else:
        sol = [None] * len(reqs)
    return steps, sol


def one(tracks, grp, reqs, opt):
    full = [{k: v for k, v in r.items()} for r in reqs]
    return [tracks[0].camera_step(opt_adjust=opt, opt_solve=opt, **full[0])] if grp is None else \
        grp.camera_step(full, opt_adjust=opt, opt_solve=opt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--groups", default="1,32,132")
    args = ap.parse_args()
    from frame_step_bench import store
    from group_select_bench import card
    from limo_b200 import capi, synth
    info = card()
    h = capi.Handle(0)
    opt = capi.default_options()
    opt.solver_time_sec = 0.0
    scenes = [synth.make_lidar_scene(seed=0xBA5E0004 + s) for s in range(N_SCENES)]
    T = scenes[0][1]
    groups = [int(g) for g in args.groups.split(",")]
    made = [store(h, N_KF, N_LM, seed=s) for s in range(max(groups))]
    for lidar in (False, True):
        for G in groups:
            for solve in ("always", "never"):
                reqs = []
                for i, (_t, r) in enumerate(made[:G]):
                    q = dict(r, **solve_kw(r, solve))
                    if lidar:
                        del q["d"]
                        q.update(cloud=scenes[i % N_SCENES][0], T_cam_lidar=T)
                    reqs.append(q)

                def fresh():
                    ts = [m[0].clone() for m in made[:G]]
                    return ts, (capi.TrackGroup(h, ts) if G > 1 else None)

                def close(ts, grp):
                    if grp is not None:
                        grp.close()
                    for t in ts:
                        t.close()

                # both paths' outputs and stores, once
                ta, ga = fresh()
                tb, gb = fresh()
                steps, sol = chain(ta, ga, reqs, opt)
                got = one(tb, gb, reqs, opt)
                for s, x, o in zip(steps, sol, got):
                    assert o["step"]["selected"] == s["selected"] and np.array_equal(o["step"]["flags"], s["flags"])
                    assert o["solved"] == (x is not None)
                    if x is not None:
                        assert np.array_equal(o["solve"]["result"].kf_pose.view(np.int64), x["result"].kf_pose.view(np.int64))
                        assert np.array_equal(o["solve"]["cand"], x["cand"])
                assert all(bytes(a.snapshot()) == bytes(b.snapshot()) for a, b in zip(ta, tb))
                close(ta, ga); close(tb, gb)
                paths = (("chain", chain), ("one", one))
                ts = {what: [] for what, _ in paths}
                for rep in range(2 + args.repeats):
                    for what, f in paths:
                        tr, gr = fresh()
                        t0 = time.perf_counter()
                        f(tr, gr, reqs, opt)
                        if rep >= 2:
                            ts[what].append(1e3 * (time.perf_counter() - t0))
                        close(tr, gr)
                for what, _ in paths:
                    print(json.dumps(dict(what=what, tracks=G, lidar=lidar, frame="solving" if solve == "always" else "not_solving",
                                          keyframes=N_KF, landmarks=N_LM, median_ms=round(float(np.median(ts[what])), 3),
                                          p90_ms=round(float(np.percentile(ts[what], 90)), 3), outputs_equal=True, **info)), flush=True)
    for t, _ in made:
        t.close()
    h.close()


if __name__ == "__main__":
    main()
