"""A parameter sweep of limo's tuning script as one track group: windows/s with one kba_options per track.

keyframe_bundle_adjustment_ros_tool/res/tune_parameters_kitti.py runs 110 settings (depth_thres 0.10 .. 0.19 x repr_thres
1.0 .. 2.0, shrubbery weight 0.9) one after another.  Here G tracks replay one synthetic 12-keyframe ground-plane recording
(tests/sweep_drive.py), track i with grid point i.  A step tracks the next frame against each store (adjust_pose), pushes it as
a keyframe and solves each sliding window, which writes the window back into its store.  Three ways to run it:
  - per-window group : kba_track_group_adjust_pose_opts + kba_track_group_solve_opts, one launch each for all G tracks;
  - single           : G kba_track_adjust_pose + G kba_track_solve calls with the same options (what a sweep costs without them);
  - uniform group    : the same group calls with one option set for every track (limo's defaults): the cost of per-window
                       options on their own.
Reported per way: windows/s of the solves and of the whole step, and the LM iterations per window and step (mean, max); and the
largest pose difference between the per-window group and the single solves.  The timed region of a call ends with its device
synchronise.

    python scripts/sweep_bench.py --groups 110 --steps 6 --warmup 2 --out /tmp/sweep.json
    python scripts/sweep_bench.py --dry-run        # the grid and the drive on the CPU, no device
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import sweep_drive as sw  # noqa: E402


def _card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    text=True).splitlines()[0]
        name, pl, smax = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=pl, sm_clock_max=smax)
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return dict(gpu="unknown (%s)" % e)


def _iters(res):
    return sum(s.num_iterations for s in res.solves)


def run(args):
    from limo_b200 import capi
    G = args.groups
    dr = sw.SweepDrive(W=args.window, steps=args.warmup + args.steps)
    opts = sw.options(sw.grid(G))
    uniform = capi.default_options()
    h = capi.Handle(0)
    ways = {}
    for way in ("per_window_group", "single", "uniform_group"):
        tracks = [dr.make(h) for _ in range(G)]
        ways[way] = dict(tracks=tracks, grp=None if way == "single" else capi.TrackGroup(h, [t for t, _ in tracks]),
                         t_solve=0.0, t_step=0.0, iters=[], poses=[])
    for step in range(dr.steps):
        timed = step >= args.warmup
        for way, st in ways.items():
            tracks, grp = st["tracks"], st["grp"]
            o = [uniform] * G if way == "uniform_group" else opts
            t0 = time.perf_counter()
            if step:
                frames = [dr.frame(m, step) for _, m in tracks]
                if grp is not None:
                    fr = grp.adjust_pose(frames, o if way == "per_window_group" else uniform)
                else:
                    fr = [t.adjust_pose(opt=o[i], **frames[i]) for i, (t, _) in enumerate(tracks)]
                for i, (t, m) in enumerate(tracks):
                    dr.push(t, m, step, fr[i].kf_pose[0])
            reqs = [m.request(step) for _, m in tracks]
            t1 = time.perf_counter()
            if grp is not None:
                res = grp.solve(reqs, o if way == "per_window_group" else uniform)
            else:
                res = [t.solve(opt=o[i], **reqs[i]) for i, (t, _) in enumerate(tracks)]
            t2 = time.perf_counter()
            for (_, m), r in zip(tracks, res):
                m.record(r)
            if timed:
                st["t_solve"] += t2 - t1
                st["t_step"] += t2 - t0
                st["iters"].append([_iters(r) for r in res])
            st["poses"] = [r.kf_pose.copy() for r in res]
    dpose = max(np.abs(a - b).max() for a, b in zip(ways["per_window_group"]["poses"], ways["single"]["poses"]))
    out = dict(card=_card(), groups=G, window_keyframes=args.window, steps=args.steps, warmup=args.warmup,
               max_pose_diff_group_vs_single=float(dpose))
    for way, st in ways.items():
        it = np.array(st["iters"])
        out[way] = dict(solve_windows_per_s=G * args.steps / st["t_solve"], step_windows_per_s=G * args.steps / st["t_step"],
                        lm_iterations_mean=float(it.mean()), lm_iterations_max=int(it.max()))
        if st["grp"] is not None:
            st["grp"].close()
        for t, _ in st["tracks"]:
            t.close()
    h.close()
    return out


def dry_run(args):
    """the grid, the options and the drive's requests of every track, on the CPU"""
    pts = sw.grid(args.groups)
    assert len(pts) == args.groups and len(set(sw.grid())) == 100
    dr = sw.SweepDrive(W=args.window, steps=args.warmup + args.steps)
    reqs = [dr.base.request(s) for s in range(dr.steps)]
    frames = [dr.frame(dr.base, s) for s in range(1, dr.steps)]
    return dict(groups=args.groups, grid_points=len(set(pts)), depth_thres=sw.DEPTH_THRES, repr_thres=sw.REPR_THRES,
                shrubbery_landmarks=len(dr.shrubbery), landmarks=int(dr.base.win.n_lm),
                window_landmarks=[len(r["lm_slots"]) for r in reqs], frame_measurements=[len(f["lm_slot"]) for f in frames])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--groups", type=int, default=110, help="tracks in the group (grid points, in the tuning script's order)")
    ap.add_argument("--window", type=int, default=12, help="keyframes per sliding window")
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dry-run", action="store_true")
    args = ap.parse_args()
    out = dry_run(args) if args.dry_run else run(args)
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
