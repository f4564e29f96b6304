#!/usr/bin/env python
"""adjustPoseOnly per frame (reference cpp:820-888) through three paths, and frames/s of track groups:
  - kba_solve_window on the equivalent landmarks_fixed window (what the facade did per frame: allocate, pack, capture, solve, free);
  - a resident one-window kba_batch_solve (the general kernels, cached CUDA graph) plus its download;
  - kba_track_adjust_pose (k_adjust_pose: one kernel per frame, landmarks read from the track's store).
Frames: the ~1000-observation frames of scripts/motion_only_bench.py, and a production-size frame (<= 500 landmarks).
Prints one JSON line; the card's name, power limit and SM clock are read in the same call."""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from limo_b200 import capi, synth, geometry as g
from limo_b200.capi_types import Window


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [x.strip() for x in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


class Frame:
    """the newest keyframe of a seeded synthetic window: one run per landmark, store slot = landmark id, speed prior"""

    def __init__(self, seed, n_lm, n_obs, max_lm=None):
        win, truth = synth.make_window(2, n_kf=12, n_lm=n_lm, n_obs=n_obs, seed=seed, return_truth=True)
        k = win.n_kf - 1
        lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
        sel = np.nonzero(win.obs_kf == k)[0]
        if max_lm:
            sel = sel[:max_lm]
        self.lm = lm_of_obs[sel].astype(np.int32)
        self.u, self.v, self.d = win.obs_u[sel], win.obs_v[sel], win.obs_d[sel]
        self.cam_intr, self.cam_pose, self.n_lm_store = win.cam_intr, win.cam_pose, win.n_lm
        self.lm_pos, self.pose7 = truth["lm_pos"], win.kf_pose[k]
        Tb, Tb2 = g.pose_to_iso(truth["kf_pose"][k - 1]), g.pose_to_iso(truth["kf_pose"][k - 2])
        self.speed = dict(weight=0.7, dt=0.1, v_before=(Tb @ g.iso_inv(Tb2))[:3, 3] / 0.1, T_origin_before=g.iso_to_pose(g.iso_inv(Tb)))

    def window(self):
        n = len(self.lm)  # one observation per landmark in a mono frame
        s = self.speed
        return Window(kf_pose=self.pose7[None], kf_fixed=[0], cam_intr=self.cam_intr, cam_pose=self.cam_pose, lm_pos=self.lm_pos[self.lm],
                      lm_weight=np.ones(n), lm_obs_ptr=np.arange(n + 1), obs_kf=np.zeros(n, np.int32), obs_u=self.u, obs_v=self.v,
                      obs_d=self.d, landmarks_fixed=True, speed_kf=0, speed_weight=s["weight"], speed_dt=s["dt"],
                      speed_v_before=s["v_before"], speed_T_origin_before=s["T_origin_before"])

    def track(self, h):
        t = capi.Track(h, self.cam_intr, self.cam_pose, max_keyframes=3, max_landmarks=self.n_lm_store, max_measurements=1,
                       win_keyframes=3, win_landmarks=len(self.lm), win_observations=len(self.lm))
        t.set_landmarks(np.arange(self.n_lm_store, dtype=np.int32), pos=self.lm_pos, weight=np.ones(self.n_lm_store))
        return t

    def args(self):
        return dict(pose7=self.pose7, lm_slot=self.lm, u=self.u, v=self.v, d=self.d, speed=self.speed)


def lat(fn, n, warm=20):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    ts = np.array(ts) * 1e3
    return {"median_ms": float(np.median(ts)), "p90_ms": float(np.percentile(ts, 90))}


def main():
    n_calls = int(os.environ.get("ADJUST_POSE_BENCH_CALLS", "200"))
    info = gpu_info()
    h = capi.Handle(0)
    opt = capi.default_options()
    opt.min_landmarks_for_trimming = 30  # adjustPoseOnly (cpp:865)
    out = {"gpu": info, "calls": n_calls}
    shapes = {"motion_only_bench_1000obs": dict(n_lm=1200, n_obs=12000), "production_500lm": dict(n_lm=1200, n_obs=12000, max_lm=500)}
    for name, kw in shapes.items():
        fr = Frame(100, **kw)
        win = fr.window()
        t = fr.track(h)
        b = h.batch([win])
        rg = h.solve_window(win, opt)
        rt = t.adjust_pose(opt=opt, **fr.args())
        r = {"observations": len(fr.lm),
             "solve_window": lat(lambda: h.solve_window(win, opt), n_calls),
             "batch_resident": lat(lambda: (b.solve(opt), b.download()), n_calls),
             "track_adjust_pose": lat(lambda: t.adjust_pose(opt=opt, **fr.args()), n_calls),
             "max_dt_m_vs_general": float(np.linalg.norm(rt.kf_pose[0, 4:] - rg.kf_pose[0, 4:])),
             "iterations": [int(sum(s.num_iterations for s in rt.solves)), int(sum(s.num_iterations for s in rg.solves))],
             "h2d_d2h_bytes_track": list(t.transfer_bytes()[:2])}
        b.close(); t.close()
        out[name] = r
    # ---- group throughput against the resident batch of the same motion-only windows
    base = [Frame(200 + i, n_lm=1200, n_obs=12000) for i in range(8)]
    grp = {}
    worst = 0.0
    for G in (1, 32, 132, 264, 1024):
        frames = [base[i % 8] for i in range(G)]
        tracks = [f.track(h) for f in frames]
        grp_h = capi.TrackGroup(h, tracks)
        fargs = [f.args() for f in frames]
        batch = h.batch([f.window() for f in frames])
        reps = 20 if G <= 264 else 8
        for _ in range(2):
            res = grp_h.adjust_pose(fargs, opt, iterations_capacity=1)
            batch.solve(opt)
        t0 = time.perf_counter()
        for _ in range(reps):
            grp_h.adjust_pose(fargs, opt, iterations_capacity=1)
        tg = (time.perf_counter() - t0) / reps
        t0 = time.perf_counter()
        for _ in range(reps):
            batch.solve(opt)
            bres = batch.download()
        tb = (time.perf_counter() - t0) / reps
        for a, c in zip(res, bres):
            worst = max(worst, float(np.linalg.norm(a.kf_pose[0, 4:] - c.kf_pose[0, 4:])))
        # per call (Python binding included) and per device time of the solve (k_adjust_pose / the batch's graph launch)
        grp[str(G)] = {"group_frames_per_s": G / tg, "batch_frames_per_s": G / tb,
                       "group_device_frames_per_s": G / res[0].c.time_sec, "batch_device_frames_per_s": G / bres[0].c.time_sec}
        batch.close(); grp_h.close()
        for t in tracks:
            t.close()
    out["group"] = grp
    out["group_max_dt_m_vs_batch"] = worst
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    h.close()


if __name__ == "__main__":
    main()
