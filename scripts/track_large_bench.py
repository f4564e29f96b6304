"""Per-solve latency and upload of limo's default mono-lidar window, 20 keyframes with ground-plane residuals (201 reduced rows,
the large-window path): rebuilt by kba_solve_window against a track with device attachment.

A seeded synthetic config-3 drive (ground plane 0.31 m below the vehicle, 40 % lidar depth, 10 % ground landmarks) with a
20-keyframe sliding window, the max_size_optimization_window default of the mono-lidar node.  A step pushes one keyframe and solves
the window two ways:
  - rebuild  : kba_solve_window of the whole window, ground-plane lists and scale rule computed on the host;
  - device   : kba_track_solve on a track with win_rows = 201, the selected ground landmarks as candidates (4 B each), attached by
               k_track_ground; the window goes to the track's large-window solver, packed on the device.
The two agree to 1e-6 m at every step (bit for bit when ground points are attached).  Then groups of G such tracks
(kba_track_group_solve, every track replaying the same drive), and the device time of the chunk-range kernel k_pack_ranges<32> and
of the whole gather from torch.profiler in a run of its own.  Latency is host wall time around a call that returns after its
download (it ends in a device synchronise).

    python scripts/track_large_bench.py --steps 10 --warmup 3 --groups 1,32,132 --out /tmp/track_large.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W = 20
PLANE = np.array([0.0, 0.0, 1.0, 0.31])


def _card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                    text=True).splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=pl, sm_clock=sm, sm_clock_max=smax)
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return dict(gpu="unknown (%s)" % e)


class Drive:
    """keyframe k in slot k % (W + 1); step s solves keyframes s .. s + W - 1; the host mirrors the store"""

    def __init__(self, seed, n_steps):
        from limo_b200 import synth
        n_kf = W + n_steps
        win, truth = synth.make_window(3, seed=seed, n_kf=n_kf, n_lm=int(3000 * n_kf / 30), n_obs=int(40000 * n_kf / 30),
                                       return_truth=True)
        lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
        self.per_kf = []
        for k in range(n_kf):
            s = np.nonzero(win.obs_kf == k)[0]
            self.per_kf.append((lm_of_obs[s].astype(np.int32), win.obs_u[s], win.obs_v[s], win.obs_d[s]))
        self.win, self.ground = win, truth["is_gp"]
        self.poses, self.planes, self.lm = win.kf_pose.copy(), np.tile(PLANE, (n_kf, 1)), win.lm_pos.copy()

    def make_track(self, capi, h, caps):
        t = capi.Track(h, self.win.cam_intr, self.win.cam_pose, max_keyframes=W + 1, **caps)
        t.set_landmarks(np.arange(self.win.n_lm, dtype=np.int32), pos=self.win.lm_pos, weight=self.win.lm_weight)
        for k in range(W):
            self.push(t, k)
        return t

    def push(self, t, k):
        if k >= W + 1:
            t.drop_keyframe(k % (W + 1))
        lm, u, v, d = self.per_kf[k]
        t.push_keyframe(k % (W + 1), self.win.kf_pose[k], lm, u, v, d, plane4=PLANE)

    def step(self, s):
        """the step's window: base request, candidates, host lists (from the mirror) and the rebuild-path window"""
        from limo_b200.capi_types import Window
        from tests.test_track import _scale, _window_lists
        from tests.test_track_ground import _attach
        first, last = s, s + W - 1
        lm_sel, ptr, okf, ou, ov, od = _window_lists(self.per_kf, first, last)
        fixed = np.zeros(W, np.uint8); fixed[0] = 1
        sc = _scale(self.poses[first:last + 1], 0)
        base = dict(kf_slots=[k % (W + 1) for k in range(first, last + 1)], kf_fixed=fixed, lm_slots=lm_sel,
                    scale_kf0=0, scale_kf1=1, scale_weight=-1.0, scale_value=sc["scale_value"])
        cand = np.nonzero(self.ground[lm_sel])[0].astype(np.int32)
        keep, best, wgt = _attach(self.poses[first:last + 1], self.planes[first:last + 1], self.lm[lm_sel][cand])
        lists = dict(gp_lm=cand[keep], gp_kf=best[keep].astype(np.int32), gp_weight=wgt[keep]) if keep.any() else {}
        n_depth, n_gp = int((od > 0).sum()), int(keep.sum())
        weight = 1000.0   # addScaleRegularization's weight (reference cpp:703-716) for the rebuilt window
        if n_depth > 10 or n_gp > 10:
            weight = 1000.0 / (n_depth + n_gp) if n_gp < 30 else 0.0
        rebuild = Window(self.poses[first:last + 1], fixed, self.win.cam_intr, self.win.cam_pose, self.lm[lm_sel],
                         self.win.lm_weight[lm_sel], ptr, okf, ou, ov, od, kf_plane=self.planes[first:last + 1],
                         plane_reg_weight=10.0 if n_gp else 0.0, plane_dist_fixed=n_depth < 10, scale_kf0=0, scale_kf1=1,
                         scale_weight=weight, scale_value=sc["scale_value"], **lists)
        return dict(base, gp_lm=cand, plane_reg_weight=-1.0), rebuild, n_gp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--groups", default="1,32,132")
    ap.add_argument("--profile-solves", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from limo_b200 import capi
    n_steps = a.warmup + a.steps
    dr = Drive(0x6A0E, n_steps)
    h = capi.Handle(0)
    opt = capi.default_options()
    caps = dict(max_landmarks=dr.win.n_lm, max_measurements=sum(len(x[0]) for x in dr.per_kf), win_keyframes=W,
                win_landmarks=dr.win.n_lm, win_observations=max(sum(len(dr.per_kf[k][0]) for k in range(s, s + W)) for s in range(n_steps)),
                win_ground=dr.win.n_lm, win_rows=10 * W + 1)
    out = dict(card=_card(), window=dict(keyframes=W, config=3, reduced_rows=10 * W + 1), steps=a.steps, warmup=a.warmup)
    # ---- one window two ways
    td = dr.make_track(capi, h, caps)
    steps = []   # requests of every step, kept for the group runs (the group replays the same states)
    lat = {"rebuild": [], "device": []}
    up = {"rebuild": [], "device": []}
    attached, max_dt = [], 0.0
    for s in range(n_steps):
        if s:
            dr.push(td, W - 1 + s)
        dev, rebuild, n_gp = dr.step(s)
        steps.append(dev)
        t0 = time.perf_counter(); rw = h.solve_window(rebuild, opt); t1 = time.perf_counter()
        rd = td.solve(opt=opt, **dev); t2 = time.perf_counter()
        up_d = td.transfer_bytes()[0]
        assert rw.c.status == 0 and rd.c.status == 0
        max_dt = max(max_dt, float(np.max(np.abs(rw.kf_pose[:, 4:] - rd.kf_pose[:, 4:]))))
        assert max_dt <= 1e-6, max_dt
        n_lm = len(dev["lm_slots"])
        dr.lm[dev["lm_slots"]] = rd.lm_pos[:n_lm]
        dr.poses[s:s + W], dr.planes[s:s + W] = rd.kf_pose, rd.kf_plane
        if s >= a.warmup:
            b = h.batch([rebuild]); up["rebuild"].append(b.transfer_bytes()[0]); b.close()
            lat["rebuild"].append(t1 - t0); lat["device"].append(t2 - t1)
            up["device"].append(up_d)
            attached.append(n_gp)
    td.close()
    out["single"] = {k: dict(ms_median=round(1e3 * float(np.median(lat[k])), 3), ms_p90=round(1e3 * float(np.percentile(lat[k], 90)), 3),
                             h2d_bytes_mean=int(np.mean(up[k]))) for k in lat}
    out["attached_per_step"] = attached
    out["max_translation_difference_m"] = max_dt
    print(json.dumps(out["single"]), flush=True)
    # ---- groups of device-attached tracks
    out["groups"] = []
    for G in [int(x) for x in a.groups.split(",")]:
        tracks = [dr.make_track(capi, h, caps) for _ in range(G)]
        grp = capi.TrackGroup(h, tracks)
        times = []
        for s in range(n_steps):
            if s:
                for t in tracks:
                    dr.push(t, W - 1 + s)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = grp.solve([steps[s]] * G, opt, iterations_capacity=1)
            t1 = time.perf_counter()
            assert all(r.c.status == 0 for r in res)
            if s >= a.warmup:
                times.append(t1 - t0)
        row = dict(G=G, ms_per_group_solve_median=round(1e3 * float(np.median(times)), 3),
                   windows_per_s=round(G / float(np.median(times)), 1), h2d_bytes=grp.transfer_bytes()[0])
        out["groups"].append(row)
        print(json.dumps(row), flush=True)
        grp.close()
        for t in tracks:
            t.close()
    # ---- chunk-range kernel and gather device time (profiler run of its own: a single track and a group of the largest G)
    from torch.profiler import ProfilerActivity, profile
    G = max(int(x) for x in a.groups.split(","))
    t1, tracks = dr.make_track(capi, h, caps), [dr.make_track(capi, h, caps) for _ in range(G)]
    grp = capi.TrackGroup(h, tracks)
    kern = {}
    us = lambda e: getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    for name, fn in (("single", lambda: t1.solve(opt=opt, **steps[0])), ("group_%d" % G, lambda: grp.solve([steps[0]] * G, opt, 1))):
        fn()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_solves):
                fn()
        avg = prof.key_averages()
        rng = [e for e in avg if "k_pack_ranges" in e.key]
        pack = [e for e in avg if "k_pack_" in e.key or "k_track_" in e.key]
        kern[name] = dict(k_pack_ranges_us_per_solve=round(sum(us(e) for e in rng) / a.profile_solves, 2) if rng else "not measured",
                          gather_and_pack_us_per_solve=round(sum(us(e) for e in pack) / a.profile_solves, 2) if pack else "not measured",
                          kernels=sorted(e.key for e in rng))
    out["kernel"] = kern
    print(json.dumps(kern), flush=True)
    grp.close(); t1.close()
    for t in tracks:
        t.close()
    h.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
