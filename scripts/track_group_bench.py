"""Windows/s of track groups (kba_track_group_solve) against single track solves and the resident batch.

G tracks each replay their own seeded synthetic drive of config-2-sized windows (30 keyframes, about 3 000 landmarks and
40 000 observations per window).  A step is one keyframe push per track and one solve of every track's sliding window:
  - group      : one kba_track_group_solve for all G tracks;
  - sequential : (at --seq-groups) twin tracks over the same steps, one kba_track_solve per track;
  - resident   : kba_batch_solve of the same G windows uploaded as a batch (inputs resident, no gather, no push): the ceiling.
A drive is one of --bases synthetic sequences with the track's own seeded pixel noise on top (synthesising hundreds of
config-2 sequences would take longer than the measurement).  The selection lists of every step are built before timing (a
caller's landmark selector makes them); the timed region is pushes + solves and ends with a device synchronise.

    python scripts/track_group_bench.py --groups 1,32,132,264 --steps 5 --warmup 2 --out /tmp/track_group.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W = 30


def _card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                    text=True).splitlines()[0]
        name, pl, sm, smax = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=pl, sm_clock=sm, sm_clock_max=smax)
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return dict(gpu="unknown (%s)" % e)


class Drive:
    """keyframe k in slot k % (W + 1); step s solves keyframes s .. s + W - 1"""

    def __init__(self, base, seed):
        self.base = base
        rng = np.random.default_rng(seed)
        self.per_kf = [(lm, (u + rng.normal(0, 0.3, len(u))).astype(np.float32), (v + rng.normal(0, 0.3, len(v))).astype(np.float32), d)
                       for lm, u, v, d in base["per_kf"]]

    def window(self, step):
        """selected landmarks (>= 2 observations in the window, ascending id) and the landmark-major CSR of the window"""
        first, last = step, step + W - 1
        ks = range(first, last + 1)
        lm = np.concatenate([self.per_kf[k][0] for k in ks])
        kf = np.concatenate([np.full(len(self.per_kf[k][0]), k - first, np.int32) for k in ks])
        u, v, d = (np.concatenate([self.per_kf[k][q] for k in ks]) for q in (1, 2, 3))
        uniq, cnt = np.unique(lm, return_counts=True)
        sel = uniq[cnt >= 2].astype(np.int32)
        keep = np.isin(lm, sel)
        lm, kf, u, v, d = lm[keep], kf[keep], u[keep], v[keep], d[keep]
        order = np.lexsort((kf, lm))
        ptr = np.zeros(len(sel) + 1, np.int32)
        ptr[1:] = np.cumsum(np.bincount(np.searchsorted(sel, lm[order]), minlength=len(sel)))
        return sel, ptr, kf[order], u[order], v[order], d[order]

    def request(self, step):
        from limo_b200 import geometry as g
        sel, ptr, kf, u, v, d = self.window(step)
        poses = self.base["kf_pose"]
        T10 = g.pose_to_iso(poses[step + 1]) @ g.iso_inv(g.pose_to_iso(poses[step]))
        fixed = np.zeros(W, np.uint8); fixed[0] = 1
        return dict(kf_slots=[k % (W + 1) for k in range(step, step + W)], kf_fixed=fixed, lm_slots=sel, scale_kf0=0, scale_kf1=1,
                    scale_weight=1000.0 / max(int((d > 0).sum()), 1), scale_value=float(np.linalg.norm(T10[:3, 3])))

    def make_track(self, capi, h, caps):
        t = capi.Track(h, self.base["cam_intr"], self.base["cam_pose"], max_keyframes=W + 1, **caps)
        n_lm = self.base["n_lm"]
        t.set_landmarks(np.arange(n_lm, dtype=np.int32), pos=self.base["lm_pos"], weight=np.ones(n_lm))
        for k in range(W):
            self.push(t, k)
        return t

    def push(self, t, k):
        if k >= W + 1:
            t.drop_keyframe(k % (W + 1))
        t.push_keyframe(k % (W + 1), self.base["kf_pose"][k], *self.per_kf[k])


def make_base(seed, n_kf):
    from limo_b200 import synth
    per_window = 40000
    win = synth.make_window(2, seed=seed, n_kf=n_kf, n_lm=int(3000 * n_kf / W), n_obs=int(per_window * n_kf / W))
    lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
    per_kf = []
    for k in range(n_kf):
        s = np.nonzero(win.obs_kf == k)[0]
        per_kf.append((lm_of_obs[s].astype(np.int32), win.obs_u[s], win.obs_v[s], win.obs_d[s]))
    return dict(per_kf=per_kf, kf_pose=win.kf_pose, lm_pos=win.lm_pos, n_lm=win.n_lm, cam_intr=win.cam_intr, cam_pose=win.cam_pose)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", default="1,32,132,264")
    ap.add_argument("--seq-groups", default="132", help="group sizes at which the sequential and resident rates are measured")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--bases", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=5, help="timed solves of the resident batch")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from limo_b200 import capi
    from limo_b200.capi_types import Window
    groups = [int(x) for x in a.groups.split(",")]
    seq_groups = {int(x) for x in a.seq_groups.split(",") if x}
    n_steps = a.warmup + a.steps
    n_kf = W + n_steps
    t0 = time.time()
    bases = [make_base(0xC0DE00 + b, n_kf) for b in range(a.bases)]
    drives = [Drive(bases[i % a.bases], 0x7A0000 + i) for i in range(max(groups))]
    reqs = [[dr.request(s) for s in range(n_steps)] for dr in drives]
    win_obs = max(sum(len(dr.per_kf[k][0]) for k in range(s, s + W)) for dr in drives for s in range(n_steps))
    win_lm = max(len(r["lm_slots"]) for rr in reqs for r in rr)
    caps = dict(max_landmarks=max(b["n_lm"] for b in bases), max_measurements=max(sum(len(x[0]) for x in b["per_kf"]) for b in bases),
                win_keyframes=W, win_landmarks=win_lm, win_observations=win_obs)
    setup_s = time.time() - t0
    h = capi.Handle(0)
    opt = capi.default_options()
    out = dict(card=_card(), window=dict(keyframes=W, landmarks_max=win_lm, observations_max=win_obs), steps=a.steps,
               warmup=a.warmup, setup_s=round(setup_s, 1), results=[])

    def run(G, solve_step):
        """pushes + solves of every step; returns (windows/s over the timed steps, results of the timed steps)"""
        kept = []
        for s in range(n_steps):
            if s == a.warmup:
                torch.cuda.synchronize()
                t = time.perf_counter()
            kept.append(solve_step(s))
        torch.cuda.synchronize()
        return G * a.steps / (time.perf_counter() - t), kept[a.warmup:]

    for G in groups:
        tracks = [drives[i].make_track(capi, h, caps) for i in range(G)]
        grp = capi.TrackGroup(h, tracks)

        def group_step(s):
            if s:
                for i in range(G):
                    drives[i].push(tracks[i], W - 1 + s)
            res = grp.solve([reqs[i][s] for i in range(G)], opt, iterations_capacity=1)
            assert all(r.c.status == 0 for r in res)
            return [r.kf_pose.copy() for r in res]

        rate, group_poses = run(G, group_step)
        row = dict(G=G, group_windows_per_s=round(rate, 1), group_h2d_bytes=grp.transfer_bytes()[0])
        grp.close()
        for t in tracks:
            t.close()
        if G in seq_groups:
            twins = [drives[i].make_track(capi, h, caps) for i in range(G)]

            def seq_step(s):
                if s:
                    for i in range(G):
                        drives[i].push(twins[i], W - 1 + s)
                res = [twins[i].solve(opt=opt, **reqs[i][s]) for i in range(G)]
                assert all(r.c.status == 0 for r in res)
                return [r.kf_pose.copy() for r in res]

            seq_rate, seq_poses = run(G, seq_step)
            for t in twins:
                t.close()
            dmax = max(float(np.abs(gp[:, 4:] - sp[:, 4:]).max()) for gs, ss in zip(group_poses, seq_poses) for gp, sp in zip(gs, ss))
            # resident ceiling: the windows of the first timed step, uploaded whole
            s = a.warmup
            wins = []
            for i in range(G):
                sel, ptr, kf, u, v, d = drives[i].window(s)
                r = reqs[i][s]
                wins.append(Window(drives[i].base["kf_pose"][s:s + W], r["kf_fixed"], drives[i].base["cam_intr"], drives[i].base["cam_pose"],
                                   drives[i].base["lm_pos"][sel], np.ones(len(sel)), ptr, kf, u, v, d, scale_kf0=0, scale_kf1=1,
                                   scale_weight=r["scale_weight"], scale_value=r["scale_value"]))
            batch = h.batch(wins)
            batch.solve(opt)
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(a.repeats):
                batch.solve(opt)
            torch.cuda.synchronize()
            res_rate = G * a.repeats / (time.perf_counter() - t)
            row.update(sequential_windows_per_s=round(seq_rate, 1), group_over_sequential=round(rate / seq_rate, 2),
                       resident_windows_per_s=round(res_rate, 1), batch_upload_h2d_bytes=batch.transfer_bytes()[0],
                       max_translation_diff_group_vs_single_m=dmax)
            batch.close()
        out["results"].append(row)
        print(json.dumps(row), flush=True)
    h.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
