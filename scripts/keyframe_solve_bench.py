"""limo's solve block -- deactivateKeyframes, updateLabels, solve() -- as one store call against the chain of calls it replaces, for
one track and for groups of tracks.

Stores as in scripts/rank_bench.py (every landmark measured by 6 consecutive keyframes, one camera, limo's mono-lidar voxel
parameters; 12 keyframes / 4k landmarks and 20 / 8k), a quarter of the landmarks ground.  Each step passes every keyframe and
landmark as active with min_window above the window, so that the deactivation keeps them all and every step is the same work;
200 tracklets per track with outlier, shrubbery and ground labels, 20 retained outliers, caps 400 per bin and AddDepth (i, 50) for
every keyframe.  The solve is one Levenberg-Marquardt iteration without trimming rounds, so that it stays small next to the rest.
  chain: deactivate_keyframes, the caller's compaction and updateLabels (numpy), set_landmarks (shrubbery weights),
         rank_landmarks, solve_ranked -- or their group forms (G > 1);
  one:   keyframe_solve (G = 1) or TrackGroup.keyframe_solve.
  one_c_call: the C call of `one` alone, on requests built once before the timing (the binding's per-call builders left out).
chain and one go through the Python binding.  Per path: wall time per step (median and p90 of --repeats after warm-up, the paths
alternating, each step ending in its calls' synchronisation), bytes up and down per step (transfer_bytes summed over the calls),
and, in a run of its own under torch.profiler, the summed device time of every kernel per step.  One JSON line per measurement,
with the GPU name, its power limit and its max SM clock.
Usage: python scripts/keyframe_solve_bench.py [--repeats 30] [--groups 1,32,132] [--stores 12:4000,20:8000]"""
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

PRM = dict(voxel_size=(0.5, 0.5, 0.3), roi_far=40.0, roi_middle=15.0)
CAPS = dict(max_near=400, max_middle=400, max_far=400)
CLASSES = {1: 1, 2: 2, 3: 4}  # outliers, shrubbery, ground


def request(n_kf, n_lm, seed):
    rng = np.random.default_rng(seed)
    lm = np.arange(n_lm, dtype=np.int32)
    trk = np.column_stack([rng.choice(n_lm, 200, replace=False), rng.choice([0, 1, 2, 3], 200, p=[0.5, 0.05, 0.2, 0.25]),
                           (rng.random(200) < 0.02).astype(int)])
    return dict(kf_slots=np.arange(n_kf, dtype=np.int32), lm_slots=lm, min_window=n_kf + 2, max_window=n_kf,
                lm_ground=(rng.random(n_lm) < 0.25).astype(np.uint8), tracklets=trk, label_classes=CLASSES,
                outliers=np.sort(rng.choice(n_lm, 20, replace=False)).astype(np.int32), shrubbery_weight=0.5,
                depth=[(i, 50) for i in range(n_kf)], **CAPS, **PRM)


def labels(r, lm_active):
    """the caller's updateLabels between the deactivation and the ranking: candidates, their ground flags, shrubbery slots"""
    lm = r["lm_slots"]
    active = lm_active.astype(bool)
    outl = np.zeros(len(lm), bool)
    outl[np.searchsorted(lm, r["outliers"])] = True
    outl &= active
    ground = r["lm_ground"].astype(bool).copy()
    slot, label, iso = r["tracklets"].T
    cls = np.array([CLASSES.get(int(x), 0) for x in label])
    outl[slot[(iso == 1) | (cls & 1 > 0)]] = True
    act = active[slot]
    shrub = slot[act & (cls & 2 > 0)].astype(np.int32)
    ground[slot[act]] = cls[act] & 4 > 0
    keep = active & ~outl
    return lm[keep], ground[keep].astype(np.uint8), shrub


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--groups", default="1,32,132")
    ap.add_argument("--stores", default="12:4000,20:8000")
    args = ap.parse_args()
    import torch
    from group_select_bench import card
    from limo_b200 import capi
    from rank_bench import store
    from torch.profiler import ProfilerActivity, profile
    info = card()
    lib = capi.lib()
    h = capi.Handle(0)
    with profile(activities=[ProfilerActivity.CUDA]):  # CUPTI's set-up, outside every measured session
        torch.cuda.synchronize()
    opt = capi.default_options()
    opt.num_trim_rounds, opt.final_solver_iterations = 0, 1
    groups = [int(g) for g in args.groups.split(",")]
    for spec in args.stores.split(","):
        n_kf, n_lm = (int(x) for x in spec.split(":"))
        made = [store(h, n_kf, n_lm, seed=s)[0] for s in range(max(groups))]
        reqs = [request(n_kf, n_lm, s) for s in range(max(groups))]
        rng = np.random.default_rng(0)
        draws = lambda n: rng.integers(0, 2**31 - 1, n)  # noqa: E731
        for G in groups:
            tracks, rs = made[:G], [dict(r, draws=draws) for r in reqs[:G]]
            grp = capi.TrackGroup(h, tracks) if G > 1 else None
            rank_keys = ("depth", "draws", *CAPS, *PRM)
            deact_keys = ("kf_slots", "lm_slots", "min_window", "max_window")

            def chain():
                up = down = 0

                def add(tb):
                    nonlocal up, down
                    up, down = up + tb[0], down + tb[1]
                if grp is None:
                    t, r = tracks[0], rs[0]
                    kf_active, _c, lm_active = t.deactivate_keyframes(**{k: r[k] for k in deact_keys})
                    add(t.transfer_bytes())
                    cand, elig, shrub = labels(r, lm_active)
                    kf = r["kf_slots"][kf_active.astype(bool)]
                    if len(shrub):
                        t.set_landmarks(shrub, weight=np.full(len(shrub), r["shrubbery_weight"]))
                        add(t.transfer_bytes())
                    t.rank_landmarks(kf, cand, elig=elig, **{k: r[k] for k in rank_keys})
                    add(t.transfer_bytes())
                    t.solve_ranked(kf, np.r_[[1], np.zeros(len(kf) - 1)].astype(np.uint8), opt=opt)
                    add(t.transfer_bytes())
                    return up, down
                out = grp.deactivate_keyframes([{k: r[k] for k in deact_keys} for r in rs])
                add(grp.transfer_bytes())
                lab = [labels(r, o[2]) for r, o in zip(rs, out)]
                kfs = [r["kf_slots"][o[0].astype(bool)] for r, o in zip(rs, out)]
                grp.set_landmarks([dict(lm_slot=s, weight=np.full(len(s), r["shrubbery_weight"])) if len(s) else None
                                   for (_c, _e, s), r in zip(lab, rs)])
                add(grp.transfer_bytes())
                grp.rank_landmarks([dict(kf_slots=kf, lm_slots=c, elig=e, **{k: r[k] for k in rank_keys})
                                    for kf, (c, e, _s), r in zip(kfs, lab, rs)])
                add(grp.transfer_bytes())
                grp.solve_ranked([dict(kf_slots=kf, kf_fixed=np.r_[[1], np.zeros(len(kf) - 1)].astype(np.uint8)) for kf in kfs], opt=opt)
                add(grp.transfer_bytes())
                return up, down

            def one():
                if grp is None:
                    tracks[0].keyframe_solve(opt=opt, **rs[0])
                    return tracks[0].transfer_bytes()[:2]
                grp.keyframe_solve(rs, opt=opt)
                return grp.transfer_bytes()

            # the C call alone, on requests built once: what the call costs without the binding's per-call request builders
            keep = []
            if grp is None:
                q, o, k, _d, rc = tracks[0]._keyframe_solve_request(256, **rs[0])
                keep.append((q, o, k, rc))
                c_args = (lib.kba_track_keyframe_solve, tracks[0]._p, C.byref(q), C.byref(opt), C.byref(o), C.byref(rc))
            else:
                cq, co, cr = (capi.KbaKfsolveRequest * G)(), (capi.KbaKfsolveOut * G)(), (capi.KbaResult * G)()
                for i, (t, r) in enumerate(zip(tracks, rs)):
                    q, o, k, _d, rc = t._keyframe_solve_request(256, **r)
                    cq[i], co[i], cr[i] = q, o, rc
                    keep.append(k)
                c_args = (lib.kba_track_group_keyframe_solve, grp._p, cq, C.byref(opt), co, cr)

            def one_c():
                capi._check(c_args[0](*c_args[1:]))
                return (tracks[0].transfer_bytes()[:2] if grp is None else grp.transfer_bytes())

            paths = (("chain", chain), ("one", one), ("one_c_call", one_c))
            ts = {what: [] for what, _ in paths}
            moved = {what: fn() for what, fn in paths}
            for rep in range(3 + args.repeats):  # the two paths alternate, so that both see the same host and GPU load
                for what, fn in paths:
                    t0 = time.perf_counter()
                    fn()
                    if rep >= 3:
                        ts[what].append(1e3 * (time.perf_counter() - t0))
            for what, fn in paths:
                with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
                    for _ in range(3):
                        fn()
                dev_us = sum(e.self_device_time_total for e in prof.key_averages()
                             if "k_" in e.key and "Memcpy" not in e.key and "Memset" not in e.key)
                up, down = moved[what]
                print(json.dumps(dict(what=what, tracks=G, keyframes=n_kf, landmarks=n_lm, median_ms=round(float(np.median(ts[what])), 3),
                                      p90_ms=round(float(np.percentile(ts[what], 90)), 3), h2d_bytes=int(up), d2h_bytes=int(down),
                                      kernel_device_ms=round(dev_us / 1e3 / 3, 3), **info)), flush=True)
            if grp is not None:
                grp.close()
        for t in made:
            t.close()
    h.close()


if __name__ == "__main__":
    main()
