"""The ranked selection and its solve against the host-ranked path, for one track and for groups of tracks.

Stores as in scripts/select_bench.py (every landmark measured by 6 consecutive keyframes, one camera, limo's mono-lidar voxel
parameters; 12 keyframes / 1.1k landmarks, 20 / 8k and 20 / 20k), sized here so that every landmark fits a solve; a quarter of
the landmarks carry the AddDepth flag; caps 400 per bin and AddDepth (i, 50) for every keyframe, as limo configures them.
  ranked:  kba_track_rank_landmarks + kba_track_solve_ranked (G = 1), or their group forms (G > 1);
  host:    kba_track_select_landmarks + kba_track_depth_costs + kba_track_solve on the uploaded list (or the group forms), the
           ranking done between them by the caller.  The caller's ranking is not in this wall time: it is timed on its own in
           `host_rank_ms`, as the Python restatement of tests/test_track_rank.py does it (Python: slower than a C++ caller).
Both paths solve the same selection with one Levenberg-Marquardt iteration and no trimming round, so that the solve stays small
next to the selection.  Per path: wall time per step (median and p90, each step ending in the call's synchronisation), bytes up
and down per step (kba_track_{,group_}transfer_bytes summed over the calls), and, in a run of its own under torch.profiler, the
summed device time of the selection kernels per step: k_sel_* + k_rk_* (ranked), k_sel_* + k_up_* (host).  One JSON line per measurement, with the
GPU name, its power limit and its max SM clock.
Usage: python scripts/rank_bench.py [--repeats 10] [--groups 1,32,132] [--stores 12:1100,20:8000,20:20000]"""
import argparse
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


def store(h, n_kf, n_lm, seed):
    """select_bench's store with window capacities for a solve of every landmark"""
    from limo_b200 import capi
    rng = np.random.default_rng(seed)
    per_kf = 6 * n_lm // n_kf + 1
    t = capi.Track(h, [[700.0, 600.0, 190.0]], [[0.5, 0.5, -0.5, 0.5, 0.0, 0.0, 0.0]], max_keyframes=n_kf, max_landmarks=n_lm,
                   max_measurements=n_kf * per_kf, win_keyframes=n_kf, win_landmarks=n_lm, win_observations=n_kf * per_kf)
    pos = np.column_stack([rng.uniform(-5, 80, n_lm), rng.uniform(-30, 30, n_lm), rng.uniform(-2, 6, n_lm)])
    t.set_landmarks(np.arange(n_lm, dtype=np.int32), pos=pos, weight=np.ones(n_lm))
    first = rng.integers(0, n_kf - 5, n_lm)
    for k in range(n_kf):
        lm = np.nonzero((first <= k) & (k < first + 6))[0].astype(np.int32)
        pose = [1.0, 0.0, 0.0, 0.0, -1.5 * k, 0.0, 0.0]
        t.push_keyframe(k, pose, lm, rng.uniform(0, 1200, len(lm)), rng.uniform(0, 380, len(lm)), np.full(len(lm), -1.0))
    elig = (rng.random(n_lm) < 0.25).astype(np.uint8)
    return t, elig


def host_rank(q, elig, depth_out, n_kf):
    """the caller's ranking of the selection quantities and the depth costs (tests/test_track_rank.py's restatement)"""
    from tests.test_track_rank import rank_quantities
    n = len(q["bin"])
    flow = {c: q["flow"][c] for c in range(n)}
    seen = {c: int(q["seen"][c]) for c in range(n)}
    off, cand, cost = depth_out
    el = np.flatnonzero(q["cheiral"].astype(bool) & elig.astype(bool))
    ent = [(50, [(int(el[cand[i]]), float(cost[i])) for i in range(off[k], off[k + 1])]) for k in range(n_kf)]
    out, _ = rank_quantities(list(q["near_order"]), flow, [c for c in range(n) if q["bin"][c] == 1],
                             [c for c in range(n) if q["bin"][c] == 2], seen, ent, (400, 400, 400), np.random.randint(0, 2**31 - 1, n))
    return np.array(sorted(out), np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--groups", default="1,32,132")
    ap.add_argument("--stores", default="12:1100,20:8000,20:20000")
    args = ap.parse_args()
    import torch
    from group_select_bench import card, timed
    from limo_b200 import capi
    from torch.profiler import ProfilerActivity, profile
    info = card()
    h = capi.Handle(0)
    with profile(activities=[ProfilerActivity.CUDA]):  # CUPTI's set-up, outside every measured session
        torch.cuda.synchronize()
    opt = capi.default_options()
    opt.num_trim_rounds, opt.final_solver_iterations = 0, 1
    groups = [int(g) for g in args.groups.split(",")]
    for spec in args.stores.split(","):
        n_kf, n_lm = (int(x) for x in spec.split(":"))
        kf = np.arange(n_kf, dtype=np.int32)
        lm = np.arange(n_lm, dtype=np.int32)
        fixed = np.r_[[1, 1], np.zeros(n_kf - 2)].astype(np.uint8)
        depth = [(i, 50) for i in range(n_kf)]
        made = [store(h, n_kf, n_lm, seed=s) for s in range(max(groups))]
        rng = np.random.default_rng(0)
        for G in groups:
            tracks, eligs = [m[0] for m in made[:G]], [m[1] for m in made[:G]]
            grp = capi.TrackGroup(h, tracks) if G > 1 else None
            draws = lambda n: rng.integers(0, 2**31 - 1, n)  # noqa: E731
            rank_req = [dict(kf_slots=kf, lm_slots=lm, elig=e, depth=depth, draws=draws, **CAPS, **PRM) for e in eligs]
            sel = {}  # the ranked selection of each track: the list the host path solves

            def ranked():
                if grp is None:
                    r = [tracks[0].rank_landmarks(**rank_req[0])]
                    b = tracks[0].transfer_bytes()[:2]
                    tracks[0].solve_ranked(kf, fixed, opt=opt)
                    c = tracks[0].transfer_bytes()[:2]
                else:
                    r = grp.rank_landmarks(rank_req)
                    b = grp.transfer_bytes()
                    grp.solve_ranked([dict(kf_slots=kf, kf_fixed=fixed)] * G, opt=opt)
                    c = grp.transfer_bytes()
                for i, x in enumerate(r):
                    sel[i] = x["cand"]
                return b[0] + c[0], b[1] + c[1]

            def host():
                if grp is None:
                    q = [tracks[0].select_landmarks(kf, lm, **PRM)]
                    b = tracks[0].transfer_bytes()[:2]
                    el = np.flatnonzero(q[0]["cheiral"].astype(bool) & eligs[0].astype(bool)).astype(np.int32)
                    tracks[0].depth_costs(kf, el)
                    c = tracks[0].transfer_bytes()[:2]
                    tracks[0].solve(kf, fixed, sel[0], opt=opt)
                    d = tracks[0].transfer_bytes()[:2]
                else:
                    q = grp.select_landmarks([dict(kf_slots=kf, lm_slots=lm, **PRM)] * G)
                    b = grp.transfer_bytes()
                    grp.depth_costs([dict(kf_slots=kf, lm_slots=np.flatnonzero(x["cheiral"].astype(bool) & e.astype(bool)).astype(np.int32))
                                     for x, e in zip(q, eligs)])
                    c = grp.transfer_bytes()
                    grp.solve([dict(kf_slots=kf, kf_fixed=fixed, lm_slots=sel[i]) for i in range(G)], opt=opt)
                    d = grp.transfer_bytes()
                return b[0] + c[0] + d[0], b[1] + c[1] + d[1]

            up_r, down_r = ranked()
            up_h, down_h = host()
            q0 = tracks[0].select_landmarks(kf, lm, **PRM)
            el0 = np.flatnonzero(q0["cheiral"].astype(bool) & eligs[0].astype(bool)).astype(np.int32)
            t0 = time.perf_counter()
            host_rank(q0, eligs[0], tracks[0].depth_costs(kf, el0), n_kf)
            host_rank_ms = 1e3 * (time.perf_counter() - t0)
            for what, fn, up, down, keys in (("ranked", ranked, up_r, down_r, ("k_sel_", "k_rk_")), ("host", host, up_h, down_h, ("k_sel_", "k_up_"))):
                med, p90 = timed(fn, args.repeats, warmup=2)
                fn()
                with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
                    for _ in range(3):
                        fn()
                avg = prof.key_averages()
                sel_us = sum(e.device_time_total for e in avg if any(k in e.key for k in keys))
                line = dict(what=what, tracks=G, keyframes=n_kf, landmarks=n_lm, selected=int(len(sel[0])), median_ms=round(med, 3),
                            p90_ms=round(p90, 3), h2d_bytes=int(up), d2h_bytes=int(down),
                            selection_kernels=list(keys), selection_device_ms=round(sel_us / 1e3 / 3, 3), **info)
                if what == "host":
                    line["host_rank_ms_per_track"] = round(host_rank_ms, 3)
                print(json.dumps(line), flush=True)
            if grp is not None:
                grp.close()
        for t, _ in made:
            t.close()
    h.close()


if __name__ == "__main__":
    main()
