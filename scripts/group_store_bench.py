"""Store writes of a track group against the same writes as single calls: wall time per call, the kernels' device time, the arena
compaction against another build of the library, and the sweep's whole keyframe step with group calls only.

  (a) writes: for G tracks, G single calls against one group call, for a push of 300 and of 2500 measurements, a landmark write of
      300 rows and a keyframe-pose write of 12 rows.  Each way's time runs from the first call to the end of the last one, which
      synchronises; median and p90 over --iters calls after --warmup.
  (b) single pushes into a 20-keyframe store, one whose arena compacts on every timed push and one whose arena never does, timed
      with this library and with --other-lib (e.g. a build of the parent commit), alternately, in worker processes.
  (c) the sweep step of tests/sweep_drive.py for G tracks: group adjust_pose, group drop, group push, group solve, against the
      per-window group step of scripts/sweep_bench.py, which pushes track by track; windows/s of the whole step.
  The device time of k_store_append, k_arena_compact and k_scatter_rows comes from torch.profiler, in a run of its own.

    python scripts/group_store_bench.py --out /tmp/group_store.json [--other-lib build/parent/libkba_b200.so]
    python scripts/group_store_bench.py --dry-run        # requests and the drive on the CPU, no device
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import sweep_drive as sw  # noqa: E402
from tests.test_track_group import PLANE  # noqa: E402

KF_SLOTS = 13          # ring of keyframe slots of a write track
N_LM = 5000
CAM_INTR = np.array([[700.0, 320.0, 240.0]])
CAM_POSE = np.array([[1.0, 0, 0, 0, 0, 0, 0]])


def _card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    text=True).splitlines()[0]
        name, pl, smax = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=pl, sm_clock_max=smax)
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return dict(gpu="unknown (%s)" % e)


def _push_rows(rng, n):
    lm = np.sort(rng.choice(N_LM, n, replace=False)).astype(np.int32)
    u, v = rng.uniform(0, 640, n).astype(np.float32), rng.uniform(0, 480, n).astype(np.float32)
    d = np.where(rng.uniform(size=n) < 0.3, rng.uniform(2, 40, n), -1.0).astype(np.float32)
    return dict(lm_slot=lm, u=u, v=v, d=d)


def _pose(rng):
    q = rng.normal(size=4)
    return np.r_[q / np.linalg.norm(q), rng.normal(size=3)]


def _requests(rng, G, n_meas, n_lm_rows=300, n_kf_rows=12):
    """per track: the pushes' rows (one set reused), a landmark write and a keyframe-pose write"""
    push = [dict(pose7=_pose(rng), plane4=PLANE, **_push_rows(rng, n_meas)) for _ in range(G)]
    lmw = [dict(lm_slot=rng.choice(N_LM, n_lm_rows, replace=False).astype(np.int32), pos=rng.normal(size=(n_lm_rows, 3)),
                weight=rng.uniform(0.5, 1, n_lm_rows)) for _ in range(G)]
    kfw = [dict(kf_slots=np.arange(n_kf_rows, dtype=np.int32), pose7s=np.stack([_pose(rng) for _ in range(n_kf_rows)]),
                plane4s=np.tile(PLANE, (n_kf_rows, 1))) for _ in range(G)]
    return push, lmw, kfw


def _stats(ts):
    ts = np.asarray(ts) * 1e3
    return dict(median_ms=round(float(np.median(ts)), 4), p90_ms=round(float(np.percentile(ts, 90)), 4))


def bench_writes(args, capi, h, G, n_meas):
    rng = np.random.default_rng(G * 10 + n_meas)
    pushes, lmw, kfw = _requests(rng, G, n_meas)
    calls = args.warmup + args.iters
    caps = dict(max_keyframes=KF_SLOTS, max_landmarks=N_LM, max_measurements=n_meas * (calls + KF_SLOTS + 2), win_keyframes=12,
                win_landmarks=3000, win_observations=40000)
    out = {}
    for way in ("single", "group"):
        tracks = [capi.Track(h, CAM_INTR, CAM_POSE, **caps) for _ in range(G)]
        grp = capi.TrackGroup(h, tracks)
        t_push, t_lm, t_kf = [], [], []
        for it in range(calls):
            slot = it % KF_SLOTS
            if it >= KF_SLOTS:
                grp.drop_keyframes([slot] * G)
            t0 = time.perf_counter()
            if way == "group":
                grp.push_keyframes([dict(p, slot=slot) for p in pushes])
            else:
                for t, p in zip(tracks, pushes):
                    t.push_keyframe(slot, p["pose7"], p["lm_slot"], p["u"], p["v"], p["d"], plane4=p["plane4"])
            t1 = time.perf_counter()
            if way == "group":
                grp.set_landmarks(lmw)
            else:
                for t, r in zip(tracks, lmw):
                    t.set_landmarks(r["lm_slot"], pos=r["pos"], weight=r["weight"])
            t2 = time.perf_counter()
            if way == "group":
                grp.set_keyframe_poses(kfw)
            else:
                for t, r in zip(tracks, kfw):
                    t.set_keyframe_poses(r["kf_slots"], r["pose7s"], r["plane4s"])
            t3 = time.perf_counter()
            if it >= args.warmup:
                t_push.append(t1 - t0); t_lm.append(t2 - t1); t_kf.append(t3 - t2)
        out[way] = dict(push=_stats(t_push), set_landmarks_300=_stats(t_lm), set_keyframe_poses_12=_stats(t_kf))
        grp.close()
        for t in tracks:
            t.close()
    return out


def compaction_worker(args):
    """single pushes of --compact-meas rows into a 20-keyframe store, through the C functions every build of the library has
    (KBA_LIB_PATH): one store whose arena compacts on every timed push, one whose arena never does"""
    import ctypes as C
    from limo_b200.capi_types import KbaTrackCaps
    L = C.CDLL(os.environ["KBA_LIB_PATH"])
    vp, ip = C.c_void_p, C.c_int32
    L.kba_create.argtypes = [C.POINTER(vp), C.c_int]
    L.kba_track_create.argtypes = [vp, C.POINTER(KbaTrackCaps), ip, vp, vp, C.POINTER(vp)]
    L.kba_track_push_keyframe.argtypes = [vp, ip, vp, vp, ip, vp, vp, vp, vp, vp]
    L.kba_track_drop_keyframe.argtypes = [vp, ip]
    L.kba_track_destroy.argtypes = [vp]
    L.kba_destroy.argtypes = [vp]
    rng = np.random.default_rng(3)
    n, K, calls = args.compact_meas, 20, args.warmup + args.iters
    rows = [_push_rows(rng, n) for _ in range(K)]
    poses = [_pose(rng) for _ in range(K)]
    h = vp()
    assert L.kba_create(C.byref(h), 0) == 0
    out = {}
    # live keyframes hold K * n entries after a push: room for half a keyframe more compacts on every push
    for name, m_cap in (("compacting", K * n + n // 2), ("appending", n * (K + calls + 1))):
        t = vp()
        caps = KbaTrackCaps(K, N_LM, m_cap, 12, 3000, 40000, 0, 0)
        assert L.kba_track_create(h, C.byref(caps), 1, CAM_INTR.ctypes.data, CAM_POSE.ctypes.data, C.byref(t)) == 0

        def push(k):
            r = rows[k]
            assert L.kba_track_push_keyframe(t, k, poses[k].ctypes.data, None, n, r["lm_slot"].ctypes.data, None,
                                             r["u"].ctypes.data, r["v"].ctypes.data, r["d"].ctypes.data) == 0
        for k in range(K):
            push(k)
        ts = []
        for it in range(calls):
            k = it % K
            assert L.kba_track_drop_keyframe(t, k) == 0
            t0 = time.perf_counter()
            push(k)
            if it >= args.warmup:
                ts.append(time.perf_counter() - t0)
        L.kba_track_destroy(t)
        out[name] = _stats(ts)
    L.kba_destroy(h)
    print(json.dumps(out))


def bench_compaction(args):
    libs = [("this", os.path.join(ROOT, "limo_b200", "libkba_b200.so"))]
    if args.other_lib:
        libs.append(("other", os.path.abspath(args.other_lib)))
    out = {name: [] for name, _ in libs}
    for _ in range(args.rounds):
        for name, path in libs:
            env = dict(os.environ, KBA_LIB_PATH=path)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--compaction-worker", "--iters", str(args.iters),
                                "--warmup", str(args.warmup), "--compact-meas", str(args.compact_meas)], env=env, capture_output=True,
                               text=True, check=True)
            out[name].append(json.loads(r.stdout.strip().splitlines()[-1]))
    if not args.other_lib:
        out["other"] = "not measured (no --other-lib)"
    return out


def _sweep_step(dr, way, G, steps, warmup, capi, h, opts):
    tracks = [dr.make(h) for _ in range(G)]
    grp = capi.TrackGroup(h, [t for t, _ in tracks])
    t_step = 0.0
    for step in range(dr.steps):
        t0 = time.perf_counter()
        if step:
            frames = [dr.frame(m, step) for _, m in tracks]
            fr = grp.adjust_pose(frames, opts)
            if way == "group_only":
                k = dr.W - 1 + step
                slot = k % (dr.W + 1)
                if k >= dr.W + 1:
                    grp.drop_keyframes([slot] * G)
                reqs = []
                for (_, m), r in zip(tracks, fr):
                    m.poses[k] = r.kf_pose[0]
                    lm, u, v, d, cam = m.measurements(k)
                    reqs.append(dict(slot=slot, pose7=r.kf_pose[0], lm_slot=lm, u=u, v=v, d=d, cam=cam, plane4=PLANE))
                grp.push_keyframes(reqs)
            else:
                for i, (t, m) in enumerate(tracks):
                    dr.push(t, m, step, fr[i].kf_pose[0])
        res = grp.solve([m.request(step) for _, m in tracks], opts)
        if step >= warmup:
            t_step += time.perf_counter() - t0
        for (_, m), r in zip(tracks, res):
            m.record(r)
    poses = [r.kf_pose.copy() for r in res]
    grp.close()
    for t, _ in tracks:
        t.close()
    return G * steps / t_step, poses


def bench_sweep(args, capi, h):
    G = args.sweep_groups
    dr = sw.SweepDrive(W=12, steps=args.sweep_warmup + args.sweep_steps)
    opts = sw.options(sw.grid(G))
    out, poses = {}, {}
    for rnd in range(2):  # alternately
        for way in ("per_window_group", "group_only"):
            rate, poses[way] = _sweep_step(dr, way, G, args.sweep_steps, args.sweep_warmup, capi, h, opts)
            out.setdefault(way, []).append(round(rate, 1))
    same = all(np.array_equal(a, b) for a, b in zip(poses["per_window_group"], poses["group_only"]))
    return dict(groups=G, steps=args.sweep_steps, step_windows_per_s=out, final_poses_bit_identical=bool(same))


def profile_kernels(args, capi, h):
    """device time of the store kernels under torch.profiler: group pushes of 2500 rows on 132 tracks (every 8th call compacts),
    landmark and pose writes"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    rng = np.random.default_rng(11)
    G, n = 132, 2500
    pushes, lmw, kfw = _requests(rng, G, n)
    tracks = [capi.Track(h, CAM_INTR, CAM_POSE, max_keyframes=KF_SLOTS, max_landmarks=N_LM, max_measurements=n * (KF_SLOTS + 8),
                         win_keyframes=12, win_landmarks=3000, win_observations=40000) for _ in range(G)]
    grp = capi.TrackGroup(h, tracks)
    names = ("k_store_append", "k_arena_compact", "k_scatter_rows")
    calls = 40
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for it in range(calls):
            slot = it % KF_SLOTS
            if it >= KF_SLOTS:
                grp.drop_keyframes([slot] * G)
            grp.push_keyframes([dict(p, slot=slot) for p in pushes])
            grp.set_landmarks(lmw)
            grp.set_keyframe_poses(kfw)
        torch.cuda.synchronize()
    tot = {k: dict(calls=0, device_ms=0.0) for k in names}
    for e in prof.events():
        for k in names:
            if k in e.name and e.device_type.name == "CUDA":
                tot[k]["calls"] += 1
                tot[k]["device_ms"] += e.device_time / 1e3
    for k in names:
        c = tot[k]["calls"]
        tot[k]["mean_us_per_launch"] = round(1e3 * tot[k]["device_ms"] / c, 2) if c else None
        tot[k]["device_ms"] = round(tot[k]["device_ms"], 3)
    grp.close()
    for t in tracks:
        t.close()
    return dict(groups=G, push_rows=n, group_calls=calls, kernels=tot)


def dry_run(args):
    rng = np.random.default_rng(0)
    shapes = {}
    for G in args.groups:
        for n in args.push_meas:
            pushes, lmw, kfw = _requests(rng, G, n)
            shapes["G%d_n%d" % (G, n)] = dict(push_rows=sum(len(p["lm_slot"]) for p in pushes),
                                              landmark_rows=sum(len(r["lm_slot"]) for r in lmw),
                                              pose_rows=sum(len(r["kf_slots"]) for r in kfw))
    dr = sw.SweepDrive(W=12, steps=3)
    m = dr.base
    reqs = []
    for step in (1, 2):
        k = dr.W - 1 + step
        lm, u, v, d, cam = m.measurements(k)
        reqs.append(dict(slot=k % (dr.W + 1), n_meas=len(lm), cams=sorted(set(cam.tolist()))))
    return dict(dry_run=True, writes=shapes, sweep_pushes=reqs, frames=[len(dr.frame(m, s)["lm_slot"]) for s in (1, 2)])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--groups", type=int, nargs="+", default=[1, 32, 132])
    ap.add_argument("--push-meas", type=int, nargs="+", default=[300, 2500])
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--other-lib", default=None, help="another build of libkba_b200.so for the compaction timing")
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of the compaction timing")
    ap.add_argument("--compact-meas", type=int, default=2500)
    ap.add_argument("--sweep-groups", type=int, default=110)
    ap.add_argument("--sweep-steps", type=int, default=6)
    ap.add_argument("--sweep-warmup", type=int, default=2)
    ap.add_argument("--skip", nargs="*", default=[], choices=["writes", "compaction", "sweep", "profile"])
    ap.add_argument("--out", default=None)
    ap.add_argument("--dry-run", action="store_true")
    ap.add_argument("--compaction-worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.compaction_worker:
        return compaction_worker(args)
    if args.dry_run:
        out = dry_run(args)
    else:
        from limo_b200 import capi
        out = dict(card=_card())
        h = capi.Handle(0)
        if "writes" not in args.skip:
            out["writes"] = {"G%d_n%d" % (G, n): bench_writes(args, capi, h, G, n) for G in args.groups for n in args.push_meas}
        if "sweep" not in args.skip:
            out["sweep"] = bench_sweep(args, capi, h)
        h.close()
        if "compaction" not in args.skip:
            out["compaction"] = bench_compaction(args)
        if "profile" not in args.skip:
            h = capi.Handle(0)
            out["profile"] = profile_kernels(args, capi, h)
            h.close()
        out["card_after"] = _card()
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
