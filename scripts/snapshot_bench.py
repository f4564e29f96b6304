"""Snapshots of a track's store: save, load and clone against what a caller does without them, replaying the pushes and the
landmark writes into a fresh track.

Stores: the shapes of scripts/upkeep_bench.py and scripts/rank_bench.py (12 keyframes / 1.1k landmarks, 20 keyframes / 8k
landmarks) and a facade-sized one (20 keyframes, 131072 landmark slots).  Each keyframe is pushed with its measurements, and every
landmark slot is written once.  Timed, each call ending in a synchronisation (the calls synchronise themselves), median and p90
over --iters calls after --warmup:
  - save:   Track.snapshot (one download);
  - load:   Track.load on the same handle (track creation, one upload), the track closed outside the timing;
  - clone:  Track.clone on the same handle (creation, a store-to-store copy);
  - replay: a fresh track, the pushes and one set_landmarks call -- what rebuilds the same store today;
  - group save at G = 1, 32 and 132 tracks of the 12-keyframe store.
Bytes moved: the snapshot's size, and for the replay its upload (kba_track_transfer_bytes' push count).

    python scripts/snapshot_bench.py --out /tmp/snapshot.json
    python scripts/snapshot_bench.py --dry-run        # the stores' shapes and snapshot sizes on the CPU, no device
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

CAM_INTR = np.array([[700.0, 320.0, 240.0]])
CAM_POSE = np.array([[1.0, 0, 0, 0, 0, 0, 0]])
# name: (keyframes, landmarks measured, landmark slots, measurements per keyframe)
STORES = dict(kf12_lm1k=(12, 1100, 1100, 300), kf20_lm8k=(20, 8000, 8000, 2000), facade=(20, 8000, 131072, 2000))
GROUPS = (1, 32, 132)


def _card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    text=True).splitlines()[0]
        name, pl, smax = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=pl, sm_clock_max=smax)
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return dict(gpu="unknown (%s)" % e)


def _store(name, seed=0):
    """the pushes and the landmark values of a store: (caps, pushes, (slots, pos, weight))"""
    K, n_lm, slots, per_kf = STORES[name]
    rng = np.random.default_rng(seed)
    pushes = []
    for k in range(K):
        lm = np.sort(rng.choice(n_lm, per_kf, replace=False)).astype(np.int32)
        q = rng.normal(size=4)
        pushes.append(dict(slot=k, pose7=np.r_[q / np.linalg.norm(q), rng.normal(size=3)], lm_slot=lm,
                           u=rng.uniform(0, 640, per_kf).astype(np.float32), v=rng.uniform(0, 480, per_kf).astype(np.float32),
                           d=np.where(rng.uniform(size=per_kf) < 0.3, rng.uniform(2, 40, per_kf), -1.0).astype(np.float32)))
    lms = (np.arange(slots, dtype=np.int32), rng.normal(size=(slots, 3)) * 20, rng.uniform(0.5, 1, slots))
    caps = dict(max_keyframes=K + 1, max_landmarks=slots, max_measurements=2 * K * per_kf, win_keyframes=K, win_landmarks=n_lm,
                win_observations=K * per_kf)
    return caps, pushes, lms


def _replay(h, caps, pushes, lms):
    from limo_b200 import capi
    t = capi.Track(h, CAM_INTR, CAM_POSE, **caps)
    for p in pushes:
        t.push_keyframe(**p)
    t.set_landmarks(lms[0], pos=lms[1], weight=lms[2])
    return t


def _stats(ts):
    a = np.array(ts) * 1e3
    return dict(median_ms=round(float(np.median(a)), 4), p90_ms=round(float(np.percentile(a, 90)), 4))


def _time(fn, warmup, iters, after=None):
    out = []
    for i in range(warmup + iters):
        t0 = time.perf_counter()
        r = fn()
        dt = time.perf_counter() - t0
        if after:
            after(r)
        if i >= warmup:
            out.append(dt)
    return _stats(out)


def run(args):
    from limo_b200 import capi
    h = capi.Handle(0)
    res = dict(card=_card(), warmup=args.warmup, iters=args.iters, stores={}, group_save={})
    close = lambda t: t.close()  # noqa: E731
    for name in STORES:
        caps, pushes, lms = _store(name)
        src = _replay(h, caps, pushes, lms)
        snap = src.snapshot()
        _, _, push_bytes = src.transfer_bytes()
        assert capi.Track.load(h, snap).snapshot().tobytes() == snap.tobytes()
        res["stores"][name] = dict(snapshot_bytes=int(len(snap)), replay_upload_bytes=int(push_bytes),
                                   save=_time(src.snapshot, args.warmup, args.iters),
                                   load=_time(lambda: capi.Track.load(h, snap), args.warmup, args.iters, close),
                                   clone=_time(lambda: src.clone(), args.warmup, args.iters, close),
                                   replay=_time(lambda: _replay(h, caps, pushes, lms), args.warmup, args.iters, close))
        src.close()
    caps, pushes, lms = _store("kf12_lm1k")
    for G in GROUPS:
        ts = [_replay(h, caps, pushes, lms) for _ in range(G)]
        g = capi.TrackGroup(h, ts)
        g.snapshot()
        _, d2h = g.transfer_bytes()
        res["group_save"]["G%d" % G] = dict(bytes=int(d2h), group=_time(g.snapshot, args.warmup, args.iters),
                                            single_calls=_time(lambda: [t.snapshot() for t in ts], args.warmup, args.iters))
        g.close()
        for t in ts:
            t.close()
    h.close()
    return res


def dry_run(args):
    from limo_b200 import capi_types as T
    out = dict(dry_run=True, stores={})
    for name in STORES:
        caps, pushes, lms = _store(name)
        M = sum(len(p["lm_slot"]) for p in pushes)
        out["stores"][name] = dict(keyframes=len(pushes), entries=M, landmark_slots=len(lms[0]),
                                   snapshot_bytes=T._snapshot_layout(1, len(pushes), M, len(lms[0]))["end"])
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dry-run", action="store_true")
    args = ap.parse_args()
    res = dry_run(args) if args.dry_run else run(args)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
