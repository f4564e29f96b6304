"""Evaluation of the stored window (kba_track_evaluate / kba_track_group_evaluate) against what a caller can do without it:
kba_eval of the same window packed on the host, and a kba_track_solve of the same request.

Window: a 12-keyframe mono drive with lidar depth (tests/test_track_group.py::_Drive, 900 landmarks, 9000 observations), its
step-0 request.  Timed, each call ending in a synchronisation (the calls synchronise themselves), median and p90 over --iters
calls after --warmup:
  - evaluate: Track.evaluate (single), TrackGroup.evaluate at G = 1, 32 and 132 tracks of the same drive;
  - kba_eval: Handle.evaluate of the host-built window of the same request (the rebuild path's upload);
  - solve:    Track.solve of the same request on a clone (the store of the evaluated track does not change).
Bytes moved: kba_track_transfer_bytes / kba_track_group_transfer_bytes of the evaluation and of the solve.
A second run (--profile) records the device time of the evaluation kernels (k_ev_obs, k_ev_finish) and of the gather with
torch.profiler; the first run has the profiler off.  The card's name and power limit are read in the same command.

    python scripts/evaluate_bench.py --out /tmp/evaluate.json
    python scripts/evaluate_bench.py --profile --out /tmp/evaluate_prof.json
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

GROUPS = (1, 32, 132)


def _card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    text=True).splitlines()[0]
        name, pl, smax = [x.strip() for x in q.split(",")]
        return dict(gpu=name, power_limit=pl, sm_clock_max=smax)
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return dict(gpu="unknown (%s)" % e)


def _timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return dict(median_ms=float(np.median(ts)), p90_ms=float(np.percentile(ts, 90)))


def _host_window(dr, req):
    from limo_b200.capi_types import Window
    from tests.test_track import _window_lists
    first, last = 0, dr.W - 1
    lm_sel, ptr, okf, ou, ov, od = _window_lists(dr.per_kf, first, last)
    sc = {k: req[k] for k in ("scale_kf0", "scale_kf1", "scale_weight", "scale_value")}
    return Window(dr.win.kf_pose[first:last + 1], req["kf_fixed"], dr.cam_intr, dr.cam_pose, dr.win.lm_pos[lm_sel], dr.win.lm_weight[lm_sel],
                  ptr, okf, ou, ov, od, **sc)


def run(iters, warmup, profile):
    from limo_b200 import capi
    from tests.test_track_group import _Drive
    out = dict(card=_card(), iters=iters, warmup=warmup)
    h = capi.Handle(0)
    dr = _Drive(seed=501, W=12, n_lm=900, n_obs=9000)
    req = dr.request(0)
    t = dr.make_track(h)
    twin = t.clone()
    if profile:
        import torch
        from torch.profiler import ProfilerActivity, profile as tprofile
        t.evaluate(**req)
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                t.evaluate(**req)
        torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if e.key.startswith(("kba::k_ev_", "void kba::k_ev_", "kba::k_track_", "void kba::k_track_")):
                kern[e.key] = dict(calls=e.count, device_us_total=getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)))
        out["kernels"] = kern
    else:
        out["single"] = _timed(lambda: t.evaluate(**req), iters, warmup)
        up, down, _ = t.transfer_bytes()
        out["single"].update(h2d_bytes=up, d2h_bytes=down, n_obs=int(t.evaluate(**req)["n_obs"]))
        win = _host_window(dr, req)
        out["kba_eval"] = _timed(lambda: h.evaluate(win), iters, warmup)
        out["solve"] = _timed(lambda: twin.solve(**req), iters, warmup)
        up, down, _ = twin.transfer_bytes()
        out["solve"].update(h2d_bytes=up, d2h_bytes=down)
        for G in GROUPS:
            tracks = [t.clone() for _ in range(G)]
            grp = capi.TrackGroup(h, tracks)
            r = _timed(lambda: grp.evaluate([req] * G), iters, warmup)
            up, down = grp.transfer_bytes()
            r.update(h2d_bytes=up, d2h_bytes=down)
            out["group_%d" % G] = r
            grp.close()
            for x in tracks:
                x.close()
    twin.close(); t.close(); h.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="device time of the kernels under torch.profiler (a separate run)")
    ap.add_argument("--out", help="write the JSON record here as well")
    a = ap.parse_args()
    res = run(a.iters, a.warmup, a.profile)
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
