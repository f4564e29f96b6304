#!/usr/bin/env python
"""Solve time of large ground-plane windows, on each side of the 640-row panel bound: 60 keyframes (601 reduced rows, the
k_chol_trail factorisation), 64 (641), 100 (1001) and 128 (1281, the largest window) -- alone and as a resident batch of 8
copies.

   python scripts/large_window_bench.py [--solves 10] [--warmup 2]      one JSON line per (keyframes, batch)
   python scripts/large_window_bench.py --profile                       kernel breakdown of one solve per window, alone

Timing: a resident batch (kba_batch_create once), `--warmup` solves, then `--solves` solves each timed by a host clock around
kba_batch_solve (which returns when every window is done); median and p90.  The profile run traces one solve kernel by kernel
(KBA_GRAPH=0) with torch.profiler and reports the shares of the trailing update (k_chol_trail / k_chol_trail_band), stage 1
and stage 2 of k_reduced_solve (assembly; the two one-CTA triangular solves and the candidate state), the rest of the
factorisation (k_chol_diag, k_chol_panel), the Schur complement (k_schur_syrk, k_sred_reduce) and everything else.  Every line
carries the card's name and power limit, read in the same call."""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KEYFRAMES = (60, 64, 100, 128)


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    if q.returncode != 0 or not q.stdout.strip():
        return dict(gpu="unknown", power_limit_w=None)
    name, pl = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit_w=float(pl))


def windows(n_kf, n):
    """n copies of a ground-plane window of n_kf keyframes, 50 landmarks and 600 observations per keyframe (every window of a
    batch does the same work, so the batch time is that of n such windows)"""
    from limo_b200 import synth
    return [synth.make_window(3, seed=1000 + n_kf, n_kf=n_kf, n_lm=50 * n_kf, n_obs=600 * n_kf)] * n


def timing(args):
    import numpy as np
    from limo_b200 import capi
    h = capi.Handle(0)
    opt = capi.default_options()
    c = card()
    for n_kf in KEYFRAMES:
        for n in (1, 8):
            ws = windows(n_kf, n)
            batch = h.batch(ws)
            for _ in range(args.warmup):
                batch.solve(opt)
            ts = []
            for _ in range(args.solves):
                t0 = time.perf_counter()
                batch.solve(opt)
                ts.append(1e3 * (time.perf_counter() - t0))
            res = batch.download()
            assert all(r.c.status == 0 for r in res)
            print(json.dumps(dict(c, keyframes=n_kf, rows=10 * n_kf + 1, batch=n, solves=args.solves,
                                  median_ms=round(float(np.median(ts)), 3), p90_ms=round(float(np.percentile(ts, 90)), 3),
                                  iterations=sum(s.num_iterations for s in res[0].solves))), flush=True)
            batch.close()
    h.close()


GROUPS = (("trailing update", ("k_chol_trail", "k_chol_trail_band")), ("stage 1", ("k_reduced_solve/1",)),
          ("stage 2", ("k_reduced_solve/2",)), ("diag + panel", ("k_chol_diag", "k_chol_panel")),
          ("Schur", ("k_schur_syrk", "k_sred_reduce")))


def profile_run(args):
    os.environ["KBA_GRAPH"] = "0"
    import torch
    from torch.profiler import ProfilerActivity, profile
    from limo_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("large_window_bench.py: no CUDA device")
    torch.cuda.set_stream(torch.cuda.Stream())
    h = capi.Handle(0, stream=torch.cuda.current_stream().cuda_stream)
    opt = capi.default_options()
    c = card()
    for n_kf in KEYFRAMES:
        batch = h.batch(windows(n_kf, 1))
        for _ in range(args.warmup):
            batch.solve(opt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            batch.solve(opt)
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as td:
            path = os.path.join(td, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                events = json.load(f)["traceEvents"]
        kernels = sorted((ev for ev in events if ev.get("cat") == "kernel" and ev.get("ph") == "X"), key=lambda ev: ev["ts"])
        agg = collections.defaultdict(float)
        n_solve = 0
        for ev in kernels:
            name = re.sub(r"^void\s+", "", re.sub(r"[(<].*", "", ev["name"])).replace("kba::", "")
            if name == "k_reduced_solve":  # on the split factorisation each pass launches stage 1, then stage 2
                n_solve += 1
                name += "/1" if n_solve % 2 else "/2"
            agg[name] += float(ev["dur"])
        total = sum(agg.values())
        shares = {}
        for label, names in GROUPS:
            shares[label] = sum(agg.pop(k, 0.0) for k in names)
        shares["other"] = sum(agg.values())
        print(json.dumps(dict(c, keyframes=n_kf, rows=10 * n_kf + 1, kernel_ms=round(total / 1e3, 3),
                              share={k: round(v / total, 4) for k, v in shares.items()})), flush=True)
        batch.close()
    h.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--solves", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    (profile_run if args.profile else timing)(args)


if __name__ == "__main__":
    main()
