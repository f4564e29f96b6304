#!/usr/bin/env python
"""Sweep of the CTAs per window of k_linearize / k_backsub_v (KBA_LIN_GRID / KBA_BS_GRID are read when a batch is created) on the
headline workload, in one process: ms per step of a resident batch of 264 config-2 windows (--batch N: N windows), 5 steps after 2
warm-ups each.  Arguments: LIN,BS pairs (KBA_LIN_GRID, KBA_BS_GRID)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from limo_b200 import capi, parallel  # noqa: E402

torch.cuda.set_stream(torch.cuda.Stream())
stream = torch.cuda.current_stream()
args = sys.argv[1:]
n_win = 264
if "--batch" in args:
    k = args.index("--batch")
    n_win = int(args[k + 1])
    del args[k:k + 2]
base = parallel.windows_for_rank(16, 0, 2)
wins = [base[i % 16] for i in range(n_win)]
h = capi.Handle(0, stream=stream.cuda_stream)
opt = capi.default_options()
configs = [(-1, -1), (64, 63), (128, 63), (160, 63), (80, 63), (112, 63), (98, 32), (98, 94), (98, 126), (-1, -1)]
if args:
    configs = [tuple(int(x) for x in a.split(",")) for a in args]
for lin, bs in configs:
    os.environ["KBA_LIN_GRID"], os.environ["KBA_BS_GRID"] = str(lin), str(bs)
    batch = h.batch(wins)
    for _ in range(2):
        batch.solve(opt)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(5):
        batch.solve(opt)
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    print(json.dumps({"batch": n_win, "lin_grid": lin, "bs_grid": bs, "ms_per_step": round(ms, 2),
                      "windows_per_s": round(n_win / (ms * 1e-3), 1)}), flush=True)
    batch.close()
h.close()
