#!/usr/bin/env python
"""Sweep of the residual/Jacobian kernel's launch knobs on the bench workload (264 config-2 windows resident in HBM): the
kernel alone (kba_batch_jacobian_pass: every window active, 20 back-to-back launches between CUDA events), algorithmic
187 B/observation against the H100 SXM data sheet's 3.35 TB/s.  Knobs are read when a batch is created:
  KBA_EVAL_TILES_JAC  256-observation tiles a CTA walks      KBA_EVAL_MIN_BLOCKS  CTAs per SM (register cap)
  KBA_EVAL_CS         streaming (evict-first) stores
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from limo_b200 import capi, parallel  # noqa: E402

peak = 3350.0
base = parallel.windows_for_rank(16, 0, 2)
wins = [base[i % 16] for i in range(264)]
n_obs = sum(w.n_obs for w in wins)
h = capi.Handle(0)
print("| tiles | CTAs/SM | streaming stores | ms per launch | GB/s (187 B/obs) | of data-sheet peak |\n|---|---|---|---|---|---|")
for tiles, mb, cs in [(8, 2, 0), (8, 2, 1), (8, 3, 0), (8, 3, 1), (8, 4, 0), (8, 4, 1), (4, 2, 0), (4, 3, 1), (16, 2, 0), (16, 3, 1), (2, 3, 1), (2, 4, 1)]:
    os.environ.update(KBA_EVAL_TILES_JAC=str(tiles), KBA_EVAL_MIN_BLOCKS=str(mb), KBA_EVAL_CS=str(cs))
    b = h.batch(wins)
    b.jacobian_pass(repeats=5)
    ms = min(b.jacobian_pass(repeats=20) for _ in range(3)) / 20
    gbs = 187.0 * n_obs / (ms * 1e-3) / 1e9
    print("| %d | %d | %d | %.4f | %.0f | %.3f |" % (tiles, mb, cs, ms, gbs, gbs / peak), flush=True)
    b.close()
h.close()
