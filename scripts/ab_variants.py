#!/usr/bin/env python
"""A/B of library builds on the headline workload (resident batch of 264 config-2 windows):
   python scripts/ab_variants.py lib1.so[:KBA_GRAPH[:NAME=VALUE,...]] lib2.so ...  -- each in its own process (the library and its
   switches are read once), two repetitions of 5 steps; prints a digest of the results (equal digests = bit-identical solves)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if len(sys.argv) > 1 and sys.argv[1] == "--child":
    sys.path.insert(0, ROOT)
    import torch
    from limo_b200 import capi, parallel
    torch.cuda.set_stream(torch.cuda.Stream())
    stream = torch.cuda.current_stream()
    base = parallel.windows_for_rank(16, 0, 2)
    h = capi.Handle(0, stream=stream.cuda_stream)
    opt = capi.default_options()
    batch = h.batch([base[i % 16] for i in range(264)])
    out = []
    for rep in range(2):
        for _ in range(3 if rep == 0 else 1):
            batch.solve(opt)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(5):
            batch.solve(opt)
        e1.record(stream)
        torch.cuda.synchronize()
        out.append(round(e0.elapsed_time(e1) / 5, 2))
    import hashlib
    res = batch.download()
    digest = hashlib.sha1(b"".join(r.kf_pose.tobytes() + r.lm_pos.tobytes() for r in res[:16])).hexdigest()[:12]
    print(json.dumps({"lib": os.path.basename(os.environ.get("KBA_LIB_PATH", "default")),
                      "env": {k: v for k, v in os.environ.items() if k.startswith("KBA_") and k != "KBA_LIB_PATH"},
                      "ms_per_step": out, "windows_per_s": round(264 / (min(out) * 1e-3), 1),
                      "results_sha1": digest, "cost0": res[0].c.final_cost, "done": all(r.c.status == 0 for r in res)}))
    sys.exit(0)

# spec: lib.so[:GRAPHMODE][:NAME=VALUE,NAME=VALUE...]
for spec in sys.argv[1:]:
    parts = spec.split(":")
    lib, g = parts[0], (parts[1] if len(parts) > 1 and parts[1] else "0")
    env = dict(os.environ, KBA_LIB_PATH=os.path.join(ROOT, lib), KBA_GRAPH=g)
    if len(parts) > 2:
        env.update(kv.split("=") for kv in parts[2].split(","))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=300)
    print(r.stdout.strip() or ("FAILED " + spec + " " + r.stderr[-300:]))
    sys.stdout.flush()
