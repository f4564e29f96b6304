#!/usr/bin/env python
"""Per-kernel breakdown of the headline workload (resident batch of 264 config-2 windows): one full solve step traced with
torch.profiler (CUDA activities), after two warm-up steps.  Prints the card, its power limit and a markdown table of launches,
mean, sum and share of the traced kernel time per kernel.

   python scripts/kernel_breakdown.py [--batch N]      (KBA_LIB_PATH selects another build of the library)

The solve runs kernel by kernel on the stream (KBA_GRAPH=0 unless set) so that every launch is a trace record of its own; the
kernels and their device times are those of the graph path.  Run it on its own: tracing slows the host, not the kernels."""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("KBA_GRAPH", "0")


def kernel_name(raw):
    name = re.sub(r"\(.*", "", raw)                  # argument list
    name = re.sub(r"^void\s+", "", name)
    return name.replace("kba::", "")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=264)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from limo_b200 import capi, parallel
    if not torch.cuda.is_available():
        raise SystemExit("kernel_breakdown.py: no CUDA device")
    torch.cuda.set_stream(torch.cuda.Stream())
    stream = torch.cuda.current_stream()
    base = parallel.windows_for_rank(16, 0, 2)
    h = capi.Handle(0, stream=stream.cuda_stream)
    opt = capi.default_options()
    batch = h.batch([base[i % 16] for i in range(args.batch)])
    for _ in range(2):
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
    agg = collections.defaultdict(list)
    for ev in events:
        if ev.get("cat") == "kernel" and ev.get("ph") == "X":
            agg[kernel_name(ev["name"])].append(float(ev["dur"]))
    total = sum(sum(v) for v in agg.values())
    print("card: %s; lib: %s; batch %d, one solve step" % (card(), os.path.basename(capi.LIB_PATH), args.batch))
    print("| kernel | launches | mean us | sum ms | share |")
    print("|---|---|---|---|---|")
    for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
        print("| `%s` | %d | %.1f | %.2f | %.1f %% |" % (k, len(v), sum(v) / len(v), sum(v) / 1e3, 100.0 * sum(v) / total))
    print("| total | %d | | %.2f | |" % (sum(len(v) for v in agg.values()), total / 1e3))
    batch.close()
    h.close()


if __name__ == "__main__":
    main()
