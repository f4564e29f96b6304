#!/usr/bin/env python
"""SASS opcode histogram of the shipped library (the evidence for which hardware paths the kernels use): per kernel the counts of
the FP64 tensor-core (DMMA), bulk / async copy (UBLKCP, LDGSTS), mbarrier (SYNCS), 128-bit global / shared access opcodes.
usage: scripts/sass_histogram.py [limo_b200/libkba_b200.so]"""
import collections
import re
import subprocess
import sys

so = sys.argv[1] if len(sys.argv) > 1 else "limo_b200/libkba_b200.so"
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
COLS = [("DMMA", r"^DMMA"), ("UBLKCP (cp.async.bulk)", r"^UBLKCP"), ("LDGSTS (cp.async)", r"^LDGSTS"), ("SYNCS (mbarrier)", r"^SYNCS"),
        ("USETMAXREG", r"^USETMAXREG"), ("LDG.E.128", r"^LDG.*\.128"), ("LDG.E.64", r"^LDG.*\.64"), ("STG.E.128", r"^STG.*\.128"),
        ("STG.E.64", r"^STG.*\.64"), ("LDS.128", r"^LDS.*\.128"), ("STS.128", r"^STS.*\.128"), ("DFMA+DMUL+DADD", r"^(DFMA|DMUL|DADD)"),
        ("MUFU", r"^MUFU"), ("SHFL", r"^SHFL"), ("spills (STL/LDL)", r"^(STL|LDL)")]
kern = collections.OrderedDict()
name = None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = re.sub(r"^_ZN3kba\d*", "", m.group(1))
        kern[name] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
    if m and name:
        op = m.group(1)
        kern[name]["n"] += 1
        for label, pat in COLS:
            if re.match(pat, op):
                kern[name][label] += 1
print("# SASS opcode histogram of `%s` (`cuobjdump -sass`, sm_90a)\n" % so)
print("| kernel | instructions | " + " | ".join(c for c, _ in COLS) + " |")
print("|---|---|" + "---|" * len(COLS))
for k in sorted(kern):
    c = kern[k]
    print("| %s | %d | " % (k[:70], c["n"]) + " | ".join(str(c[l]) for l, _ in COLS) + " |")
