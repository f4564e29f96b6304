"""How closely the CUDA path reproduces the oracle's iteration log: the worst deviation per log field on every window of
tests/test_iteration_log.py -- whole log, head of the log, and beside them the oracle against itself with its sums split over
another number of threads -- on the kernel variants and the FP32 linearisation mode, and the deviation of the first LM step
from the dense extended-precision step of tests/test_first_step_dense.py (oracle and CUDA path, every window there).  The
tolerances of tests/iter_log.py and tests/test_first_step_dense.py and the figures in DESIGN.md section 2 come from this table;
the card's name and power limit are printed with it.  Needs an H100.

    python scripts/iteration_log_agreement.py [output file] [--dense-only]
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from limo_b200 import capi
from oracle import oracle as orc
from tests import iter_log as il
from tests import test_first_step_dense as fs
from tests import test_iteration_log as tl

args = [a for a in sys.argv[1:] if a != "--dense-only"]
dense_only = "--dense-only" in sys.argv[1:]   # only the dense first step: the iteration logs take most of the run
out = open(args[0], "w") if args else None


def say(*a):
    line = " ".join(str(x) for x in a)
    print(line, flush=True)
    if out:
        out.write(line + "\n")
        out.flush()


def row(label, gpu, cpu, prefix, solves=None, head=False):
    try:
        worst = il.log_deviations(gpu, cpu, prefix_rule=prefix, solves=solves, label=label, head=head)
        say("%-36s records %3d / %3d  " % (label, gpu.c.num_iteration_records, cpu.c.num_iteration_records) +
            "  ".join("%s %.1e" % (f, worst[f][0]) for f in il.FIELDS))
    except AssertionError as e:
        say("%-36s MISMATCH %s" % (label, e))
    return gpu


say(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
h = capi.Handle(0)
for name in [] if dense_only else tl.CASES:
    win, opt, prefix, threads = tl.build_case(name)
    rc = orc.solve_window(win, opt, num_threads=threads, iterations_capacity=tl.LOG_CAPACITY)
    rg = row(name + (" (prefix rule)" if prefix else ""), h.solve_window(win, opt, iterations_capacity=tl.LOG_CAPACITY), rc, prefix)
    row("    head (solve 0, iterations 0..%d)" % il.HEAD_ITERATIONS, rg, rc, prefix, head=True)
    # the oracle against itself with its sums split over another number of threads: what re-association alone does to a log
    row("    oracle, %d threads against %d" % (threads + 3, threads),
        orc.solve_window(win, opt, num_threads=threads + 3, iterations_capacity=tl.LOG_CAPACITY), rc, prefix)
    for who, res in (("cuda", rg), ("oracle", rc)):
        try:
            il.check_log_invariants(res, opt, name)
        except AssertionError as e:
            say("    invariants (%s) FAIL %s" % (who, e))
for name in [] if dense_only else ("config2_slice", "config3_kf8"):
    win, opt, prefix, threads = tl.build_case(name)
    rc = orc.solve_window(win, opt, num_threads=threads, iterations_capacity=tl.LOG_CAPACITY)
    for variant in ("KBA_LINEARIZE", "KBA_FUSED"):
        os.environ[variant] = "0"
        row("%s %s=0" % (name, variant), h.solve_window(win, opt, iterations_capacity=tl.LOG_CAPACITY), rc, prefix)
        del os.environ[variant]
if not dense_only:
    win, opt, prefix, threads = tl.build_case("config2_full")
    rc = orc.solve_window(win, opt, num_threads=threads, iterations_capacity=tl.LOG_CAPACITY)
    opt.precision = 1
    row("config2_full precision=1, solve 0", h.solve_window(win, opt, iterations_capacity=tl.LOG_CAPACITY), rc, False, solves=(0,))


def dense_row(label, devs):
    """the worst deviation of each record field over `devs` (one dict per window of a batch)"""
    say("%-44s " % label + "  ".join("%s %.1e" % (k, max(d[k] for d in devs)) for k in devs[0]))


for name in fs.WINDOWS:   # the oracle against the dense step (needs no GPU; the CPU suite holds it)
    win, opt = fs.build(name)
    ref = fs.dense_first_step(win, opt, orc.evaluate(win, opt), lambda w: orc.evaluate(w, opt), orc)
    dense_row("dense step, oracle: %s (%s)" % (name, fs.WINDOWS[name][1]),
              [fs._check_first_step(orc.solve_window(win, opt), ref, float("inf"), name)])
for name in fs.CUDA_CASES:
    ref, results, tol = fs.cuda_first_step(h, orc, name)
    dense_row("dense step, cuda: %s (%s)" % (name, tol), [fs._check_first_step(r, ref, float("inf"), name) for r in results])
h.close()
