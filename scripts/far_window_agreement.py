"""How closely the CUDA path follows its references on windows far from the origin (tests/far_windows.py): per case and per
distance, the worst deviation of the first LM step from the dense extended-precision step, of the iteration log and the final
state from the oracle's, and of the FP32 solve from the FP64 one.  The tolerances of tests/test_far_windows.py come from this
table; the card's name and power limit are printed with it.  Needs an H100.

    python scripts/far_window_agreement.py [output file] [--workers N]
"""
import multiprocessing as mp
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

_handle = None


def _h():
    global _handle
    if _handle is None:
        from limo_b200 import capi
        _handle = capi.Handle(0)
    return _handle


def first_step(name, dist):
    from oracle import oracle as orc
    from tests import test_far_windows as tf
    from tests import test_first_step_dense as fs
    window, precision, copies, _ = fs.CUDA_CASES[name]
    win, opt, _ = tf.far_case(window, dist)
    opt.precision = precision
    h = _h()
    ref = fs.cuda_reference(h, orc, win, opt)
    worst = {}
    for res in h.solve_batch([win] * copies, opt, iterations_capacity=256):
        for k, v in fs._check_first_step(res, ref, 1.0, name).items():
            worst[k] = max(worst.get(k, 0.0), v)
    k = max(worst, key=worst.get)
    return "first step %-28s %5s  worst %.1e (%s)  step_norm %.1e  cost 1 %.1e  relative_decrease %.1e" % (
        name, dist, worst[k], k, worst["step_norm"], worst["cost 1"], worst["relative_decrease"])


def log(name, dist):
    from oracle import oracle as orc
    from tests import iter_log as il
    from tests import test_far_windows as tf
    m = tf.measure_log(_h(), orc, name, dist)
    out = "log %-24s %5s " % (name, dist)
    try:
        head = il.log_deviations(m.rg, m.rc, m.prefix, label=name, head=True)
        whole = il.log_deviations(m.rg, m.rc, m.prefix, label=name)
        out += " head " + " ".join("%s %.1e" % (f[:4], head[f][0]) for f in il.FIELDS)
        out += " | whole " + " ".join("%s %.1e" % (f[:4], whole[f][0]) for f in il.FIELDS)
    except AssertionError as e:
        out += " FLAGS DIFFER " + repr(e)[:300]
    out += " | decisions %s" % ("equal" if tf._decisions(m.rg) == tf._decisions(m.rc) else
                                "DIFFER %s %s" % (tf._decisions(m.rg), tf._decisions(m.rc)))
    dev = tf.final_deviation(m.rg, m.rc, m.win.n_lm)
    return out + " | final " + " ".join("%s %.1e" % kv for kv in dev.items())


def fp32(name, dist):
    from tests import test_far_windows as tf
    dev, n_lm = tf.measure_fp32(_h(), name, dist)
    return "fp32 %-24s %5s  " % (name, dist) + " ".join("%s %.1e" % kv for kv in dev.items()) + "  (of %d landmarks)" % n_lm


def fp32_log(dist):
    from oracle import oracle as orc
    from tests import iter_log as il
    from tests import test_far_windows as tf
    from tests import test_first_step_dense as fs
    win, opt, _ = tf.far_case("config2_slice", dist) if dist != "0" else fs.build("config2_slice") + (None,)
    rc = orc.solve_window(win, opt, iterations_capacity=1024)
    opt.precision = 1
    rg = _h().solve_window(win, opt, iterations_capacity=1024)
    try:
        w = il.log_deviations(rg, rc, solves=(0,), label="fp32")
        return "fp32 log config2_slice %5s  " % dist + " ".join("%s %.1e" % (f, w[f][0]) for f in il.FIELDS)
    except AssertionError as e:
        return "fp32 log config2_slice %5s  FLAGS DIFFER %s" % (dist, repr(e)[:300])


def _run(task):
    fn, args = task
    try:
        return globals()[fn](*args)
    except Exception as e:  # a case that fails is a row of the table, not the end of it
        return "%s %s FAILED %r" % (fn, args, e)


def main():
    args = sys.argv[1:]
    workers = 8
    if "--workers" in args:
        i = args.index("--workers")
        workers = int(args[i + 1])
        del args[i:i + 2]
    out = open(args[0], "w") if args else None
    from tests import far_windows as fw
    from tests import test_far_windows as tf
    from tests import test_first_step_dense as fs
    dists = list(fw.DISTANCES)
    tasks = [("fp32", (n, d)) for n in tf.FP32_CASES for d in ["0"] + dists] + [("fp32_log", (d,)) for d in ["0"] + dists]
    tasks += [("log", (n, d)) for n in tf.LOG_CASES for d in dists]
    tasks += [("first_step", (n, d)) for n in fs.CUDA_CASES for d in dists]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("GPU:", gpu, flush=True)
    if out:
        out.write("GPU: %s\n" % gpu)
    with mp.get_context("spawn").Pool(workers) as pool:
        for line in pool.imap(_run, tasks):
            print(line, flush=True)
            if out:
                out.write(line + "\n")
                out.flush()


if __name__ == "__main__":
    main()
