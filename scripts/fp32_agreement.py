"""How closely the FP32 mode (kba_options.precision = 1) follows its references, at the origin and far from it: the first LM
step of every FP32 case of tests/test_first_step_dense.CUDA_CASES (and of the 651-row ground window) against the mixed system
the FP32 solve forms and against the system of the FP32 blocks alone, what one perturbed FP32 block does to the mixed reference,
and the FP32 blocks against the FP64 ones per column family (tests/test_far_windows.fp32_block_deviation).  The tolerances of
those tests come from this table; the card's name and power limit are printed with it.  Needs an H100.

    python scripts/fp32_agreement.py [output file] [--workers N] [--blocks]

--blocks prints the block rows only (they take seconds; KBA_LIB_PATH selects the library they measure).
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


def _window(name, dist):
    from tests import test_far_windows as tf
    from tests import test_first_step_dense as fs
    if name == "ground_651":
        from oracle import oracle as orc
        from tests import test_large_reduced_rows as lr
        return lr._ground_651(), orc.default_options()
    return fs.build(name) if dist == "0" else tf.far_case(name, dist)[:2]


def _worst(results, ref):
    from tests import test_first_step_dense as fs
    worst = {}
    for res in results:
        assert res.c.status == 0
        for k, v in fs._check_first_step(res, ref, 1.0, "").items():
            worst[k] = max(worst.get(k, 0.0), v)
    k = max(worst, key=worst.get)
    return "%.1e (%s)" % (worst[k], k)


def first_step(name, dist):
    from oracle import oracle as orc
    from tests import test_first_step_dense as fs
    window, precision, copies = fs.CUDA_CASES[name][:3] if name in fs.CUDA_CASES else (name, 1, 1)
    win, opt = _window(window, dist)
    opt.precision = precision
    h = _h()
    results = h.solve_batch([win] * copies, opt, iterations_capacity=256)
    mixed = fs.cuda_reference(h, orc, win, opt)
    one = fs.cuda_reference(h, orc, win, opt, fp32_pose_rows=True)
    return "first step %-34s %5s  mixed system %s  | FP32 blocks alone %s" % (name, dist, _worst(results, mixed),
                                                                             _worst(results, one))


def perturbed(name):
    from oracle import oracle as orc
    from tests import test_first_step_dense as fs
    win, opt = fs.build(name)
    h = _h()
    b64 = h.evaluate(win, opt)
    opt.precision = 1
    b32 = h.evaluate(win, opt)
    [res] = h.solve_batch([win], opt, iterations_capacity=256)
    out = "perturbed %-20s" % name
    for what in ("jl", "r"):
        ref = fs.dense_first_step(win, opt, fs.tampered(b32, what), lambda w: h.evaluate(w, opt), orc, fp64_blocks=b64)
        out += "  one %s row x (1 + 1e-6): %s" % (what, _worst([res], ref))
    return out


def blocks(name, dist):
    from tests import test_far_windows as tf
    win, opt = _window(name, dist)
    h = _h()
    b64 = h.evaluate(win, opt)
    opt.precision = 1
    b32 = h.evaluate(win, opt)
    dev = tf.fp32_block_deviation(win, b32, b64)
    return "blocks %-20s %5s  " % (name, dist) + " ".join("%s %.1e" % kv for kv in dev.items())


def mixed_self_check(name):
    from oracle import oracle as orc
    from tests import test_first_step_dense as fs
    win, opt = fs.build(name)
    b = orc.evaluate(win, opt)
    ev = lambda w: orc.evaluate(w, opt)  # noqa: E731
    mixed = fs.dense_first_step(win, opt, b, ev, orc, fp64_blocks=b)
    out = "mixed self-check %-20s (CPU)  row form %.1e" % (name, fs.record_deviation(mixed, fs.dense_first_step(win, opt, b, ev, orc)))
    for what in ("jl", "r"):
        out += "  one %s row x (1 + 1e-6): %.1e" % (
            what, fs.record_deviation(fs.dense_first_step(win, opt, fs.tampered(b, what), ev, orc, fp64_blocks=b), mixed))
    return out


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
    only_blocks = "--blocks" in args
    args = [a for a in args if a != "--blocks"]
    out = open(args[0], "w") if args else None
    from tests import far_windows as fw
    from tests import test_first_step_dense as fs
    dists = ["0"] + list(fw.DISTANCES)
    tasks = [("blocks", (n, d)) for n in ("config2_slice", "config3_kf30_lm600") for d in dists]
    if not only_blocks:
        tasks += [("perturbed", (n,)) for n in ("config2_slice", "config3_kf30_lm600")]
        tasks += [("first_step", ("ground_651", "0"))]
        tasks += [("first_step", (n, d)) for n in fs.CUDA_CASES if fs.CUDA_CASES[n][1] == 1 for d in dists]
        tasks += [("mixed_self_check", (n,)) for n in ("config2_slice", "free_kf30_none_fixed", "config3_kf30_lm600",
                                                      "config5_kf40_lm700")]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print("GPU:", gpu, "library:", os.environ.get("KBA_LIB_PATH", "limo_b200/libkba_b200.so"), flush=True)
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
