"""The solves bench.py times, at the batch sizes it times them, against the oracle and against single-window solves.

At bench.py's batch sizes the launch plan (limo_b200/csrc/kba_plan.h) puts each window's Schur sum on one CTA (p_split = 1):
264 config-2 windows (the headline), 1024 of them (the throughput sub-record) and 132 config-3 windows (FP64 and FP32).  That
runs code no smaller batch runs: k_sred_reduce is not launched, k_reduced_solve gathers A from the single sum itself (tiled, or
row-major in one CTA for config 3), one k_schur_fused CTA owns all of a window's landmark groups, and k_schur_syrk runs at a grid
depth of 1.  The timed loop also solves a resident batch several times without uploading it again, with kernel timing on (the
stream issue mode), packs on host threads, and runs several handles at once in its end-to-end leg.

So this file holds, on those shapes:
  - every record of the iteration log of config2_full (264 copies) and config3_full (132 copies) to the oracle's log;
  - the first LM step of the split factorisation (k_chol_*) at p_split = 1 to the dense step of tests/test_first_step_dense.py;
  - what bench.py itself returns from its timed loop: copies of a window bit-identical, each window bit-identical to a
    single-window solve with the same plan, four windows to the oracle;
  - config 2 at 64 (p_split = 3) and 1024 windows, config 3 at 132 windows in FP64 and FP32, and two steps in flight, each
    bit-identical to single-window solves with the same plan (or to the one-lane batch); the converging config-3 windows also
    to the oracle, and FP32 to FP64 at BASELINE.md section 3's tolerance.
A single-window solve pins the batch's Schur split and factorisation with KBA_P_SPLIT / KBA_SOLVE_SPLIT; the other choices that
follow the batch size (strided grids, issue mode) give bit-identical results (tests/test_gpu_parity.py and
tests/test_graph_modes.py), so the batch and the single solve must agree to the bit.  test_single_solves_run_the_batch_plan
checks that on the CPU.
"""
import json
import os
import subprocess
import sys
import threading
from types import SimpleNamespace

import numpy as np
import pytest

from limo_b200 import parallel
from tests import iter_log as il
from tests import test_first_step_dense as fs
from tests import test_iteration_log as tl
from tests.test_gpu_parity import COST_REL_TOL, TRANSLATION_TOL, _compare_solves
from tests.test_launch_plan import FIELDS, _query, driver  # noqa: F401  (the plan driver fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADLINE_BATCH, HEADLINE_DISTINCT = 264, 16       # bench.py's --batch and --distinct defaults
CONFIG3_BATCH, CONFIG3_DISTINCT = 132, 8          # bench.py sub_config3
IN_FLIGHT_STEPS = 3
# The config-3 windows held to the oracle: those whose trimmed solve converges.  Windows 0 and 3 stop at the 100-iteration cap
# with their last iterations at radii above 1e12, where whether a step is valid is decided by rounding (iter_log's prefix
# rule), so the count of accepted steps differs between two oracle runs (8 and 11 threads: 65 and 66 on window 3; the oracle
# deals landmarks to threads dynamically, so even two runs with 8 threads gave 69 and 70 on window 0).  Window 6's plane
# blocks are flat enough that two oracle runs differ by 2e-5 in cost within the prefix.
CONFIG3_ORACLE_WINDOWS = (1, 2, 4, 5, 7)


@pytest.fixture(scope="module")
def config2_windows():
    """the distinct windows of bench.py's headline batch"""
    return parallel.windows_for_rank(HEADLINE_DISTINCT, 0, 2)


@pytest.fixture(scope="module")
def config3_windows():
    """the distinct windows of bench.py's config-3 sub-record"""
    return parallel.windows_for_rank(CONFIG3_DISTINCT, 0, 3)


def tiled(windows, n):
    """a batch of n windows cycling through `windows`, as bench.py builds it"""
    return [windows[i % len(windows)] for i in range(n)]


def plan(driver, windows, p_split=0, solve_split=-1):  # noqa: F811
    """the launch plan of kba_solve_batch on `windows` (an H100's SMs), with KBA_P_SPLIT / KBA_SOLVE_SPLIT as given"""
    q = _query("plan", [fs.plan_shape(w) for w in windows], "batch", 1, p_split, 1, solve_split)
    return dict(zip(FIELDS, map(int, driver(q)[0].split())))


def test_single_solves_run_the_batch_plan(driver, config2_windows, config3_windows):  # noqa: F811
    """the batch shapes of this file take the plan named in each test, and a single window with the knobs pinned as the tests
    pin them takes the same plan, field for field"""
    c2 = plan(driver, tiled(config2_windows, HEADLINE_BATCH))
    assert {k: c2[k] for k in ("fused", "fused_slots", "p_split", "solve_tiled", "device_pack")} == dict(
        fused=1, fused_slots=6, p_split=1, solve_tiled=1, device_pack=1)
    assert plan(driver, tiled(config2_windows, 1024)) == c2
    assert plan(driver, config2_windows[:1], p_split=1) == c2
    c2_64 = plan(driver, tiled(config2_windows, 64))
    assert c2_64["p_split"] == 3 and plan(driver, config2_windows[:1], p_split=3) == c2_64
    c3 = plan(driver, tiled(config3_windows, CONFIG3_BATCH))
    assert {k: c3[k] for k in ("fused", "p_split", "solve_tiled", "solve_split", "device_pack")} == dict(
        fused=0, p_split=1, solve_tiled=0, solve_split=0, device_pack=0)
    assert plan(driver, config3_windows[:1], p_split=1, solve_split=0) == c3
    for name, copies in (("config2_full", HEADLINE_BATCH), ("config3_full", CONFIG3_BATCH)):
        assert plan(driver, [tl.build_case(name)[0]] * copies)["p_split"] == 1, name
    split = plan(driver, [fs.build("config3_kf30_lm600")[0]], p_split=1)
    assert (split["p_split"], split["solve_tiled"], split["solve_split"]) == (1, 0, 32)


# ---- GPU ------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


SOLVE_FIELDS = ("initial_cost", "final_cost", "num_iterations", "num_successful_steps", "termination", "num_landmarks",
                "num_residual_blocks")


def state(res, win):
    """what a caller receives for one window, copied out of the result buffers (which a later download overwrites)"""
    return dict(kf_pose=res.kf_pose.copy(), kf_plane=res.kf_plane.copy(), lm_pos=res.lm_pos[:win.n_lm].copy(),
                lm_rejected=res.lm_rejected[:win.n_lm].copy(), initial_cost=res.c.initial_cost, final_cost=res.c.final_cost,
                status=res.c.status, lm_iterations=sum(s.num_iterations for s in res.solves),
                solves=[tuple(getattr(s, f) for f in SOLVE_FIELDS) for s in res.solves])


def as_result(s):
    """a state in the shape tests/test_gpu_parity.py::_compare_solves reads"""
    solves = [SimpleNamespace(**dict(zip(SOLVE_FIELDS, t))) for t in s["solves"]]
    return SimpleNamespace(c=SimpleNamespace(status=s["status"], num_solves=len(solves)), solves=solves,
                           kf_pose=s["kf_pose"], lm_pos=s["lm_pos"], lm_rejected=s["lm_rejected"])


def same(a, b, label):
    """bit-identical in every field both states carry"""
    keys = set(a) & set(b)
    assert {"kf_pose", "lm_pos", "lm_rejected", "final_cost", "lm_iterations"} <= keys, label
    for k in sorted(keys):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (label, k)


def resident(handle, windows, opt, solves=2):
    """bench.py's timed loop: a batch created (packed and uploaded) once, solved `solves` times, then downloaded"""
    b = handle.batch(windows)
    try:
        for _ in range(solves):
            b.solve(opt)
        return [state(r, w) for r, w in zip(b.download(), windows)]
    finally:
        b.close()


def singles(handle, windows, opt, **knobs):
    """each window solved alone, with the plan knobs pinned (read when the solve creates its batch)"""
    with pytest.MonkeyPatch.context() as mp:
        for k, v in knobs.items():
            mp.setenv(k, v)
        return [state(handle.solve_window(w, opt), w) for w in windows]


def options(precision=0):
    from limo_b200 import capi
    opt = capi.default_options()
    opt.precision = precision
    return opt


@pytest.fixture(scope="module")
def config2_singles(handle, config2_windows):
    """the distinct config-2 windows solved alone at p_split = 1, the headline batch's plan"""
    return singles(handle, config2_windows, options(), KBA_P_SPLIT="1")


@pytest.fixture(scope="module")
def config2_batch264(handle, config2_windows):
    """the headline batch solved through one handle"""
    return resident(handle, tiled(config2_windows, HEADLINE_BATCH), options())


@pytest.mark.gpu
@pytest.mark.parametrize("name, copies", [("config2_full", HEADLINE_BATCH), ("config3_full", CONFIG3_BATCH)])
def test_every_iteration_at_one_cta_per_window(handle, oracle, driver, name, copies):  # noqa: F811
    """every record of every window's log against the oracle's log of that window, at the tolerances and under the rules of
    tests/test_iteration_log.py::test_iteration_log_matches_oracle, with the Schur sum of each window on one CTA"""
    win, opt, prefix, threads = tl.build_case(name)
    assert plan(driver, [win] * copies)["p_split"] == 1
    rc = oracle.solve_window(win, opt, num_threads=threads, iterations_capacity=tl.LOG_CAPACITY)
    il.check_log_invariants(rc, opt, name + " (oracle)")
    results = handle.solve_batch([win] * copies, opt, iterations_capacity=tl.LOG_CAPACITY)
    il.check_log_invariants(results[-1], opt, "%s, window %d" % (name, copies - 1))
    for i, rg in enumerate(results):
        label = "%s, window %d" % (name, i)
        assert rg.c.status == 0, label
        assert [s.termination for s in rg.solves] == [s.termination for s in rc.solves], label
        il.compare_logs(rg, rc, il.TOL["fp64_head"], prefix_rule=prefix, label=label, head=True)
        il.compare_logs(rg, rc, il.TOL["fp64"], prefix_rule=prefix, label=label)


@pytest.mark.gpu
@pytest.mark.skipif(np.finfo(fs.LD).eps >= np.finfo(np.float64).eps, reason="numpy.longdouble is not an extended type here")
def test_split_factorisation_first_step_at_one_cta_schur_sum(handle, oracle, driver, monkeypatch):  # noqa: F811
    """config3_kf30_lm600 alone with KBA_P_SPLIT=1: k_reduced_solve gathers A from the single Schur sum, then k_chol_* factorise
    it over 32 CTAs -- records 0 and 1 against the dense extended-precision step"""
    win, opt = fs.build("config3_kf30_lm600")
    got = plan(driver, [win], p_split=1)
    assert (got["p_split"], got["solve_tiled"], got["solve_split"]) == (1, 0, 32)
    ref = fs.dense_first_step(win, opt, handle.evaluate(win, opt), lambda w: handle.evaluate(w, opt), oracle)
    monkeypatch.setenv("KBA_P_SPLIT", "1")
    res = handle.solve_window(win, opt)
    assert res.c.status == 0
    fs._check_first_step(res, ref, fs.TOL[fs.WINDOWS["config3_kf30_lm600"][1]], "config3_kf30_lm600, KBA_P_SPLIT=1")


def dump_states(out_dir, windows):
    """bench.py --dump-outputs split back into one state per window (every window of the batch was written)"""
    d = {f[:-4]: np.load(os.path.join(out_dir, f)) for f in os.listdir(out_dir) if f.endswith(".npy")}
    assert np.array_equal(d["window_index"], np.arange(len(windows)))
    kf = np.concatenate([[0], np.cumsum([w.n_kf for w in windows])])
    lm = np.concatenate([[0], np.cumsum([w.n_lm for w in windows])])
    assert d["kf_pose"].shape == (kf[-1], 7) and d["lm_pos"].shape == (lm[-1], 3)
    return [dict(kf_pose=d["kf_pose"][kf[i]:kf[i + 1]], kf_plane=d["kf_plane"][kf[i]:kf[i + 1]],
                 lm_pos=d["lm_pos"][lm[i]:lm[i + 1]], lm_rejected=d["lm_rejected"][lm[i]:lm[i + 1]].astype(np.uint8), initial_cost=d["initial_cost"][i],
                 final_cost=d["final_cost"][i], status=int(d["status"][i]), lm_iterations=int(d["lm_iterations"][i]))
            for i in range(len(windows))]


def hold_to_oracle(s, rc, win, label):
    """tests/test_gpu_parity.py::_compare_solves on what a dumped window carries: status, total LM iterations, initial and
    final cost, rejections, poses and landmarks"""
    assert s["status"] == 0, label
    assert s["lm_iterations"] == sum(x.num_iterations for x in rc.solves), label
    assert s["initial_cost"] == pytest.approx(rc.c.initial_cost, rel=COST_REL_TOL), label
    assert s["final_cost"] == pytest.approx(rc.c.final_cost, rel=COST_REL_TOL, abs=1e-14), label
    assert np.array_equal(s["lm_rejected"], rc.lm_rejected[:win.n_lm]), label
    assert np.linalg.norm(s["kf_pose"][:, 4:] - rc.kf_pose[:, 4:], axis=1).max() <= TRANSLATION_TOL, label
    assert np.abs(s["kf_pose"][:, :4] - rc.kf_pose[:, :4]).max() <= 1e-7, label
    dl = np.linalg.norm(s["lm_pos"] - rc.lm_pos[:win.n_lm], axis=1)
    assert np.percentile(dl, 95) <= 1e-6 and (dl > 0.1).sum() == 0, (label, np.percentile(dl, 95), dl.max())


@pytest.mark.gpu
def test_bench_timed_path(tmp_path, oracle, config2_windows, config2_singles):
    """bench.py's own timed loop (default batch and distinct windows, kernel timing on, resident batch solved three times):
    what it returns for every window of the batch"""
    out = tmp_path / "dump"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "2", "--warmup", "1", "--no-sub",
                        "--cpu-sample", "0", "--in-flight", "1", "--dump-outputs", str(out)],
                       cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    assert (d["config"]["batch_windows_per_gpu"], d["config"]["distinct_windows_per_gpu"]) == (HEADLINE_BATCH, HEADLINE_DISTINCT)
    windows = tiled(config2_windows, HEADLINE_BATCH)
    got = dump_states(str(out), windows)
    for i, s in enumerate(got):
        j = i % HEADLINE_DISTINCT
        same(s, got[j], "window %d against window %d of the batch" % (i, j))
        same(s, config2_singles[j], "window %d against its single solve" % i)
    for j in range(0, HEADLINE_DISTINCT, 4):
        hold_to_oracle(got[j], oracle.solve_window(config2_windows[j], num_threads=8), config2_windows[j], "window %d" % j)


@pytest.mark.gpu
def test_config2_at_64_windows(handle, driver, config2_windows):  # noqa: F811
    """bench.py's 64-window config-2 sub-record: three CTAs per window's Schur sum, k_sred_reduce folds them"""
    windows = tiled(config2_windows, 64)
    assert plan(driver, windows)["p_split"] == 3
    want = singles(handle, config2_windows, options(), KBA_P_SPLIT="3")
    for i, s in enumerate(resident(handle, windows, options())):
        same(s, want[i % HEADLINE_DISTINCT], "window %d" % i)


@pytest.mark.gpu
def test_config2_at_1024_windows(handle, config2_windows, config2_singles, config2_batch264):
    """bench.py's 1024-window config-2 sub-record (about 7 GB resident): every window as in the headline batch"""
    for i, s in enumerate(config2_batch264):
        same(s, config2_singles[i % HEADLINE_DISTINCT], "headline batch, window %d" % i)
    for i, s in enumerate(resident(handle, tiled(config2_windows, 1024), options())):
        same(s, config2_batch264[i % HEADLINE_DISTINCT], "window %d" % i)


@pytest.mark.gpu
def test_config3_at_132_windows(handle, oracle, monkeypatch, config3_windows):
    """bench.py's config-3 sub-record, packed on host threads: the row-major factorisation in one CTA with A gathered by
    k_reduced_solve, in FP64 and FP32; FP64 against the oracle, FP32 against FP64 at BASELINE.md section 3's tolerance"""
    monkeypatch.setenv("KBA_HOST_THREADS", "8")
    windows = tiled(config3_windows, CONFIG3_BATCH)
    got = {}
    for precision in (0, 1):
        got[precision] = resident(handle, windows, options(precision))
        want = singles(handle, config3_windows, options(precision), KBA_P_SPLIT="1", KBA_SOLVE_SPLIT="0")
        for i, s in enumerate(got[precision]):
            j = i % CONFIG3_DISTINCT
            same(s, got[precision][j], "precision %d, window %d against window %d of the batch" % (precision, i, j))
            same(s, want[j], "precision %d, window %d against its single solve" % (precision, i))
    # tests/test_gpu_parity.py::test_config3_ground_plane_matches_oracle's tolerances, on the windows whose solves converge
    for j in CONFIG3_ORACLE_WINDOWS:
        win, s = config3_windows[j], got[0][j]
        rc = oracle.solve_window(win, num_threads=8)
        _compare_solves(as_result(s), rc, win, "config3, window %d" % j, iter_slack=3)
        assert np.abs(s["kf_plane"] - rc.kf_plane).max() <= 1e-3, j
        assert np.allclose(np.linalg.norm(s["kf_plane"][:, :3], axis=1), 1.0, atol=1e-12), j
    for j, (a, b) in enumerate(zip(got[0][:CONFIG3_DISTINCT], got[1][:CONFIG3_DISTINCT])):
        assert a["status"] == b["status"] == 0
        assert np.linalg.norm(a["kf_pose"][:, 4:] - b["kf_pose"][:, 4:], axis=1).max() <= 1e-2, j
        if np.array_equal(a["lm_rejected"], b["lm_rejected"]):
            assert abs(a["final_cost"] - b["final_cost"]) <= 1e-5 * a["final_cost"], j


@pytest.mark.gpu
def test_steps_in_flight(monkeypatch, config2_windows, config2_batch264):
    """bench.py's end-to-end leg: two handles on their own streams, blocking-sync waits, two host threads each running upload,
    solve and download of the headline batch at the same time -- every step of every lane as the one-lane batch"""
    import torch
    from limo_b200 import capi
    monkeypatch.setenv("KBA_BLOCKING_SYNC", "1")   # read at kba_create
    windows = tiled(config2_windows, HEADLINE_BATCH)
    opt = options()
    lanes, got, errors = [], [[], []], []
    try:
        for _ in range(2):
            st = torch.cuda.Stream()
            h = capi.Handle(0, stream=st.cuda_stream)
            lanes.append((st, h, h.batch(windows)))

        def lane(i):
            try:
                torch.cuda.set_device(0)
                b, res = lanes[i][2], None
                for _ in range(IN_FLIGHT_STEPS):
                    b.upload()
                    b.solve(opt)
                    res = b.download(results=res)
                    got[i].append([state(r, w) for r, w in zip(res, windows)])
            except Exception as e:  # noqa: BLE001  (reported below, on the test's thread)
                errors.append(e)

        threads = [threading.Thread(target=lane, args=(i,)) for i in range(2)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        for _, h, b in lanes:
            b.close()
            h.close()
    assert not errors, errors
    for i, steps in enumerate(got):
        assert len(steps) == IN_FLIGHT_STEPS
        for k, states in enumerate(steps):
            for j, (s, want) in enumerate(zip(states, config2_batch264)):
                same(s, want, "lane %d, step %d, window %d" % (i, k, j))
