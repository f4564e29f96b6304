"""The per-iteration log of a window solve, CUDA path against CPU oracle, record by record.

The other solver tests compare the END of a solve, and a converged Levenberg-Marquardt solve forgives a lot: a Jacobian, Schur
complement, Cholesky or back-substitution kernel that is wrong at the 1e-6 level lands in the same minimum, usually after the
same number of iterations.  Step norm, model decrease (through relative_decrease) and candidate cost of every iteration are
direct functions of the whole pass chain (k_linearize / k_eval_obs, k_pose_hessian, the Schur kernel, k_reduced_solve or
k_chol_*, k_backsub*, k_lm_update), so holding every record of kba_result.iterations to the oracle's is a per-step check of
that chain -- on windows that between them select every solver path a window shape can select.
"""
import pytest

from limo_b200 import synth
from tests import edge_windows as ew
from tests import iter_log as il

LOG_CAPACITY = 1024   # three inner solves of up to 100 iterations do not fit the bindings' default of 256


def _motion_only(with_prior):
    from tests.test_gpu_parity import _motion_only_window
    return _motion_only_window(31, with_prior)[0]


def _motion_options(opt):
    opt.min_landmarks_for_trimming = 30


def _shapes(name):
    from tests import test_schur_fused_shapes as sf
    return getattr(sf, name)()


# name -> (window builder, prefix rule, oracle threads, options hook); what each window pins is in the comment behind it
CASES = {
    "config1": (lambda: synth.make_window(1), False, 1, None),                            # fused Schur kernel, small
    "config1_seed11": (lambda: synth.make_window(1, seed=11), False, 1, None),
    "config2_full": (lambda: synth.make_window(2), False, 8, None),                       # fused six-slot, the bench workload
    # 187 rows over all 31 keyframes: the large-window path (k_schur_syrk, tiled k_reduced_solve at 192 rows), not the seven-slot
    # kernel its 30 free keyframes would select on the fused path
    "free_keyframes_30": (lambda: synth.make_window(2, n_kf=31, n_lm=700, n_obs=7000, seed=5), False, 1, None),
    "gap_over_fixed_keyframe": (lambda: _shapes("_gap_over_fixed_keyframe"), False, 1, None),   # per-observation copies
    "stereo_rig": (lambda: _shapes("_stereo_rig"), False, 1, None),                       # rank > 0: synchronous producer
    "ragged": (ew.CASES["ragged"], False, 1, None),                                       # empty CSR rows
    "short_tracks": (lambda: synth.make_window(2, n_kf=10, n_lm=1500, n_obs=3000, seed=9), False, 1, None),  # 16 landmarks / tile
    "config3_kf8": (lambda: synth.make_window(3, seed=41, n_kf=8, n_lm=300, n_obs=1800, gp_frac=0.2), True, 1, None),
    "config3_kf14": (lambda: synth.make_window(3, seed=41, n_kf=14, n_lm=500, n_obs=4500), True, 1, None),  # fused + plane blocks
    "config3_full": (lambda: synth.make_window(3, seed=41), True, 8, None),     # 300 rows: k_schur_syrk, global k_reduced_solve
    "config5_kf40": (lambda: synth.make_window(5, n_kf=40, n_lm=3000, n_obs=45000), False, 8, None),  # 234 rows, plane-free large
    "motion_only": (lambda: _motion_only(False), False, 1, _motion_options),              # landmarks_fixed: a 6x6 system
    "motion_only_speed_prior": (lambda: _motion_only(True), False, 1, _motion_options),
    "evaluation_failure": (ew.CASES["evaluation_failure"], False, 1, None),               # a FAILURE solve without records
    "tiny": (ew.CASES["tiny"], False, 1, None),                                           # a single solve
    "all_keyframes_fixed": (ew.CASES["all_keyframes_fixed"], False, 1, None),             # no reduced system
}
# the window of the kernel-variant tests (the config-2 shape of test_fused_schur_equals_round_one_schur)
VARIANT_CASES = dict(CASES, config2_slice=(lambda: synth.make_window(2, n_kf=16, n_lm=900, n_obs=9000, seed=9), False, 1, None))
CPU_CASES = ["config1", "config2_slice", "config3_kf8", "evaluation_failure", "tiny", "all_keyframes_fixed"]


def build_case(name):
    """(window, options, prefix rule, oracle threads) of a case"""
    from oracle import oracle as orc
    make, prefix, threads, hook = VARIANT_CASES[name]
    opt = orc.default_options()
    if hook:
        hook(opt)
    return make(), opt, prefix, threads


@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


@pytest.mark.parametrize("name", CPU_CASES)
def test_oracle_log_satisfies_the_invariants(oracle, name):
    """check_log_invariants on the oracle's own logs (no GPU): numbering, summaries, the radius recurrence of Ceres 1.13, the
    bookkeeping of cost_change -- and a log that does not fit its buffer is clipped, not overrun"""
    win, opt, _, threads = build_case(name)
    res = oracle.solve_window(win, opt, num_threads=threads, iterations_capacity=LOG_CAPACITY)
    assert res.c.num_iteration_records >= res.c.num_solves - (name == "evaluation_failure")
    il.check_log_invariants(res, opt, name)
    il.log_deviations(res, res, prefix_rule=True, label=name)   # a log agrees with itself under either rule
    assert all(d == 0.0 for d, _ in il.log_deviations(res, res, label=name).values())
    short = oracle.solve_window(win, opt, num_threads=threads, iterations_capacity=3)
    assert short.c.num_iteration_records == min(3, res.c.num_iteration_records)


def test_a_wrong_record_breaks_the_invariants(oracle):
    """the helper can fail: one radius, one cost_change and one missing record, each caught"""
    win, opt, _, _ = build_case("config1")
    for field, value in (("trust_region_radius", lambda v: v * (1 + 1e-9)), ("cost_change", lambda v: v * (1 + 1e-6)),
                         ("iteration", lambda v: v + 1)):
        res = oracle.solve_window(win, opt, iterations_capacity=LOG_CAPACITY)
        i = next(i for i, e in enumerate(res.iterations) if e.step_is_successful)
        setattr(res._iters[i], field, value(getattr(res._iters[i], field)))
        with pytest.raises(AssertionError):
            il.check_log_invariants(res, opt, field)
    a = oracle.solve_window(win, opt, iterations_capacity=LOG_CAPACITY)
    b = oracle.solve_window(win, opt, iterations_capacity=LOG_CAPACITY)
    i = next(i for i, e in enumerate(b.iterations) if e.step_is_successful)
    b._iters[i].step_norm *= 1 + 1e-7
    with pytest.raises(AssertionError, match="step_norm"):
        il.compare_logs(b, a, il.TOL["fp64_head"], head=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_iteration_log_matches_oracle(handle, oracle, name):
    """every record of the CUDA log against the oracle's: flags exactly, the six numbers of the log's head at the sharp row
    of iter_log.TOL and of every record at the loose one (why there are two is said there).
    Plane-free windows: the whole log.  Ground-plane windows: the prefix rule of iter_log.log_deviations."""
    win, opt, prefix, threads = build_case(name)
    rg = handle.solve_window(win, opt, iterations_capacity=LOG_CAPACITY)
    rc = oracle.solve_window(win, opt, num_threads=threads, iterations_capacity=LOG_CAPACITY)
    assert rg.c.status == 0
    il.check_log_invariants(rc, opt, name + " (oracle)")
    il.check_log_invariants(rg, opt, name + " (cuda)")
    assert [s.termination for s in rg.solves] == [s.termination for s in rc.solves]
    il.compare_logs(rg, rc, il.TOL["fp64_head"], prefix_rule=prefix, label=name, head=True)
    il.compare_logs(rg, rc, il.TOL["fp64"], prefix_rule=prefix, label=name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["config2_slice", "config3_kf8"])
@pytest.mark.parametrize("variant", ["KBA_LINEARIZE", "KBA_FUSED"])
def test_kernel_variants_write_the_same_log(handle, oracle, monkeypatch, variant, name):
    """the three materialising linearisation kernels (KBA_LINEARIZE=0) and the round-1 Schur path (KBA_FUSED=0; both read when
    a batch is created) against the same oracle log, at the same tolerances as the default kernels"""
    win, opt, prefix, threads = build_case(name)
    monkeypatch.setenv(variant, "0")
    rg = handle.solve_window(win, opt, iterations_capacity=LOG_CAPACITY)
    rc = oracle.solve_window(win, opt, num_threads=threads, iterations_capacity=LOG_CAPACITY)
    il.check_log_invariants(rg, opt, "%s %s=0" % (name, variant))
    il.compare_logs(rg, rc, il.TOL["fp64_head"], prefix_rule=prefix, label="%s %s=0" % (name, variant), head=True)
    il.compare_logs(rg, rc, il.TOL["fp64"], prefix_rule=prefix, label="%s %s=0" % (name, variant))


@pytest.mark.gpu
def test_fp32_linearisation_log(handle, oracle):
    """kba_options.precision = 1 on config 2: single-precision blocks move every step a little, so only the first inner solve
    is compared (the same landmarks are in it whatever the precision), in cost, step_norm and the accept / reject flags"""
    win, opt, _, threads = build_case("config2_full")
    rc = oracle.solve_window(win, opt, num_threads=threads, iterations_capacity=LOG_CAPACITY)
    opt.precision = 1
    rg = handle.solve_window(win, opt, iterations_capacity=LOG_CAPACITY)
    il.check_log_invariants(rg, opt, "fp32")
    il.compare_logs(rg, rc, il.TOL["fp32_linearize"], solves=(0,), label="fp32")
