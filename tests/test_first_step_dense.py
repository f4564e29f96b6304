"""Iteration 1 of a window's first inner solve against a dense extended-precision Levenberg-Marquardt step.

tests/test_iteration_log.py holds the CUDA log to the oracle's, and so trusts the oracle's Schur elimination, Jacobi scaling,
damping, back substitution and controller arithmetic.  This file pins the first step of both to a reference that shares none
of that code: the damped normal equations of the WHOLE program (poses, plane directions and distances, landmarks; no
elimination), assembled and solved in numpy.longdouble -- on the x86 hosts this suite runs on that is the 80-bit extended type
(64-bit significand), which is what the host provides; the test is skipped where longdouble is no wider than double.

From the implementation under test it takes the robustified observation blocks (r, J_pose, J_landmark, cost) of evaluate(),
which tests/test_gpu_parity.py::test_eval_matches_oracle and tests/test_oracle_jacobians.py pin on their own.  From the oracle
it takes the single-residual functions pose_plus, dir_plus, gp_height, gp_motion, scale_reg and speed_reg, which
tests/test_oracle_jacobians.py checks by finite differences.  Everything else -- which parameter blocks are in the program, the
Huber corrector of the ground rows, the weights of the plane chain, the FixScaleVectorPlus Jacobian of the direction-difference
rows, the step and the controller -- is restated here.

The windows between them select every solver path of limo_b200/csrc/kba_plan.h (asserted on each, through the plan driver of
tests/test_launch_plan.py): the fused path with and without plane rows, the seven-slot k_schur_fused<7> (windows with no fixed
keyframe: a free gauge makes their later iterates drift along flat directions, but the first damped step is well defined), the
large-window path with the tiled, the split (k_chol_*) and the one-CTA row-major factorisation, the 6x6 motion-only system with
its speed prior.  FP32 observation blocks (kba_options.precision = 1) run on the fused six- and seven-slot paths, the split
factorisation with and without plane blocks, config 3's batch of 132 and (tests/test_large_reduced_rows.py) the 651-row
k_chol_trail_band path, each held at its FP64 class against the mixed system the FP32 solve forms (dense_first_step).

The Schur split (p_split: the CTAs a window's Schur sum is spread over) follows the batch size, and each case asserts it.  A
window solved alone splits its sum over 25 .. 88 CTAs on the fused path and over 16 on the large-window path, the batch of 17
over 5: k_sred_reduce folds the partial sums and k_reduced_solve takes A from it.  The batches of 264 (config2_slice in FP64
and FP32, config2_kf30_lm700 with the headline's 30 keyframes), 132 (free_keyframes_30, config3_kf30_lm600 in FP64 and FP32)
and 80 (config5_kf40_lm700) windows run at p_split = 1, the shapes bench.py times: one CTA owns all of a window's landmark
groups in k_schur_fused, k_schur_syrk runs at a grid depth of 1, k_sred_reduce is not launched, and k_reduced_solve gathers A from the
single sum itself, tiled or row-major.  The split factorisation at p_split = 1 (KBA_P_SPLIT=1) is in
tests/test_bench_shapes.py.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.linalg

from limo_b200 import synth
from tests import edge_windows as ew
from tests import iter_log as il
from tests.test_launch_plan import driver  # noqa: F401  (the plan driver fixture)

LD = np.longdouble
pytestmark = pytest.mark.skipif(np.finfo(LD).eps >= np.finfo(np.float64).eps, reason="numpy.longdouble is not an extended type here")

# Records 0 and 1 against the dense step, relative (cost_change in units of the cost).  Worst observed, oracle and CUDA path on an
# NVIDIA H100 80GB HBM3 (power limit 700 W), by scripts/iteration_log_agreement.py:
#   plane-free windows (config1 .. config5_kf40_lm700, motion_only_speed_prior, the batch of 17):
#     oracle: step_norm 2.4e-12 (ragged: landmarks seen once, held by the damping alone), cost 5.7e-13, relative_decrease 2.9e-13
#     CUDA:   step_norm 1.2e-12 (stereo_rig), cost 4.2e-13, cost_change 1.7e-13, relative_decrease 3.0e-13 (config2_slice)
#   ground-plane windows (config3_kf8, config3_kf14, planes_kf18_none_fixed, config3_kf30_lm600):
#     oracle: step_norm 8.0e-13 (config3_kf14), cost 7.5e-13, relative_decrease 4.0e-13 (planes_kf18_none_fixed)
#     CUDA:   step_norm 2.8e-13 (config3_kf14), cost 3.1e-14, relative_decrease 1.7e-14
#   config2_kf30_lm700: oracle cost 7.7e-13, step_norm 2.7e-13, relative_decrease 3.9e-13; CUDA cost 6.1e-14, step_norm 1.8e-13
#   the batches at p_split = 1, worst window of each batch:
#     plane-free (config2_slice and config2_kf30_lm700 x 264, free_keyframes_30 x 132, config5_kf40_lm700 x 80):
#             cost 4.1e-13, cost_change 1.7e-13, step_norm 6.5e-13, relative_decrease 3.0e-13 (config2_slice x 264)
#     ground (config3_kf30_lm600 x 132): cost 3.0e-14, cost_change 9.2e-15, step_norm 1.8e-13, relative_decrease 1.2e-14
#     config3_kf30_lm600 alone with KBA_P_SPLIT=1, factorised by k_chol_* (tests/test_bench_shapes.py): the same figures
# STEP_TOL is about 100 times the worst plane-free deviation.  A ground window has few ground rows: one of them, or one row of
# the plane chain, wrong by 1e-6 moves the records by 9e-11 .. 1.8e-10 (test_dense_step_notices_a_wrong_ground_row), so
# GROUND_TOL sits between that and the worst ground deviation (12 times the oracle's, 36 times the CUDA path's).
#
# FP32 blocks (kba_options.precision = 1).  The FP32 solve does not form the normal equations of the blocks kba_eval reports:
# k_pose_hessian re-evaluates each observation's pose rows in FP64 for the pose blocks and the pose gradient, while the landmark
# blocks, the landmark gradient and the pose-landmark coupling come from the FP32 J_p, J_l and r.  dense_first_step forms that
# mixed system when given the FP64 blocks beside the FP32 ones (cuda_reference), and every FP32 case is held at its FP64 class.
# Worst deviation, every window of each batch, at the origin and at 1, 5 and 10 km (tests/test_far_windows.py), measured on an
# NVIDIA H100 80GB HBM3 (power limit 700 W) by scripts/fp32_agreement.py:
#   plane-free (config2_slice alone and x 264, free_kf30_none_fixed, config5_kf40_lm700): 9.6e-13 (config5_kf40_lm700, 1 km;
#     1.5e-13 at the origin)
#   ground (config3_kf30_lm600 alone and x 132): 2.5e-13 (5 km; 1.5e-13 at the origin); the 651-row window 8.4e-14
# The reference built from the FP32 blocks alone (the pose rows from FP32 as well) is off by 2.4e-06 .. 2.3e-04 on the same
# cases, and one FP32 landmark Jacobian row or one FP32 residual off by 1e-6 moves the mixed reference by 7.2e-10 .. 1.5e-09
# (config2_slice, config3_kf30_lm600): both fail the classes (test_cuda_fp32_step_is_the_mixed_system).
STEP_TOL = 1e-10
GROUND_TOL = 1e-11
TOL = {"plane_free": STEP_TOL, "ground": GROUND_TOL}


def _shapes(name):
    from tests import test_schur_fused_shapes as sf
    return getattr(sf, name)()


def _motion_only(with_prior):
    from tests import test_iteration_log as tl
    return tl._motion_only(with_prior)


def _no_fixed_keyframe(win):
    return ew.copy_window(win, kf_fixed=np.zeros(win.n_kf, dtype=np.uint8))


# name -> (window builder, tolerance class, columns of the dense system, launch plan fields the window selects as a batch of one).
# Names follow tests/test_iteration_log.CASES where the window is there; landmark counts are cut so that every dense system
# stays below 2 500 columns.
WINDOWS = {
    "config1": (lambda: synth.make_window(1), "plane_free", 624, dict(fused=1, fused_slots=6)),
    "config2_slice": (lambda: synth.make_window(2, n_kf=12, n_lm=400, n_obs=3000), "plane_free", 1266,
                      dict(fused=1, fused_slots=6)),
    "stereo_rig": (lambda: _shapes("_stereo_rig"), "plane_free", 942, dict(fused=1, fused_slots=6)),
    "gap_over_fixed_keyframe": (lambda: _shapes("_gap_over_fixed_keyframe"), "plane_free", 2148, dict(fused=1, fused_slots=6)),
    "ragged": (ew.CASES["ragged"], "plane_free", 612, dict(fused=1, fused_slots=6)),
    # plane rows, Huber ground rows and the plane chain on the fused path
    "config3_kf8": (lambda: synth.make_window(3, seed=41, n_kf=8, n_lm=300, n_obs=1800, gp_frac=0.2), "ground", 970,
                    dict(fused=1, fused_slots=6)),
    "config3_kf14": (lambda: synth.make_window(3, seed=41, n_kf=14, n_lm=500, n_obs=4500), "ground", 1630,
                     dict(fused=1, fused_slots=6)),
    # 181 rows over 18 keyframes with plane blocks, none of them fixed: k_schur_fused<7> with plane blocks
    "planes_kf18_none_fixed": (lambda: _no_fixed_keyframe(synth.make_window(3, seed=43, n_kf=18, n_lm=500, n_obs=4500)),
                               "ground", 1680, dict(fused=1, fused_slots=7)),
    # 181 rows over 30 keyframes, 175 of them free: k_schur_fused<6> at the headline's 30 keyframes (config2_slice has 67 rows)
    "config2_kf30_lm700": (lambda: synth.make_window(2, n_kf=30, n_lm=700, n_obs=7000, seed=5), "plane_free", 2274,
                           dict(fused=1, fused_slots=6)),
    # 181 rows over 30 plane-free keyframes, none of them fixed: k_schur_fused<7>
    "free_kf30_none_fixed": (lambda: _no_fixed_keyframe(synth.make_window(2, n_kf=30, n_lm=700, n_obs=7000, seed=5)),
                             "plane_free", 2280, dict(fused=1, fused_slots=7)),
    # 187 rows over 31 keyframes: the large-window path, k_reduced_solve tiled at 192 rows
    "free_keyframes_30": (lambda: synth.make_window(2, n_kf=31, n_lm=700, n_obs=7000, seed=5), "plane_free", 2280,
                          dict(fused=0, small_syrk=0, nr_cap_max=192, solve_tiled=1, solve_split=0)),
    # 301 rows with plane blocks: k_eval_obs<true>, k_schur_syrk, row-major factorisation split over 32 CTAs (k_chol_*)
    "config3_kf30_lm600": (lambda: synth.make_window(3, seed=41, n_lm=600, n_obs=6000), "ground", 2090,
                           dict(fused=0, small_syrk=0, nr_cap_max=320, solve_tiled=0, solve_split=32)),
    # 241 rows, plane-free: row-major, k_chol_* split
    "config5_kf40_lm700": (lambda: synth.make_window(5, n_kf=40, n_lm=700, n_obs=8000), "plane_free", 2334,
                           dict(fused=0, small_syrk=0, nr_cap_max=256, solve_tiled=0, solve_split=32)),
    # adjustPoseOnly: landmarks constant, one pose and the speed prior
    "motion_only_speed_prior": (lambda: _motion_only(True), "plane_free", 6, dict(fused=1, fused_slots=6)),
}


def _motion_options(opt):
    opt.min_landmarks_for_trimming = 30


OPTION_HOOKS = {"motion_only_speed_prior": _motion_options}

# CUDA runs: name -> (window of WINDOWS, kba_options.precision, copies in one kba_solve_batch, plan fields beyond the window's)
CUDA_CASES = dict({name: (name, 0, 1, {}) for name in WINDOWS},
                  # 17 windows: more than the split factorisation takes, so k_reduced_solve factorises each in one CTA
                  config5_kf40_lm700_batch17=("config5_kf40_lm700", 0, 17, dict(p_split=5, solve_tiled=0, solve_split=0)),
                  # FP32 observation blocks (k_eval_obs<float>), everything after them in FP64, on every path they take: the
                  # fused six- and seven-slot kernels, the split (k_chol_*) factorisation with and without plane blocks, and
                  # config 3's sub-record shape below
                  config2_slice_fp32=("config2_slice", 1, 1, {}),
                  free_kf30_none_fixed_fp32=("free_kf30_none_fixed", 1, 1, {}),
                  config3_kf30_lm600_fp32=("config3_kf30_lm600", 1, 1, {}),
                  config5_kf40_lm700_fp32=("config5_kf40_lm700", 1, 1, {}),
                  # The batch sizes bench.py times put each window's Schur sum on one CTA (p_split = 1): k_sred_reduce is not
                  # launched and k_reduced_solve gathers A from the sums itself.  264 windows: bench.py's headline batch, the
                  # fused six-slot kernel with one CTA owning all of a window's landmark groups, then the tiled solve
                  config2_slice_batch264=("config2_slice", 0, 264, dict(p_split=1, solve_tiled=1)),
                  config2_slice_fp32_batch264=("config2_slice", 1, 264, dict(p_split=1, solve_tiled=1)),
                  config2_kf30_lm700_batch264=("config2_kf30_lm700", 0, 264, dict(p_split=1, solve_tiled=1)),
                  # 132 windows: k_schur_syrk at a grid depth of 1, tiled k_reduced_solve<true>
                  free_keyframes_30_batch132=("free_keyframes_30", 0, 132, dict(p_split=1, solve_tiled=1, solve_split=0)),
                  # 132 windows: config 3's sub-record shape, the row-major k_reduced_solve<false> in one CTA per window
                  config3_kf30_lm600_batch132=("config3_kf30_lm600", 0, 132, dict(p_split=1, solve_tiled=0, solve_split=0)),
                  config3_kf30_lm600_fp32_batch132=("config3_kf30_lm600", 1, 132, dict(p_split=1, solve_tiled=0, solve_split=0)),
                  # the same plane-free; 80 is the smallest batch for which syrk_split(256, n, 132) == 1
                  config5_kf40_lm700_batch80=("config5_kf40_lm700", 0, 80, dict(p_split=1, solve_tiled=0, solve_split=0)))


def build(name):
    """(window, options) of a window of WINDOWS"""
    from oracle import oracle as orc
    opt = orc.default_options()
    if name in OPTION_HOOKS:
        OPTION_HOOKS[name](opt)
    return WINDOWS[name][0](), opt


def plan_shape(win):
    """(rows, free rows, 32-landmark chunks, 8-landmark groups, landmarks) of a window as kba_batch_create sizes it"""
    planes = win.n_gp > 0 or win.plane_reg_weight > 0
    per = 10 if planes else 6
    free = int((np.asarray(win.kf_fixed) == 0).sum())
    return per * win.n_kf + 1, per * free + 1, -(-win.n_lm // 32), -(-win.n_lm // 8), win.n_lm


def assert_path(driver, windows, want):  # noqa: F811
    """the launch plan of kba_solve_batch on `windows` (default knobs, an H100's SMs) has the fields of `want`"""
    from tests.test_launch_plan import FIELDS, _query
    got = dict(zip(FIELDS, map(int, driver(_query("plan", [plan_shape(w) for w in windows], "batch", 1, 0, 1))[0].split())))
    assert {k: got[k] for k in want} == want, (got, want)


def _solve_spd(A, b):
    """A y = b for a symmetric positive definite longdouble A: double-precision Cholesky, residuals and updates in longdouble
    (iterative refinement contracts by cond(A) * 2^-53 per round; the damped, Jacobi-scaled matrix has a condition of at most
    ~1e10, 5e4 on config 1).  It stops once a correction is below 1e-14 of the solution: the following one is smaller still,
    and the records it is compared with are held to 1e-9 .. 1e-11"""
    cf = scipy.linalg.cho_factor(A.astype(np.float64), lower=True)
    y = np.zeros_like(b)
    for _ in range(12):
        res = b - A @ y
        dy = scipy.linalg.cho_solve(cf, res.astype(np.float64)).astype(LD)
        y = y + dy
        if np.abs(dy).max() <= 1e-14 * np.abs(y).max():
            return y
    raise AssertionError("iterative refinement did not converge")


def program_columns(win):
    """The parameter blocks of the window's first solve and their columns, by the rules of the oracle's program_layout
    (kba_oracle.c): a pose for each keyframe that is observed, anchors a ground point, is a scale keyframe or carries the speed
    prior -- every keyframe under the plane-chain regularisation (weight > 0, at least two keyframes); a direction (3) and a
    distance (1) for each keyframe with a ground point, or every keyframe under the regularisation, no distance when
    plane_dist_fixed; nothing for a fixed keyframe; a landmark for each landmark with an observation or a ground point, none when
    landmarks_fixed.  Columns run keyframe by keyframe (pose, direction, distance), then the landmarks."""
    K = win.n_kf
    gp_lm = np.zeros(0, dtype=int) if win.n_gp == 0 else np.asarray(win.gp_lm)
    gp_kf = np.zeros(0, dtype=int) if win.n_gp == 0 else np.asarray(win.gp_kf)
    pose_in, plane_in = np.zeros(K, dtype=bool), np.zeros(K, dtype=bool)
    pose_in[np.asarray(win.obs_kf)] = True
    pose_in[gp_kf] = plane_in[gp_kf] = True
    if win.scale_weight > 0:
        pose_in[[win.scale_kf0, win.scale_kf1]] = True
    if win.plane_reg_weight > 0 and K > 1:
        pose_in[:] = plane_in[:] = True
    if win.speed_weight > 0:
        pose_in[win.speed_kf] = True
    L = SimpleNamespace(pose={}, dir={}, dist={})
    n = 0
    for k in range(K):
        if win.kf_fixed[k]:
            continue
        if pose_in[k]:
            L.pose[k] = n; n += 6
        if plane_in[k]:
            L.dir[k] = n; n += 3
            if not win.plane_dist_fixed:
                L.dist[k] = n; n += 1
    L.n_f = n
    lm_in = np.diff(np.asarray(win.lm_obs_ptr)) > 0
    lm_in[gp_lm] = True
    if win.landmarks_fixed:
        lm_in[:] = False
    L.lm_in = np.flatnonzero(lm_in)
    L.lm = np.full(win.n_lm, -1)
    L.lm[L.lm_in] = n + 3 * np.arange(len(L.lm_in))
    L.n = n + 3 * len(L.lm_in)
    return L


def _dir_plus_jacobian(n):
    """FixScaleVectorPlus at delta = 0, local_parameterizations.hpp:146-162: (I - n n^T / |n|^2) / |n|"""
    n = np.asarray(n, dtype=LD)
    nn = n @ n
    return (np.eye(3, dtype=LD) - np.outer(n, n) / nn) / np.sqrt(nn)


def _row(kind, parts, r, sqrt_rho1):
    """one residual block: (column or None (constant block), Jacobian) parts and the residual, each times sqrt(rho') -- Ceres'
    corrector for rho'' <= 0, which holds for every loss here"""
    parts = [(c, sqrt_rho1 * np.atleast_2d(np.asarray(J, dtype=LD))) for c, J in parts if c is not None and c >= 0]
    return SimpleNamespace(kind=kind, parts=parts, r=sqrt_rho1 * np.atleast_1d(np.asarray(r, dtype=LD)))


def other_rows(win, opt, orc, L, poses, planes, lms):
    """The residual blocks besides the observations, and their cost, at (poses, planes, lms):
      ground points: gp_height with ScaledLoss(Huber(gp_huber), weight) (cpp:517-562);
      scale: scale_reg with ScaledLoss(Trivial, weight) (cpp:890-904);
      plane chain (cpp:769-818), for each pair of consecutive keyframes: dir1 - dir0 (weight 3w), dist1 - dist0 (w),
      gp_motion (2w); for each keyframe (0, 0, 1) - dir (w);
      speed prior: speed_reg with weight speed_weight (cpp:835-853)."""
    rows, cost = [], LD(0)

    def trivial(kind, parts, r, weight):
        nonlocal cost
        r = np.atleast_1d(np.asarray(r, dtype=LD))
        cost += LD(weight) * (r @ r) / 2
        rows.append(_row(kind, parts, r, np.sqrt(LD(weight))))

    a = LD(opt.gp_huber)
    for g in range(win.n_gp):
        j, k = int(win.gp_lm[g]), int(win.gp_kf[g])
        res, jp, jd, jdist, jl = orc.gp_height(poses[k], planes[k, :3], planes[k, 3], lms[j])
        s, w = LD(res[0]) ** 2, LD(win.gp_weight[g])
        rho0, rho1 = (2 * a * np.sqrt(s) - a * a, a / np.sqrt(s)) if s > a * a else (s, LD(1))
        cost += w * rho0 / 2
        rows.append(_row("ground", [(L.pose.get(k), jp), (L.dir.get(k), jd), (L.dist.get(k), jdist), (L.lm[j], jl)], res,
                         np.sqrt(w * rho1)))
    if win.scale_weight > 0:
        res, j1, j0 = orc.scale_reg(poses[win.scale_kf1], poses[win.scale_kf0], win.scale_value)
        trivial("scale", [(L.pose.get(win.scale_kf1), j1), (L.pose.get(win.scale_kf0), j0)], res, win.scale_weight)
    if win.plane_reg_weight > 0 and win.n_kf > 1:
        w = win.plane_reg_weight
        for k0 in range(win.n_kf - 1):
            k1 = k0 + 1
            n0, n1 = planes[k0, :3], planes[k1, :3]
            trivial("plane_dir", [(L.dir.get(k1), _dir_plus_jacobian(n1)), (L.dir.get(k0), -_dir_plus_jacobian(n0))],
                    np.asarray(n1, dtype=LD) - np.asarray(n0, dtype=LD), 3 * w)
            trivial("plane_dist", [(L.dist.get(k1), [[1.0]]), (L.dist.get(k0), [[-1.0]])], LD(planes[k1, 3]) - LD(planes[k0, 3]), w)
            res, j0, j1, jd = orc.gp_motion(poses[k0], poses[k1], n0)
            trivial("plane_motion", [(L.pose.get(k0), j0), (L.pose.get(k1), j1), (L.dir.get(k0), jd)], res, 2 * w)
        for k in range(win.n_kf):
            trivial("plane_up", [(L.dir.get(k), -_dir_plus_jacobian(planes[k, :3]))],
                    np.array([0, 0, 1], dtype=LD) - np.asarray(planes[k, :3], dtype=LD), w)
    if win.speed_weight > 0:
        res, jp = orc.speed_reg(poses[win.speed_kf], win.speed_T_origin_before, win.speed_dt, win.speed_v_before)
        trivial("speed", [(L.pose.get(win.speed_kf), jp)], res, win.speed_weight)
    return rows, cost


def _planes(win):
    """the plane state (direction, distance) of every keyframe: the window's, or the oracle's default (0, 0, 1, 0)"""
    return np.tile([0.0, 0.0, 1.0, 0.0], (win.n_kf, 1)) if win.kf_plane is None else win.kf_plane.copy()


def dense_first_step(win, opt, blocks, evaluate, orc, tamper=None, fp64_blocks=None):
    """Records 0 and 1 of the first inner solve as a dense reference gives them.

    blocks: (r [n_obs, 3], jac_pose [n_obs, 3, 6], jac_lm [n_obs, 3, 3], cost) of the observations at the window's state;
    evaluate(window) returns the same tuple (the candidate's observation cost is taken from it); orc: the oracle binding (its
    single-residual functions).  tamper(rows), if given, may change the residual blocks at the window's state before the system
    is formed (the negative controls).  The Jacobian is never stored densely (18 000 x 2 300 longdoubles); J^T J and J^T r are
    summed from its blocks, which is the same matrix.

    fp64_blocks: the FP64 blocks of the same observations (kba_eval at precision 0), given with the FP32 `blocks` of
    kba_options.precision = 1.  The FP32 solve does not form the normal equations of one Jacobian but a mixed system, and with
    both sets given the reference forms that system:
      - k_pose_hessian re-evaluates every observation's pose rows in FP64: the pose-pose blocks B_k = sum J_p^T J_p, the pose
        gradient g_k = sum J_p^T r and so the pose columns' Jacobi norms (the diagonal of B_k, k_reduced_solve) come from the
        rows of `fp64_blocks`;
      - k_landmark_reduce sums C_j = sum J_l^T J_l and g_j = sum J_l^T r (and the landmark columns' Jacobi norms) from the FP32
        J_l and r, and k_obs_v / k_obs_v2 the coupling J_p^T J_l from the FP32 J_p and J_l, each widened to FP64 (lin_load).  The
        J_l is the stored FP32 one on the large-window path (k_eval_obs<float, true>) and the FP32 translation columns times R
        formed in FP64 on the fused path (k_eval_obs<float, false>); kba_eval reports whichever the window's path consumes;
      - ground rows, the plane chain and the regularisers are FP64 either way (k_gp_eval, k_reduced_solve).
    Then the model decrease is the one k_reduced_solve and k_backsub form from that g, the step and the damping,
    (-g^T delta + delta^T Lambda delta) / 2 with Lambda the damping in unscaled columns, summed to k_lm_update's model_change: the
    row form -(J delta)^T (r + J delta / 2) equals it only for a consistent Jacobian.  gradient_max_norm is taken from the same
    g."""
    r, jp, jl = (np.asarray(a, dtype=LD) for a in blocks[:3])
    L = program_columns(win)
    n = L.n
    lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(np.asarray(win.lm_obs_ptr)))
    kf_of_obs = np.asarray(win.obs_kf)
    planes0 = _planes(win)
    mixed = fp64_blocks is not None
    if mixed:
        r64, jp64 = (np.asarray(a, dtype=LD) for a in fp64_blocks[:2])

    rows = []
    for o in range(win.n_obs):
        pc = L.pose.get(int(kf_of_obs[o]))
        rw = SimpleNamespace(kind="observation", r=r[o], parts=[(c, J) for c, J in ((pc, jp[o]), (L.lm[lm_of_obs[o]], jl[o]))
                                                                if c is not None and c >= 0])
        # the pose part, when there is one, is the row's first: its J^T J and J^T r come from the FP64 row
        rw.pose64 = (jp64[o], r64[o]) if mixed and pc is not None else None
        rows.append(rw)
    more, other_cost = other_rows(win, opt, orc, L, win.kf_pose, planes0, win.lm_pos)
    rows += more
    if tamper:
        tamper(rows)
    rows = [(np.concatenate([np.arange(c, c + J.shape[1]) for c, J in rw.parts]), np.concatenate([J for _, J in rw.parts], axis=1),
             rw.r, getattr(rw, "pose64", None)) for rw in rows if rw.parts]

    H, g = np.zeros((n, n), dtype=LD), np.zeros(n, dtype=LD)
    for cols, vals, res, pose64 in rows:
        M, v = vals.T @ vals, vals.T @ res
        if pose64 is not None:
            M[:6, :6] = pose64[0].T @ pose64[0]
            v[:6] = pose64[0].T @ pose64[1]
        H[np.ix_(cols, cols)] += M
        g[cols] += v
    c = np.diag(H).copy()                                   # squared column norms
    s = 1 / (1 + np.sqrt(c))                                # Jacobi scaling, taken once at the first iterate
    radius = LD(opt.initial_trust_region_radius)
    D = np.clip(c * s * s, LD(opt.min_lm_diagonal), LD(opt.max_lm_diagonal)) / radius
    A = H * s[:, None] * s[None, :]
    A[np.diag_indices(n)] += D
    delta = s * _solve_spd(A, -s * g)
    if mixed:                                               # (-g^T delta + delta^T Lambda delta) / 2, Lambda = D / s^2
        model = (-(g @ delta) + (D / (s * s)) @ (delta * delta)) / 2
    else:                                                   # -(J delta)^T (r + J delta / 2)
        model = LD(0)
        for cols, vals, res, _ in rows:
            jd = vals @ delta[cols]
            model -= jd @ (res + jd / 2)

    def blocks_of(poses, planes, lms):
        """the variable blocks of a state in ambient coordinates, one vector"""
        return np.concatenate([poses[list(L.pose)].ravel(), planes[list(L.dir)][:, :3].ravel(), planes[list(L.dist)][:, 3],
                               lms[L.lm_in].ravel()]).astype(LD)

    def plus(step):
        """x + step: pose_plus on the poses, dir_plus on the directions, addition on distances and landmarks; and the norms of
        the ambient difference"""
        step = step.astype(np.float64)
        poses, planes, lms = win.kf_pose.copy(), planes0.copy(), win.lm_pos.copy()
        for k, c0 in L.pose.items():
            poses[k] = orc.pose_plus(win.kf_pose[k], step[c0:c0 + 6])
        for k, c0 in L.dir.items():
            planes[k, :3] = orc.dir_plus(planes0[k, :3], step[c0:c0 + 3])
        for k, c0 in L.dist.items():
            planes[k, 3] = planes0[k, 3] + step[c0]
        lms[L.lm_in] += step[L.n_f:].reshape(-1, 3)
        diff = blocks_of(poses, planes, lms) - blocks_of(win.kf_pose, planes0, win.lm_pos)
        return poses, planes, lms, np.sqrt(diff @ diff), np.abs(diff).max()

    out = SimpleNamespace(cost0=LD(blocks[3]) + other_cost, radius0=radius, n_columns=n)
    out.gradient_max_norm0 = plus(-g)[4]
    poses, planes, lms, out.step_norm, _ = plus(delta)
    cand = ew.copy_window(win, kf_pose=poses, kf_plane=None if win.kf_plane is None else planes, lm_pos=lms)
    cand_blocks = evaluate(cand)
    assert cand_blocks[4] == 0
    cand_cost = LD(cand_blocks[3]) + other_rows(win, opt, orc, L, poses, planes, lms)[1]
    out.cost_change = out.cost0 - cand_cost
    out.relative_decrease = out.cost_change / model
    out.successful = bool(out.relative_decrease > opt.min_relative_decrease)
    # neither tolerance test fires on the first step of these windows (the record would be written differently)
    x = blocks_of(win.kf_pose, planes0, win.lm_pos)
    assert out.step_norm > opt.parameter_tolerance * (np.sqrt(x @ x) + opt.parameter_tolerance)
    assert abs(out.cost_change) > opt.function_tolerance * out.cost0
    out.cost1 = cand_cost                                   # the accepted iterate's cost, or the rejected candidate's
    rho = out.relative_decrease
    out.radius1 = min(LD(opt.max_trust_region_radius), radius / max(LD(1) / 3, 1 - (2 * rho - 1) ** 3)) if out.successful else radius / 2
    return out


def _check_first_step(res, ref, tol, label):
    """records 0 and 1 of `res` (first inner solve) against the dense step, every field at `tol` (relative; cost_change in
    units of the cost)"""
    recs = il.records(res)
    r0, r1 = recs[0], recs[1]
    assert (r0.solve_index, r0.iteration, r1.solve_index, r1.iteration) == (0, 0, 0, 1), label
    dev = {
        "cost 0": abs(r0.cost - ref.cost0) / ref.cost0,
        "gradient_max_norm 0": abs(r0.gradient_max_norm - ref.gradient_max_norm0) / ref.gradient_max_norm0,
        "radius 0": abs(r0.trust_region_radius - ref.radius0) / ref.radius0,
        "cost 1": abs(r1.cost - ref.cost1) / ref.cost1,
        "cost_change": abs(r1.cost_change - ref.cost_change) / ref.cost0,
        "step_norm": abs(r1.step_norm - ref.step_norm) / ref.step_norm,
        "relative_decrease": abs(r1.relative_decrease - ref.relative_decrease) / abs(ref.relative_decrease),
        "radius 1": abs(r1.trust_region_radius - ref.radius1) / ref.radius1,
    }
    assert r1.valid and r1.successful == ref.successful, label
    for name, d in dev.items():
        assert d <= tol, (label, name, float(d), tol)
    return {k: float(v) for k, v in dev.items()}


@pytest.mark.parametrize("name", list(WINDOWS))
def test_oracle_first_step_matches_dense_step(oracle, driver, name):  # noqa: F811
    """the oracle's elimination, scaling, damping, back substitution and controller arithmetic, without a GPU; and the solver
    path the window selects on the CUDA side"""
    _, tol, columns, path = WINDOWS[name]
    win, opt = build(name)
    assert_path(driver, [win], path)
    ref = dense_first_step(win, opt, oracle.evaluate(win, opt), lambda w: oracle.evaluate(w, opt), oracle)
    assert ref.successful and ref.n_columns == columns
    _check_first_step(oracle.solve_window(win, opt), ref, TOL[tol], name)


def test_dense_step_notices_a_wrong_block(oracle):
    """the reference can fail: the landmark Jacobian of ONE observation of 1000 off by 1e-6 moves the candidate cost by 1.4e-9"""
    win, opt = build("config1")
    r, jp, jl, cost, failed = oracle.evaluate(win)
    jl = jl.copy()
    jl[5] *= 1 + 1e-6
    ref = dense_first_step(win, opt, (r, jp, jl, cost, failed), oracle.evaluate, oracle)
    with pytest.raises(AssertionError):
        _check_first_step(oracle.solve_window(win, opt), ref, STEP_TOL, "perturbed")


# The mixed system of the FP32 mode with both block sets the same is the system of one Jacobian: worst deviation from the row
# form over the windows below 3.8e-18 (CPU, x86 80-bit longdouble); MIXED_SELF_TOL is 26 times it.  One landmark Jacobian row
# or one residual of the observation with the largest residual, off by 1e-6, moves the records by 7.2e-10 .. 5.8e-09.
MIXED_SELF_TOL = 1e-16
RECORD_FIELDS = ("cost0", "gradient_max_norm0", "step_norm", "cost_change", "relative_decrease", "cost1", "radius1")


def record_deviation(a, b):
    """largest relative difference between the records of two dense steps (cost_change in units of the cost)"""
    scale = dict(cost_change=b.cost0)
    return max(abs(getattr(a, f) - getattr(b, f)) / abs(scale.get(f, getattr(b, f))) for f in RECORD_FIELDS)


def tampered(blocks, what, factor=1 + 1e-6):
    """a copy of observation blocks with the residual (what="r") or the first landmark Jacobian row (what="jl") of the
    observation with the largest residual times `factor`"""
    r, jp, jl = (np.array(a, copy=True) for a in blocks[:3])
    o = int(np.argmax(np.linalg.norm(r, axis=1)))
    if what == "r":
        r[o] *= factor
    else:
        jl[o, 0] *= factor
    return (r, jp, jl) + tuple(blocks[3:])


@pytest.mark.parametrize("name", ["config2_slice", "free_kf30_none_fixed", "config3_kf30_lm600", "config5_kf40_lm700"])
def test_mixed_system_of_equal_blocks_is_the_dense_step(oracle, name):
    """dense_first_step's mixed system (FP64 pose rows beside the FP32 blocks) given the oracle's FP64 blocks twice is the
    system of one Jacobian: its records are the row form's to MIXED_SELF_TOL, and the oracle's step still meets its class.  And
    it can fail: one landmark Jacobian row or one residual of the second set, off by 1e-6, moves it out of the class"""
    win, opt = build(name)
    tol = TOL[WINDOWS[name][1]]
    blocks = oracle.evaluate(win, opt)
    ev = lambda w: oracle.evaluate(w, opt)  # noqa: E731
    ref = dense_first_step(win, opt, blocks, ev, oracle)
    mixed = dense_first_step(win, opt, blocks, ev, oracle, fp64_blocks=blocks)
    assert record_deviation(mixed, ref) <= MIXED_SELF_TOL
    res = oracle.solve_window(win, opt)
    _check_first_step(res, mixed, tol, name)
    for what in ("jl", "r"):
        bad = dense_first_step(win, opt, tampered(blocks, what), ev, oracle, fp64_blocks=blocks)
        with pytest.raises(AssertionError):
            _check_first_step(res, bad, tol, "%s, %s perturbed" % (name, what))


def _scale_part(kind, which, part, factor):
    """tamper(): the `part`-th Jacobian part of the `which`-th residual block of `kind` times `factor`"""
    def tamper(rows):
        rw = [x for x in rows if x.kind == kind][which]
        c, J = rw.parts[part]
        rw.parts[part] = (c, J * LD(factor))
    return tamper


@pytest.mark.parametrize("kind, which, part", [("ground", 0, 1),          # a ground point's direction Jacobian
                                               ("plane_motion", 2, 0)])   # a plane-chain row: gp_motion, pose of keyframe 2
def test_dense_step_notices_a_wrong_ground_row(oracle, kind, which, part):
    """the reference can fail on a ground window at the tolerance ground windows are held to: one ground row or one plane-chain
    row of config3_kf8 off by 1e-6"""
    win, opt = build("config3_kf8")
    blocks = oracle.evaluate(win, opt)
    res = oracle.solve_window(win, opt)
    _check_first_step(res, dense_first_step(win, opt, blocks, oracle.evaluate, oracle), GROUND_TOL, "as it is")
    ref = dense_first_step(win, opt, blocks, oracle.evaluate, oracle, tamper=_scale_part(kind, which, part, 1 + 1e-6))
    with pytest.raises(AssertionError):
        _check_first_step(res, ref, GROUND_TOL, "perturbed")


def test_window_copy_keeps_every_field():
    """copy_window carries the ground points, plane blocks and regularisers that the no-fixed-keyframe windows need"""
    ground, speed = build("config3_kf8")[0], build("motion_only_speed_prior")[0]
    assert ground.n_gp > 0 and ground.plane_reg_weight > 0 and speed.speed_weight > 0 and speed.landmarks_fixed
    for win in (ground, speed):
        cp = ew.copy_window(win)
        for f in ew.WINDOW_FIELDS:
            a, b = getattr(win, f), getattr(cp, f)
            assert (a is None and b is None) or np.array_equal(np.asarray(a), np.asarray(b)), f


@pytest.mark.parametrize("name", list(CUDA_CASES))
def test_cuda_case_selects_its_path(driver, name):  # noqa: F811
    """the launch plan each CUDA case runs on, held without a GPU: a change to the rules that moves a case off its path fails
    here, before the GPU run compares the wrong path"""
    window, _, copies, path = CUDA_CASES[name]
    assert_path(driver, [build(window)[0]] * copies, dict(WINDOWS[window][3], **path))


@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


def cuda_reference(handle, oracle, win, opt, fp32_pose_rows=False, **kw):
    """the dense step of a window from the blocks kba_eval reports under `opt`.  Under precision 1 it is the mixed system the
    FP32 solve forms (dense_first_step): the FP64 blocks, for the pose rows, are evaluated beside the FP32 ones.
    fp32_pose_rows: take the pose rows from the FP32 blocks as well (one Jacobian for the whole system; a negative control)."""
    blocks = handle.evaluate(win, opt)
    fp64 = None
    if opt.precision and not fp32_pose_rows:
        opt.precision = 0
        fp64 = handle.evaluate(win, opt)
        opt.precision = 1
    return dense_first_step(win, opt, blocks, lambda w: handle.evaluate(w, opt), oracle, fp64_blocks=fp64, **kw)


def cuda_first_step(handle, oracle, name):
    """(the dense step of a CUDA case from kba_eval's blocks, the kba_solve_batch results of its copies, tolerance class)"""
    window, precision, copies, _ = CUDA_CASES[name]
    win, opt = build(window)
    opt.precision = precision
    ref = cuda_reference(handle, oracle, win, opt)
    results = handle.solve_batch([win] * copies, opt, iterations_capacity=256)
    return ref, results, WINDOWS[window][1]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CUDA_CASES))
def test_cuda_first_step_matches_dense_step(handle, oracle, driver, name):  # noqa: F811
    """the CUDA pass chain of one LM iteration without the oracle's solver: blocks from kba_eval, the step from the dense
    reference, records 0 and 1 of kba_solve_batch -- of every window of a batch of copies -- on the solver path the window
    selects (asserted here, in the same run)"""
    window, _, copies, path = CUDA_CASES[name]
    assert_path(driver, [build(window)[0]] * copies, dict(WINDOWS[window][3], **path))
    ref, results, tol = cuda_first_step(handle, oracle, name)
    for i, res in enumerate(results):
        assert res.c.status == 0
        _check_first_step(res, ref, TOL[tol], "%s, window %d" % (name, i))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["config2_slice", "config3_kf30_lm600"])
def test_cuda_fp32_step_is_the_mixed_system(handle, oracle, name):
    """the tight classes tell the FP32 solve's system from a near one, on the fused and on the large-window path: the mixed
    reference holds, and each of these fails -- the reference of one Jacobian, its pose rows from the FP32 blocks too; the
    mixed reference with one FP32 landmark Jacobian row, or one FP32 residual, off by 1e-6"""
    win, opt = build(name)
    opt.precision = 1
    tol = TOL[WINDOWS[name][1]]
    [res] = handle.solve_batch([win], opt, iterations_capacity=256)
    assert res.c.status == 0
    _check_first_step(res, cuda_reference(handle, oracle, win, opt), tol, name)
    with pytest.raises(AssertionError):
        _check_first_step(res, cuda_reference(handle, oracle, win, opt, fp32_pose_rows=True), tol, name + ", FP32 pose rows")
    b32 = handle.evaluate(win, opt)
    opt.precision = 0
    b64 = handle.evaluate(win, opt)
    opt.precision = 1
    for what in ("jl", "r"):
        ref = dense_first_step(win, opt, tampered(b32, what), lambda w: handle.evaluate(w, opt), oracle, fp64_blocks=b64)
        with pytest.raises(AssertionError):
            _check_first_step(res, ref, tol, "%s, %s perturbed" % (name, what))
