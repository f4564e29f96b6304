"""The solver on windows far from the origin, where limo's global coordinates put them after a long drive.

tests/far_windows.py moves a window's origin by a rigid transform (yaw 2.1 rad, offsets of 1, 5 and 10 km): the same problem,
its residuals invariant in exact arithmetic.  What changes with the distance:
  - rounding: FP64 rounding of a 10 km coordinate is 2e-12 m, and the FP32 observation blocks (kba_options.precision = 1)
    would round kilometre-sized rotated points and translations before they cancel to a camera-frame point of a few metres
    (k_eval_obs<float> evaluates them relative to an anchor in the window for that reason);
  - conditioning: the pose parametrisation rotates about the origin, so a pose's rotation columns (-2 m x a, a = R p) grow with
    the distance and become almost collinear with its translation columns, and the parameter tolerance compares the step with
    an |x| that now holds kilometre-sized coordinates.  The Levenberg-Marquardt trajectory changes with the distance even in
    exact arithmetic (config1's second inner solve takes 9, 15 and 26 iterations at 0, 1 and 10 km).

The CPU half pins the helper (residuals, costs, Jacobians and the trimming decisions are invariant; a transform with a field left
out is not) and the oracle's first step to the dense extended-precision step of tests/test_first_step_dense.py.  The GPU half
holds the CUDA path to the same dense step and to the oracle's iteration log, checks that far and origin-centred windows share a
batch without leaking into each other, runs the >640-row and sharded paths on a far window, and holds the FP32 mode to the FP64
solve at BASELINE.md section 3's tolerance.

Final states are compared by keyframe centre (origin <- keyframe translation), rotation angle and landmark position: each is a
distance or an angle, so its deviation does not depend on where the origin is.  A keyframe pose's translation (keyframe <-
origin) does: it is -R c, and a rotation error of e rad moves it by e times the distance to the origin.
"""
from types import SimpleNamespace

import numpy as np
import pytest

from limo_b200 import geometry as g
from tests import far_windows as fw
from tests import iter_log as il
from tests import test_first_step_dense as fs
from tests.test_launch_plan import driver  # noqa: F401  (the plan driver fixture)

DISTANCES = list(fw.DISTANCES)

# ---- invariance of the evaluation (CPU) -------------------------------------------------------------------------------------
# Oracle evaluate on far(win, G) against win, worst over the 14 windows of tests/test_first_step_dense.WINDOWS (CPU, FP64):
#   residual rows (px; depth rows m): 6.6e-11 at 1 km, 3.0e-10 at 5 km, 7.8e-10 at 10 km (config3_kf8), about linear in D --
#     the rounding of the moved coordinates, 2.2e-16 D, times f / z;
#   observation cost, relative: 2.4e-12 (motion_only_speed_prior at 10 km, 4.1e-13 .. 1.4e-12 elsewhere);
#   cost of the other rows (ground, scale, plane chain, speed prior), relative to the whole cost: 4e-14;
#   translation columns of J_pose and J_landmark R_G^T, relative to the largest entry: 4.0e-10 (gap_over_fixed_keyframe, 10 km);
#   trimming values (raw, unrobustified block norms, up to 1e4 px for the outliers), relative to max(value, 1): 9.8e-13 per
#     metre of distance (stereo_rig; 9.8e-9 at 10 km), the decisions equal on every window.
RESIDUAL_PER_METRE = 2e-13     # px (or m) of residual per metre of distance: 2e-9 px at 10 km, 2.6 times the worst
TRIM_PER_METRE = 3e-12         # relative: 3 times the worst
COST_TOL = 1e-11               # relative: 4 times the worst
JACOBIAN_TOL = 2e-9            # relative to the largest entry: 5 times the worst


def _other_cost(win, opt, orc):
    """cost of the residual blocks besides the observations (ground points, scale, plane chain, speed prior)"""
    L = fs.program_columns(win)
    return float(fs.other_rows(win, opt, orc, L, win.kf_pose, fs._planes(win), win.lm_pos)[1])


def trimming(win, opt, orc):
    """the first trimming round at the window's state: per landmark the largest raw reprojection norm and the largest |depth
    residual| over its observations (-1 without one), and TrimmerQuantile's decisions on each group"""
    lm_of = np.repeat(np.arange(win.n_lm), np.diff(np.asarray(win.lm_obs_ptr)))
    cams = np.zeros(win.n_obs, dtype=int) if win.obs_cam is None else np.asarray(win.obs_cam)
    tr, td = np.full(win.n_lm, -1.0), np.full(win.n_lm, -1.0)
    for o in range(win.n_obs):
        k, c, j = win.obs_kf[o], cams[o], lm_of[o]
        ok, r2, _, _ = orc.reprojection(win.kf_pose[k], win.cam_pose[c], win.cam_intr[c], win.lm_pos[j], win.obs_u[o],
                                        win.obs_v[o], jac=False)
        if not ok:
            continue
        tr[j] = max(tr[j], np.hypot(r2[0], r2[1]))
        if win.obs_d[o] > 0:
            td[j] = max(td[j], abs(orc.depth(win.kf_pose[k], win.cam_pose[c], win.lm_pos[j], win.obs_d[o])[0][0]))
    rejected = []
    for vals, q in ((tr, opt.reprojection_quantile), (td, opt.depth_quantile)):
        rej, has = np.zeros(win.n_lm, bool), vals >= 0
        if has.sum() and has.sum() >= opt.min_residual_groups:
            rej[has] = orc.trimmer_quantile(vals[has], q)[1]
        rejected.append(rej)
    return tr, td, rejected[0], rejected[1]


def check_invariance(win, moved, G, D, opt, orc, label):
    """everything the window's first evaluation yields, on the moved copy against the window (see the constants above)"""
    r0, jp0, jl0, c0, f0 = orc.evaluate(win, opt)
    r1, jp1, jl1, c1, f1 = orc.evaluate(moved, opt)
    assert f1 == f0, label
    assert np.abs(r1 - r0).max() <= RESIDUAL_PER_METRE * D, (label, "residual", np.abs(r1 - r0).max())
    if f0:
        return
    o0, o1 = _other_cost(win, opt, orc), _other_cost(moved, opt, orc)
    assert abs(c1 - c0) <= COST_TOL * c0, (label, "observation cost", c1, c0)
    assert abs(o1 - o0) <= COST_TOL * (c0 + o0), (label, "cost of the other rows", o1, o0)
    scale = np.abs(jp0).max()
    assert np.abs(jp1[..., 3:] - jp0[..., 3:]).max() <= JACOBIAN_TOL * scale, (label, "J_pose translation columns")
    assert np.abs(jl1 - jl0 @ G[:3, :3].T).max() <= JACOBIAN_TOL * np.abs(jl0).max(), (label, "J_landmark")
    t0, t1 = trimming(win, opt, orc), trimming(moved, opt, orc)
    for a, b in zip(t0[:2], t1[:2]):
        dev = (np.abs(a - b) / np.maximum(np.abs(a), 1.0)).max()
        assert np.array_equal(a < 0, b < 0) and dev <= TRIM_PER_METRE * D, (label, "trimming values", dev)
    assert np.array_equal(t0[2], t1[2]) and np.array_equal(t0[3], t1[3]), (label, "trimming decisions")


@pytest.mark.parametrize("dist", DISTANCES)
@pytest.mark.parametrize("name", list(fs.WINDOWS))
def test_far_window_evaluates_as_the_window(oracle, name, dist):
    """residuals to a bound that grows with the distance, costs to 1e-11, the first trimming round equal, on every window of the
    dense-step set (fused and large-window shapes, plane rows and plane chain, stereo cameras, the speed prior)"""
    win, opt = fs.build(name)
    G = fw.transform(fw.DISTANCES[dist])
    moved = fw.far(win, G)
    assert fw.centre_distance(moved) == pytest.approx(fw.DISTANCES[dist], rel=0.02)
    check_invariance(win, moved, G, fw.DISTANCES[dist], opt, oracle, "%s at %s" % (name, dist))


@pytest.mark.parametrize("name, field", [("motion_only_speed_prior", "speed_T_origin_before"),
                                         ("config3_kf8", "lm_pos"), ("config1", "kf_pose")])
def test_far_window_with_a_field_left_out_is_another_problem(oracle, name, field):
    """the invariance check can fail: a transform that leaves one moved field where it was changes the problem (the speed prior
    alone, for speed_T_origin_before: its residual rows are the only ones that read it)"""
    win, opt = fs.build(name)
    D = fw.DISTANCES["1km"]
    G = fw.transform(D)
    check_invariance(win, fw.far(win, G), G, D, opt, oracle, name)
    with pytest.raises(AssertionError):
        check_invariance(win, fw.far(win, G, skip=(field,)), G, D, opt, oracle, name + " without " + field)


def test_far_window_keeps_every_field_it_does_not_move():
    """far() copies every field of Window; the ones local to a keyframe, a camera or an observation are unchanged"""
    for name in ("config3_kf8", "motion_only_speed_prior"):
        win = fs.build(name)[0]
        moved = fw.far(win, fw.transform(5e3))
        for f in fs.ew.WINDOW_FIELDS:
            a, b = getattr(win, f), getattr(moved, f)
            if f in ("kf_pose", "lm_pos", "speed_T_origin_before"):
                continue
            assert (a is None and b is None) or np.array_equal(np.asarray(a), np.asarray(b)), f
        # and back: the moved poses and landmarks are the window's, in the new frame
        assert np.abs(fw.back(moved.kf_pose, fw.transform(5e3), "pose")[:, 4:] - win.kf_pose[:, 4:]).max() <= 1e-11
        assert np.abs(fw.back(moved.lm_pos, fw.transform(5e3), "lm") - win.lm_pos).max() <= 1e-11


# ---- the oracle's first step against the dense step (CPU) -------------------------------------------------------------------
# Worst deviation from the dense extended-precision step over the windows of tests/test_first_step_dense.WINDOWS, oracle (CPU):
#               plane-free                                      ground
#   origin      2.4e-12 step_norm (ragged)                      8.0e-13 step_norm (config3_kf14)
#   1 km        1.8e-11 step_norm (config2_slice)               2.0e-12 step_norm (config3_kf14)
#   5 km        1.4e-12 relative_decrease (ragged)              1.0e-12 relative_decrease (config3_kf8)
#   10 km       5.4e-12 relative_decrease (ragged)              3.4e-12 relative_decrease (config3_kf8)
# Far windows are worse conditioned, but the first step does not grow with the distance: it stays inside the existing classes
# (STEP_TOL 1e-10 is 5.5 times the worst plane-free figure, GROUND_TOL 1e-11 three times the worst ground one).  No tolerance
# test fires on a first step: at 10 km the parameter tolerance's threshold is 1e-8 |x| with |x| near 1e4 sqrt(n_landmarks).
def far_case(name, dist):
    """(moved window, options, transform) of a window of tests/test_first_step_dense.WINDOWS"""
    win, opt = fs.build(name)
    G = fw.transform(fw.DISTANCES[dist])
    return fw.far(win, G), opt, G


@pytest.mark.parametrize("dist", DISTANCES)
@pytest.mark.parametrize("name", list(fs.WINDOWS))
def test_oracle_first_step_far_matches_dense_step(oracle, name, dist):
    _, tol, columns, _ = fs.WINDOWS[name]
    win, opt, _ = far_case(name, dist)
    ref = fs.dense_first_step(win, opt, oracle.evaluate(win, opt), lambda w: oracle.evaluate(w, opt), oracle)
    assert ref.successful and ref.n_columns == columns
    fs._check_first_step(oracle.solve_window(win, opt), ref, fs.TOL[tol], "%s at %s" % (name, dist))


@pytest.mark.parametrize("dist", ["10km"])
def test_far_dense_step_notices_a_wrong_block(oracle, dist):
    """the far first-step check can fail: config1 at 10 km with the landmark Jacobian of one observation off by 1e-6"""
    win, opt, _ = far_case("config1", dist)
    r, jp, jl, cost, failed = oracle.evaluate(win, opt)
    res = oracle.solve_window(win, opt)
    fs._check_first_step(res, fs.dense_first_step(win, opt, (r, jp, jl, cost, failed), oracle.evaluate, oracle), fs.STEP_TOL,
                         "as it is")
    jl = jl.copy()
    jl[5] *= 1 + 1e-6
    ref = fs.dense_first_step(win, opt, (r, jp, jl, cost, failed), oracle.evaluate, oracle)
    with pytest.raises(AssertionError):
        fs._check_first_step(res, ref, fs.STEP_TOL, "perturbed")


# ---- GPU ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


# Worst deviation from the dense step of the CUDA first step far (every window of each batch), measured on an NVIDIA H100 80GB
# HBM3 (power limit 700 W): plane-free 2.2e-12 (stereo_rig, 10 km), ground 2.9e-12 (config3_kf8, 10 km), the p_split = 1
# batches 1.2e-12 (config2_slice x 264, 1 km).  The FP32 cases against the mixed system of their solve (dense_first_step with
# the FP64 pose rows, scripts/fp32_agreement.py): plane-free 9.6e-13 (config5_kf40_lm700, 1 km), ground 2.5e-13
# (config3_kf30_lm600, 5 km).  The existing classes hold with the same margins as at the origin.
@pytest.mark.gpu
@pytest.mark.parametrize("dist", DISTANCES)
@pytest.mark.parametrize("name", list(fs.CUDA_CASES))
def test_cuda_first_step_far_matches_dense_step(handle, oracle, driver, name, dist):  # noqa: F811
    """tests/test_first_step_dense.CUDA_CASES moved far: blocks from kba_eval, the step from the dense reference, records 0 and
    1 of every window of the batch, on the path the window selects (the p_split = 1 batches of 264, 132 and 80 included)"""
    window, precision, copies, path = fs.CUDA_CASES[name]
    win, opt, _ = far_case(window, dist)
    fs.assert_path(driver, [win] * copies, dict(fs.WINDOWS[window][3], **path))
    opt.precision = precision
    ref = fs.cuda_reference(handle, oracle, win, opt)
    tol = fs.TOL[fs.WINDOWS[window][1]]
    for i, res in enumerate(handle.solve_batch([win] * copies, opt, iterations_capacity=256)):
        assert res.c.status == 0
        fs._check_first_step(res, ref, tol, "%s at %s, window %d" % (name, dist, i))


def _centres(kf_pose):
    return np.stack([g.iso_inv(g.pose_to_iso(p))[:3, 3] for p in kf_pose])


def _angles(a, b):
    """rotation angle between the keyframe rotations of two pose arrays"""
    return np.array([g.quaternion_angle(p, q) for p, q in zip(a, b)])


def final_deviation(a, b, n_lm):
    """final state of result a against result b: keyframe centres and rotation angles, landmark positions (frame-independent
    distances) and, for the record, the pose translations; final cost relative"""
    dl = np.linalg.norm(a.lm_pos[:n_lm] - b.lm_pos[:n_lm], axis=1)
    return dict(centre=float(np.linalg.norm(_centres(a.kf_pose) - _centres(b.kf_pose), axis=1).max()),
                rotation=float(_angles(a.kf_pose, b.kf_pose).max()),
                translation=float(np.linalg.norm(a.kf_pose[:, 4:] - b.kf_pose[:, 4:], axis=1).max()),
                lm_p95=float(np.percentile(dl, 95)) if n_lm else 0.0, lm_max=float(dl.max()) if n_lm else 0.0,
                cost=abs(a.c.final_cost - b.c.final_cost) / b.c.final_cost if b.c.final_cost > 0 else 0.0,
                lm_flipped=int((a.lm_rejected[:n_lm] != b.lm_rejected[:n_lm]).sum()))


def _decisions(res):
    return [(s.termination, s.num_iterations, s.num_successful_steps, s.num_landmarks) for s in res.solves]


# Whole solves, CUDA against oracle, far: every window of tests/test_iteration_log.CASES at each distance.  Measured on an NVIDIA
# H100 80GB HBM3 (power limit 700 W) by scripts/far_window_agreement.py:
#   head of the log (iterations 0 .. 2 of the first inner solve): cost 3.8e-11, gradient_max_norm 8.4e-10, step_norm 3.6e-11,
#     relative_decrease 5.8e-11 -- within iter_log.TOL["fp64_head"], held there;
#   flags of every record: equal; decisions (termination, iterations, accepted steps, landmarks of every inner solve): equal on
#     every plane-free window; on ground windows the count of rejected steps at radii near 1e15 differs by one (config3_kf8 at
#     10 km, config3_kf14 at 1 km, config3_full at 1 km), which the prefix rule of iter_log.log_deviations allows at the origin;
#   whole log, worst over the windows other than the three below: cost 5.0e-07 (config3_kf8, 10 km), gradient_max_norm 2.3e-02
#     (config3_kf8, 10 km), step_norm 9.1e-04 (stereo_rig, 1 km), relative_decrease 8.4e-05, trust_region_radius 2.1e-05
#     (short_tracks, 10 km).  At the origin the same windows stay within cost 1.2e-10; the growth is the conditioning's, not
#     the CUDA path's: the oracle against itself on 1 and 4 threads moves as much (short_tracks at 10 km: cost 3.5e-07,
#     gradient_max_norm 5.1e-02; config1_seed11 at 10 km: cost 1.8e-07 against the CUDA path's 1.8e-07).  FAR_LOG is about
#     10 times the worst;
#   final state: keyframe centres 7.0e-08 m, rotations 2.1e-09 rad, landmarks (95th percentile) 1.2e-07 m, final cost 1.2e-09
#     (config3_kf14, 5 km) -- within north_star's tolerances, held there.
# Three windows are held to their own measured drift (CONDITIONED), each beside the oracle against itself on 1 and 4 threads
# (8 and 3 for config3_full) at the same distance:
#   ragged (config1 without depth rows, landmarks seen once or not at all: the scale and those landmarks' rays are held by the
#     damping alone): CUDA vs oracle cost 1.1e-04, step_norm 8.9e-01, centres 6.6e-04 m (5 km), rotations 2.1e-07, landmarks
#     1.0e-02 m, final cost 1.4e-08; oracle vs oracle at 10 km: cost 5.5e-05, step_norm 8.2e-01, centres 3.9e-04 m, landmarks
#     6.2e-03 m, final cost 5.0e-09 (at the origin already 1.1e-06 m and 1.7e-05 m);
#   evaluation_failure (config1 without depth rows as well): landmarks 1.3e-05 m (1 km); oracle vs oracle 1.0e-05 m (10 km);
#   config3_full (ground, 300 rows): at 10 km cost 1.2e-03, relative_decrease 1.8e-01, step_norm 3.0e-02 in the records behind
#     the prefix, final cost 1.1e-05; oracle vs oracle cost 8.3e-04, relative_decrease 1.2e-01, final cost 7.8e-06.
TRANSLATION_TOL = 1e-6   # metres: north_star's FP64 tolerance, on keyframe centres and landmarks (95th percentile)
ROTATION_TOL = 1e-7      # rad, as test_gpu_parity._compare_solves holds quaternion entries
COST_REL_TOL = 1e-8
FAR_LOG = dict(cost=5e-6, cost_change=5e-6, gradient_max_norm=0.2, step_norm=1e-2, relative_decrease=1e-3,
               trust_region_radius=2e-4)
FINAL = dict(centre=TRANSLATION_TOL, rotation=ROTATION_TOL, lm_p95=TRANSLATION_TOL, cost=COST_REL_TOL)
# name -> (whole-log row, final-state bounds), each about 10 times the measured worst
CONDITIONED = {
    "ragged": (dict(cost=1e-3, cost_change=1e-3), dict(centre=1e-2, rotation=3e-6, lm_p95=1e-1, cost=2e-7)),
    "evaluation_failure": (FAR_LOG, dict(FINAL, lm_p95=1e-4)),
    "config3_full": (dict(cost=1e-2, cost_change=1e-2, gradient_max_norm=3e-4, trust_region_radius=3e-4), dict(FINAL, cost=1e-4)),
}


def measure_log(handle, oracle, name, dist):
    """(CUDA result, oracle result, options, prefix rule, transform, window) of one case of test_iteration_log moved far"""
    from tests import test_iteration_log as tl
    win0, opt, prefix, threads = tl.build_case(name)
    G = fw.transform(fw.DISTANCES[dist])
    win = fw.far(win0, G)
    rg = handle.solve_window(win, opt, iterations_capacity=tl.LOG_CAPACITY)
    rc = oracle.solve_window(win, opt, num_threads=threads, iterations_capacity=tl.LOG_CAPACITY)
    return SimpleNamespace(rg=rg, rc=rc, opt=opt, prefix=prefix, G=G, win=win)


LOG_CASES = ["config1", "config1_seed11", "config2_full", "free_keyframes_30", "gap_over_fixed_keyframe", "stereo_rig", "ragged",
             "short_tracks", "config3_kf8", "config3_kf14", "config3_full", "config5_kf40", "motion_only",
             "motion_only_speed_prior", "evaluation_failure", "tiny", "all_keyframes_fixed"]


@pytest.mark.gpu
@pytest.mark.parametrize("dist", DISTANCES)
@pytest.mark.parametrize("name", LOG_CASES)
def test_far_iteration_log_matches_oracle(handle, oracle, name, dist):
    """every record of the CUDA log of a far window against the oracle's: the flags exactly, the head at the sharp FP64 row,
    every record at FAR_LOG; the same decisions (termination, iteration counts and trimming rejections) and the final state at
    north_star's tolerances -- the three windows of CONDITIONED at their own"""
    m = measure_log(handle, oracle, name, dist)
    label = "%s at %s" % (name, dist)
    log_tol, final_tol = CONDITIONED.get(name, (FAR_LOG, FINAL))
    assert m.rg.c.status == 0
    il.check_log_invariants(m.rc, m.opt, label + " (oracle)")
    il.check_log_invariants(m.rg, m.opt, label + " (cuda)")
    assert [s.termination for s in m.rg.solves] == [s.termination for s in m.rc.solves], label
    il.compare_logs(m.rg, m.rc, il.TOL["fp64_head"], prefix_rule=m.prefix, label=label, head=True)
    il.compare_logs(m.rg, m.rc, log_tol, prefix_rule=m.prefix, label=label)
    if not m.prefix:
        assert _decisions(m.rg) == _decisions(m.rc), label
    dev = final_deviation(m.rg, m.rc, m.win.n_lm)
    assert dev["lm_flipped"] == 0, (label, dev)
    for k, limit in final_tol.items():
        assert dev[k] <= limit, (label, k, dev)


def _bit_equal(a, b, n_lm, label):
    assert a.c.status == 0 and b.c.status == 0, label
    assert [(s.num_iterations, s.num_successful_steps, s.termination, s.final_cost) for s in a.solves] == \
        [(s.num_iterations, s.num_successful_steps, s.termination, s.final_cost) for s in b.solves], label
    assert np.array_equal(a.kf_pose, b.kf_pose) and np.array_equal(a.kf_plane, b.kf_plane), label
    assert np.array_equal(a.lm_pos[:n_lm], b.lm_pos[:n_lm]), label
    assert np.array_equal(a.lm_rejected[:n_lm], b.lm_rejected[:n_lm]), label


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("name", ["config2_slice", "config3_kf14"])
def test_far_and_origin_windows_share_a_batch(handle, name, precision):
    """one batch of the window at the origin and at 1, 5 and 10 km: each window equals the same slot of a batch of four copies
    of itself bit for bit (same shapes, so the same launch plan), so nothing of one window's coordinates leaks into another's"""
    win, opt = fs.build(name)
    opt.precision = precision
    wins = [win] + [fw.far(win, fw.transform(fw.DISTANCES[d])) for d in DISTANCES]
    mixed = handle.solve_batch(wins, opt)
    for i, w in enumerate(wins):
        alone = handle.solve_batch([w] * len(wins), opt)[i]
        _bit_equal(mixed[i], alone, w.n_lm, "%s, precision %d, slot %d" % (name, precision, i))


@pytest.mark.gpu
def test_far_large_window_matches_oracle(handle, oracle, driver):  # noqa: F811
    """the 1001-row ground window of tests/test_large_reduced_rows.py at 5 km: the >640-row factorisation (k_chol_trail_band)
    against the oracle, and the sharded solve with one rank bit for bit the plain one"""
    from limo_b200 import parallel
    from tests import test_large_reduced_rows as lr
    w = fw.far(lr.WINDOWS["ground_kf100"][0](), fw.transform(fw.DISTANCES["5km"]))
    assert fs.plan_shape(w)[0] == 1001
    fs.assert_path(driver, [w], dict(fused=0, solve_tiled=0, solve_split=32))
    opt = lr._opt(oracle)
    rg = handle.solve_window(w, opt, iterations_capacity=lr.LOG_CAPACITY)
    rc = oracle.solve_window(w, opt, num_threads=32, iterations_capacity=lr.LOG_CAPACITY)
    il.check_log_invariants(rg, opt, "ground_kf100 at 5km (cuda)")
    assert [s.termination for s in rg.solves] == [s.termination for s in rc.solves]
    il.compare_logs(rg, rc, il.TOL["fp64_head"], prefix_rule=True, label="ground_kf100 at 5km", head=True)
    dev = final_deviation(rg, rc, w.n_lm)
    assert dev["lm_flipped"] == 0 and dev["centre"] <= TRANSLATION_TOL and dev["cost"] <= COST_REL_TOL, dev
    assert np.abs(rg.kf_plane - rc.kf_plane).max() <= 1e-3
    rp = handle.solve_window(w)
    [(r1, j0, j1)] = parallel.solve_sharded_local(w, 1)
    assert (j0, j1) == (0, w.n_lm)
    _bit_equal(r1, rp, w.n_lm, "sharded, one rank")


# ---- FP32 blocks against FP64 (GPU) ---------------------------------------------------------------------------------------
# k_eval_obs<float> rounds p - c and t + R c (c: the anchor below), so the camera-frame point x = R (p - c) + (t + R c) and with
# it m = d r / d x (the translation columns of J_p), J_l = m R and r carry errors of FP32 rounding times those anchored
# magnitudes, which do not grow with the distance: each family is held relative to its own largest entry in the window.  The
# rotation columns -2 m x a carry the lever arm a = R p = R (p - c) + R c, whose size is the distance: their error is held
# relative to S (|R p| + |p - c| + |t + R c|) per observation, S the window's largest translation-column entry.  Worst over
# config2_slice (fused: J_l formed from the FP32 J_p in FP64) and config3_kf30_lm600 (large-window: J_l stored in FP32) at the
# origin and at 1, 5 and 10 km, measured on an NVIDIA H100 80GB HBM3 (power limit 700 W) by scripts/fp32_agreement.py:
#                              origin     1 km       5 km       10 km      (translation, J_l, r, rotation)
#   config2_slice              8.7e-06    3.7e-05    8.0e-05    2.2e-05    J_l as translation; r 7.6e-05 .. 2.3e-04; rotation
#   config3_kf30_lm600         1.1e-05    1.1e-05    1.5e-05    1.7e-05    6.8e-06 .. 1.4e-04 (config2_slice, 5 km)
# The anchored magnitudes are the same at every distance (|p - c| + |t + R c| at most 230 .. 280 m on config2_slice, 350 .. 440 m
# on config3_kf30_lm600); what moves the figures is the rounding of R itself: the far windows are yawed by 2.1 rad, and their
# rotations have no entries that FP32 holds exactly.  Each bound is about three times its family's worst.  The kernels from
# before the anchor, on the same windows at 1 km: translation 1.1e-03 and 4.5e-04, J_l 1.1e-03 and 5.1e-04, r 3.5e-03 and
# 2.2e-03, rotation 1.9e-03 and 7.4e-04 (config2_slice, config3_kf30_lm600) -- every family of both windows fails there.
FP32_BLOCK_TOL = dict(translation=2.5e-4, landmark=2.5e-4, residual=7e-4, rotation=4e-4)


def fp32_anchor(win):
    """the anchor c of k_eval_obs<float>: keyframe 0's centre -R_0^T t_0 on the 64 m grid"""
    T = g.pose_to_iso(win.kf_pose[0])
    return 64.0 * np.rint(-(T[:3, :3].T @ T[:3, 3]) / 64.0)


def fp32_block_deviation(win, b32, b64):
    """per column family, the largest deviation of the FP32 blocks (r, J_p, J_l) from the FP64 ones in the units above"""
    r32, jp32, jl32 = (np.asarray(a) for a in b32[:3])
    r64, jp64, jl64 = (np.asarray(a) for a in b64[:3])
    S = np.abs(jp64[..., 3:]).max()
    c = fp32_anchor(win)
    isos = np.stack([g.pose_to_iso(p) for p in win.kf_pose])
    R, t = isos[win.obs_kf, :3, :3], isos[win.obs_kf, :3, 3]
    p = np.repeat(win.lm_pos, np.diff(np.asarray(win.lm_obs_ptr)), axis=0)
    arm = (np.linalg.norm(np.einsum("oij,oj->oi", R, p), axis=1) + np.linalg.norm(p - c, axis=1)
           + np.linalg.norm(t + R @ c, axis=1))
    return dict(translation=np.abs(jp32[..., 3:] - jp64[..., 3:]).max() / S,
                landmark=np.abs(jl32 - jl64).max() / np.abs(jl64).max(),
                residual=np.abs(r32 - r64).max() / np.abs(r64).max(),
                rotation=(np.abs(jp32[..., :3] - jp64[..., :3]).max(axis=(1, 2)) / (S * arm)).max())


def check_fp32_blocks(win, b32, b64, label):
    dev = fp32_block_deviation(win, b32, b64)
    assert all(dev[k] <= FP32_BLOCK_TOL[k] for k in dev), (label, dev)
    assert np.abs(np.asarray(b32[1]) - np.asarray(b64[1])).max() > 0.0, label  # ... and it really is the FP32 path
    return dev


@pytest.mark.gpu
@pytest.mark.parametrize("dist", ["0"] + DISTANCES)
@pytest.mark.parametrize("name", ["config2_slice", "config3_kf30_lm600"])
def test_fp32_blocks_match_fp64_blocks(handle, name, dist):
    """kba_eval at precision 1 against precision 0, the window at the origin and far, every column family at FP32_BLOCK_TOL: the
    fused path's blocks (k_eval_obs<float, false>, J_l formed in FP64) and the large-window path's (k_eval_obs<float, true>)"""
    win, opt = fs.build(name)
    if dist != "0":
        win = far_case(name, dist)[0]
    b64 = handle.evaluate(win, opt)
    opt.precision = 1
    b32 = handle.evaluate(win, opt)
    assert b32[4] == 0 and b64[4] == 0 and b32[3] == pytest.approx(b64[3], rel=1e-12)  # the cost at x is FP64 either way
    check_fp32_blocks(win, b32, b64, "%s at %s" % (name, dist))


# ---- FP32 far (GPU) -------------------------------------------------------------------------------------------------------
# BASELINE.md section 3: pose translation <= 1e-2 m against the FP64 solve, final cost <= 1e-5 relative when the trimming rejects
# the same landmarks (else up to 0.5 % of the landmarks may flip, as in test_gpu_parity.test_fp32_linearisation_mode).  The
# translation is held on keyframe centres (see the module docstring: a pose translation carries the rotation error times the
# distance, 1.3e-05 rad x 10 km = 0.13 m).
# Without an anchor k_eval_obs<float> rounded R p and t, each as large as the distance, and FP32 missed the tolerance from 1 km
# on: config2_slice centres 5.3e-03 m at 1 km, 3.1e-02 m at 5 km, 0.23 m at 10 km, cost 4.1e-05 .. 0.14; config3_kf30_lm600
# 1.6e-01 m and cost 3.1e-02 at 5 km.  With the evaluation anchored at keyframe 0's centre on a 64 m grid, measured on an NVIDIA
# H100 80GB HBM3 (power limit 700 W), worst window (landmarks flipped: none in any case):
#                              origin               1 km                 5 km                 10 km
#   config2_slice              1.8e-04 m  6.4e-08   5.5e-04 m  3.3e-07   2.6e-04 m  1.1e-07   6.0e-04 m  6.2e-07
#   config3_kf30_lm600         9.0e-04 m  2.1e-07   5.0e-04 m  8.2e-07   1.8e-03 m  1.7e-06   1.1e-03 m  3.0e-06
#   config2_slice x 264        1.8e-04 m  6.4e-08   2.6e-04 m  9.1e-08   5.8e-04 m  2.7e-07   1.9e-04 m  8.4e-07
# (centres, final cost relative), rotations at most 2.2e-05 rad: the far windows sit where the origin-centred ones do, with a
# margin of 5.5 on the centres and 3.3 on the cost at the worst.  The first inner solve against the FP64 log: cost 2.6e-05,
# step_norm 1.4e-05 at the worst distance (3.0e-05 and 1.1e-05 at the origin), against iter_log.TOL["fp32_linearize"].
FP32_POSITION_TOL = 1e-2   # metres, on keyframe centres
FP32_ROTATION_TOL = 1e-4   # rad
FP32_COST_TOL = 1e-5
FP32_CASES = {"config2_slice": ("config2_slice", 1), "config3_kf30_lm600": ("config3_kf30_lm600", 1),
              "config2_slice_batch264": ("config2_slice", 264)}


def measure_fp32(handle, name, dist):
    """worst final_deviation of the FP32 solves of a case (every window of its batch) against the FP64 solve"""
    window, copies = FP32_CASES[name]
    win, opt, _ = far_case(window, dist) if dist != "0" else fs.build(window) + (None,)
    r64 = handle.solve_window(win, opt)
    opt.precision = 1
    out = None
    for res in handle.solve_batch([win] * copies, opt):
        assert res.c.status == 0 and res.c.num_solves == r64.c.num_solves
        dev = final_deviation(res, r64, win.n_lm)
        out = dev if out is None else {k: max(v, dev[k]) for k, v in out.items()}
    return out, win.n_lm


@pytest.mark.gpu
@pytest.mark.parametrize("dist", DISTANCES)
@pytest.mark.parametrize("name", list(FP32_CASES))
def test_fp32_far_meets_the_stated_tolerance(handle, name, dist):
    dev, n_lm = measure_fp32(handle, name, dist)
    label = "%s at %s" % (name, dist)
    assert dev["centre"] <= FP32_POSITION_TOL and dev["rotation"] <= FP32_ROTATION_TOL, (label, dev)
    assert dev["lm_flipped"] <= 0.005 * n_lm, (label, dev)
    if dev["lm_flipped"] == 0:
        assert dev["cost"] <= FP32_COST_TOL, (label, dev)


@pytest.mark.gpu
@pytest.mark.parametrize("dist", DISTANCES)
def test_fp32_far_first_inner_solve_log(handle, oracle, dist):
    """the first FP32 inner solve of config2_slice far against the oracle's FP64 log, at iter_log.TOL["fp32_linearize"]"""
    from tests import test_iteration_log as tl
    win, opt, _ = far_case("config2_slice", dist)
    rc = oracle.solve_window(win, opt, iterations_capacity=tl.LOG_CAPACITY)
    opt.precision = 1
    rg = handle.solve_window(win, opt, iterations_capacity=tl.LOG_CAPACITY)
    il.check_log_invariants(rg, opt, "fp32 at " + dist)
    il.compare_logs(rg, rc, il.TOL["fp32_linearize"], solves=(0,), label="fp32 at " + dist)
