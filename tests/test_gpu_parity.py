"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on identical inputs.

Tolerances are the ones BASELINE.json's north_star states for FP64: pose translation <= 1e-6 m and cost
relative <= 1e-8 against the reference solve (here: its restatement, see oracle/kba_oracle.h for what is pinned).
"""
import numpy as np
import pytest

from limo_b200 import geometry as g
from limo_b200 import synth
from tests import ref_scenes as rs

pytestmark = pytest.mark.gpu

TRANSLATION_TOL = 1e-6   # metres
COST_REL_TOL = 1e-8


@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


def _compare_solves(res_gpu, res_cpu, win, label="", iter_slack=0, lm_p95=1e-6, lm_max=0.1, lm_outliers=0):
    assert res_gpu.c.status == 0, label
    assert res_gpu.c.num_solves == res_cpu.c.num_solves, label
    for a, b in zip(res_gpu.solves, res_cpu.solves):
        assert a.termination == b.termination, (label, a.termination, b.termination)
        # iter_slack: with the ground-plane blocks the late iterations run at trust-region radii ~1e15 where the reduced
        # system is numerically singular; whether such a step is "invalid" (and retried at a smaller radius) is decided
        # at rounding level, so the count of UNSUCCESSFUL iterations may differ by a few while the accepted steps agree
        assert abs(a.num_iterations - b.num_iterations) <= iter_slack, (label, a.num_iterations, b.num_iterations)
        assert a.num_successful_steps == b.num_successful_steps, label
        assert a.num_landmarks == b.num_landmarks, label
        assert a.initial_cost == pytest.approx(b.initial_cost, rel=COST_REL_TOL), label
        assert a.final_cost == pytest.approx(b.final_cost, rel=COST_REL_TOL, abs=1e-14), label
    assert np.array_equal(res_gpu.lm_rejected[:win.n_lm], res_cpu.lm_rejected[:win.n_lm]), label
    dt = np.linalg.norm(res_gpu.kf_pose[:, 4:] - res_cpu.kf_pose[:, 4:], axis=1).max()
    dq = np.abs(res_gpu.kf_pose[:, :4] - res_cpu.kf_pose[:, :4]).max()
    dl = np.linalg.norm(res_gpu.lm_pos[:win.n_lm] - res_cpu.lm_pos[:win.n_lm], axis=1)
    assert dt <= TRANSLATION_TOL, (label, dt)
    assert dq <= 1e-7, (label, dq)
    # Landmarks seen twice with almost no parallax are nearly unobservable along the ray (condition ~1e10), so rounding
    # differences show up there first; north_star's tolerances are on poses and cost.  Typical landmarks agree to 1e-6.
    # lm_outliers: how many such landmarks may exceed lm_max (a 20 000-landmark window holds a few with condition > 1e14)
    assert np.percentile(dl, 95) <= lm_p95 and (dl > lm_max).sum() <= lm_outliers, (label, np.percentile(dl, 95), dl.max())


def test_eval_matches_oracle(handle, oracle):
    """residual / Jacobian kernel vs the oracle's Evaluate on the 5-keyframe config and on a slice of config 2"""
    for win in (synth.make_window(1), synth.make_window(2, n_kf=12, n_lm=400, n_obs=3000)):
        r, jp, jl, cost, failed = handle.evaluate(win)
        r0, jp0, jl0, cost0, failed0 = oracle.evaluate(win)
        assert failed == failed0 == 0
        assert cost == pytest.approx(cost0, rel=1e-12)
        assert np.allclose(r, r0, rtol=1e-11, atol=1e-11)
        assert np.allclose(jp, jp0, rtol=1e-10, atol=1e-9 * np.abs(jp0).max())
        assert np.allclose(jl, jl0, rtol=1e-10, atol=1e-9 * np.abs(jl0).max())
        assert np.all(jp[win.obs_kf == 0] == 0.0)  # fixed keyframe: no pose columns


@pytest.mark.parametrize("extr", ["mono", "stereo"])
@pytest.mark.parametrize("case", [0, 1, 2])
@pytest.mark.parametrize("depth", [False, True])
def test_reference_scenes_on_gpu(handle, oracle, extr, case, depth):
    """KeyFrameBundleAdjustment.solve / solve_depth of the reference, run through the CUDA path: must satisfy the
    reference's own acceptance threshold AND agree with the oracle."""
    from tests.test_oracle_reference_tests import SOLVE_CASES
    noise_lms, noise_poses, thres = SOLVE_CASES[case]
    if depth:
        noise_lms = noise_lms + (0.0,)
        ex = [np.eye(4)] if extr == "mono" else rs.stereo_extrinsics()
    else:
        ex = [rs.mono_extrinsics()] if extr == "mono" else rs.stereo_extrinsics()
    bg, poses_gt, *_ = rs.build_adjuster(handle, noise_lms, noise_poses, ex, with_depth=depth)
    bc, *_ = rs.build_adjuster(oracle.OracleBackend(), noise_lms, noise_poses, ex, with_depth=depth)
    bg.solve()
    bc.solve()
    for ts in sorted(bg.keyframes_):
        assert g.is_approx(bg.keyframes_[ts].getEigenPose(), poses_gt[ts], thres)
    _compare_solves(bg.last_result, bc.last_result, bg.last_window, "%s case %d depth %s" % (extr, case, depth))


@pytest.mark.parametrize("config,seed", [(1, None), (1, 11), (1, 12)])
def test_config1_solve_matches_oracle(handle, oracle, config, seed):
    """BASELINE config 1 (5 keyframes / 200 landmarks, mono): trimmed solve, GPU vs oracle"""
    win = synth.make_window(config, seed=seed)
    rg = handle.solve_window(win)
    rc = oracle.solve_window(win)
    _compare_solves(rg, rc, win, "config1 seed %s" % seed)


def test_config2_solve_matches_oracle(handle, oracle):
    """BASELINE config 2 (30 keyframes / 3k landmarks / 40k observations, mono + lidar depth, FP64)"""
    win = synth.make_window(2)
    rg = handle.solve_window(win)
    rc = oracle.solve_window(win, num_threads=8)
    _compare_solves(rg, rc, win, "config2")


@pytest.mark.parametrize("shape", [dict(n_kf=8, n_lm=300, n_obs=1800, gp_frac=0.2), dict(n_kf=14, n_lm=500, n_obs=4500),
                                   dict()])
def test_config3_ground_plane_matches_oracle(handle, oracle, shape):
    """BASELINE config 3 in FP64: ground-plane height residuals (Huber), plane normal / distance blocks with the
    FixScaleVectorPlus parameterisation, the regularisation chain (cpp:769-818) and trimming, GPU vs oracle"""
    win = synth.make_window(3, seed=41, **shape)
    assert win.n_gp > 0 and win.plane_reg_weight == 10.0
    rg = handle.solve_window(win)
    rc = oracle.solve_window(win, num_threads=8 if not shape else 1)
    _compare_solves(rg, rc, win, "config3 %s" % shape, iter_slack=3)
    # plane blocks are the flattest directions of the problem (a handful of ground points per keyframe): rounding
    # differences are amplified there first; poses and costs above are held to north_star's tolerances
    assert np.abs(rg.kf_plane - rc.kf_plane).max() <= 1e-3
    assert np.allclose(np.linalg.norm(rg.kf_plane[:, :3], axis=1), 1.0, atol=1e-12)  # normals stay on the sphere


def test_stereo_rig_same_landmark_in_both_cameras(handle, oracle):
    """a landmark observed by BOTH cameras of the rig in the same keyframe: two residual blocks share the pose and the
    landmark block, their Schur contributions must be summed (oracle: segments keyed by parameter block)"""
    from limo_b200.capi_types import Window
    win, truth = synth.make_window(2, n_kf=8, n_lm=250, n_obs=1500, seed=77, return_truth=True)
    T0 = g.pose_to_iso(win.cam_pose[0])
    T1 = g.iso(t=[-0.54, 0.0, 0.0]) @ T0   # second camera 0.54 m to the right of the first (KITTI stereo baseline)
    rng = np.random.default_rng(5)
    lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
    okf, ocam, ou, ov, od, ptr = [], [], [], [], [], [0]
    for j in range(win.n_lm):
        for o in range(win.lm_obs_ptr[j], win.lm_obs_ptr[j + 1]):
            k = win.obs_kf[o]
            okf.append(k); ocam.append(0); ou.append(win.obs_u[o]); ov.append(win.obs_v[o]); od.append(win.obs_d[o])
            pc = g.apply(T1 @ g.pose_to_iso(truth["kf_pose"][k]), truth["lm_pos"][j])
            if pc[2] > 0.5 and j % 3 != 0:  # two thirds of the landmarks are also seen by camera 1
                okf.append(k); ocam.append(1)
                ou.append(synth.F * pc[0] / pc[2] + synth.CX + rng.normal(0, 0.5))
                ov.append(synth.F * pc[1] / pc[2] + synth.CY + rng.normal(0, 0.5)); od.append(-1.0)
        ptr.append(len(okf))
    w2 = Window(kf_pose=win.kf_pose, kf_fixed=win.kf_fixed, cam_intr=[win.cam_intr[0]] * 2,
                cam_pose=[win.cam_pose[0], g.iso_to_pose(T1)], lm_pos=win.lm_pos, lm_weight=win.lm_weight, lm_obs_ptr=ptr,
                obs_kf=okf, obs_cam=ocam, obs_u=ou, obs_v=ov, obs_d=od, scale_kf0=0, scale_kf1=1,
                scale_weight=win.scale_weight, scale_value=win.scale_value)
    assert w2.n_obs > win.n_obs
    _compare_solves(handle.solve_window(w2), oracle.solve_window(w2), w2, "stereo duplicates")


def _motion_only_window(seed, with_prior):
    """one frame of a config-2 scene against fixed landmarks = the problem adjustPoseOnly() builds (cpp:820-888)"""
    from limo_b200.capi_types import Window
    win, truth = synth.make_window(2, n_kf=12, n_lm=600, n_obs=5000, seed=seed, return_truth=True)
    k = win.n_kf - 1
    sel = win.obs_kf == k
    lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
    lms = lm_of_obs[sel]
    args = dict(kf_pose=win.kf_pose[k:k + 1], kf_fixed=[0], cam_intr=win.cam_intr, cam_pose=win.cam_pose,
                lm_pos=truth["lm_pos"][lms], lm_weight=np.ones(len(lms)), lm_obs_ptr=np.arange(len(lms) + 1),
                obs_kf=np.zeros(len(lms), dtype=np.int32), obs_u=win.obs_u[sel], obs_v=win.obs_v[sel],
                obs_d=win.obs_d[sel], landmarks_fixed=True)
    if with_prior:
        Tb, Tb2 = g.pose_to_iso(truth["kf_pose"][k - 1]), g.pose_to_iso(truth["kf_pose"][k - 2])
        args.update(speed_kf=0, speed_weight=0.7, speed_dt=0.1, speed_v_before=(Tb @ g.iso_inv(Tb2))[:3, 3] / 0.1,
                    speed_T_origin_before=g.iso_to_pose(g.iso_inv(Tb)))
    return Window(**args), truth["kf_pose"][k]


@pytest.mark.parametrize("with_prior", [False, True])
def test_motion_only_matches_oracle(handle, oracle, with_prior):
    """adjustPoseOnly(): landmarks constant, one free pose, optional SpeedRegularizationVector2 prior, trimming rounds"""
    win, pose_true = _motion_only_window(31, with_prior)
    opt = handle.default_options()
    opt.min_landmarks_for_trimming = 30
    rg = handle.solve_window(win, opt)
    rc = oracle.solve_window(win, opt)
    _compare_solves(rg, rc, win, "motion only prior=%s" % with_prior)
    assert np.array_equal(rg.lm_pos[:win.n_lm], win.lm_pos)  # constant blocks stay untouched
    if not with_prior:
        assert np.linalg.norm(rg.kf_pose[0, 4:] - pose_true[4:]) < 0.05


def test_reference_adjust_motion_only_on_gpu(handle, oracle):
    """BundleAdjusterKeyframes.adjustMotionOnly (reference test :1340-1344) through the CUDA path"""
    from limo_b200.adjuster import Keyframe
    out = []
    for backend in (handle, oracle.OracleBackend()):
        b, poses_gt, noisy, lms, ts, cameras, l2c = rs.build_adjuster(
            backend, (0, 0, 0), (0, 0, 0, 0), [np.eye(4)], with_depth=True, motion_only=True)
        kf = Keyframe(4, ts, b.keyframes_[0].cameras_[0], noisy[4])
        b.landmark_selector_.select(b.getActiveLandmarkConstPtrs(), b.getActiveKeyframeConstPtrs())
        b.adjustPoseOnly(kf)
        assert g.is_approx(kf.getEigenPose(), poses_gt[4], 0.5)
        out.append((b.last_result, b.last_window))
    _compare_solves(out[0][0], out[1][0], out[0][1], "adjustMotionOnly")


def test_batch_equals_single(handle, monkeypatch):
    """Deterministic reductions: with the number of CTAs a window's Schur sum is split over pinned (KBA_P_SPLIT, read
    when a batch is created), a batch of different windows gives bit-identical results to solving them one by one.
    With the default split (which follows the batch size: one window alone is spread over the whole GPU) only the
    association of that one sum differs, so the results agree to rounding."""
    wins = [synth.make_window(1, seed=s) for s in (21, 22, 23)] + [synth.make_window(2, n_kf=10, n_lm=300, n_obs=2500, seed=5)]
    monkeypatch.setenv("KBA_P_SPLIT", "6")
    single = [handle.solve_window(w) for w in wins]
    batch = handle.solve_batch(wins)
    for s, b, w in zip(single, batch, wins):
        assert np.array_equal(s.kf_pose, b.kf_pose)
        assert np.array_equal(s.lm_pos[:w.n_lm], b.lm_pos[:w.n_lm])
        assert s.c.final_cost == b.c.final_cost
    monkeypatch.delenv("KBA_P_SPLIT")
    single = [handle.solve_window(w) for w in wins]
    batch = handle.solve_batch(wins)
    for s, b, w in zip(single, batch, wins):
        assert [x.num_iterations for x in s.solves] == [x.num_iterations for x in b.solves]
        assert np.abs(s.kf_pose - b.kf_pose).max() <= 1e-9
        assert s.c.final_cost == pytest.approx(b.c.final_cost, rel=1e-10)


def test_strided_grids_are_bit_identical(handle, monkeypatch):
    """k_linearize / k_backsub_v with their CTAs striding over a window's units (KBA_LIN_GRID / KBA_BS_GRID, read when a batch is
    created; by default chosen from the batch size): every unit writes the same partial sums into the same slots whichever CTA
    runs it, so any grid gives bit-identical results -- here one CTA per unit against 1, 3 and 7 CTAs per window"""
    wins = [synth.make_window(1, seed=s) for s in (21, 22)] + [synth.make_window(2, n_kf=10, n_lm=300, n_obs=2500, seed=5),
                                                               synth.make_window(3, seed=41, n_kf=8, n_lm=300, n_obs=1800, gp_frac=0.2)]
    monkeypatch.setenv("KBA_LIN_GRID", "0")
    monkeypatch.setenv("KBA_BS_GRID", "0")
    ref = handle.solve_batch(wins)
    for lg, bg in (("1", "1"), ("3", "2"), ("7", "5"), ("-1", "-1")):
        monkeypatch.setenv("KBA_LIN_GRID", lg)
        monkeypatch.setenv("KBA_BS_GRID", bg)
        res = handle.solve_batch(wins)
        for a, b, w in zip(ref, res, wins):
            assert b.c.status == 0
            assert np.array_equal(a.kf_pose, b.kf_pose) and np.array_equal(a.kf_plane, b.kf_plane), (lg, bg)
            assert np.array_equal(a.lm_pos[:w.n_lm], b.lm_pos[:w.n_lm]), (lg, bg)
            assert np.array_equal(a.lm_rejected[:w.n_lm], b.lm_rejected[:w.n_lm])
            assert a.c.final_cost == b.c.final_cost
            assert [x.num_iterations for x in a.solves] == [x.num_iterations for x in b.solves]


def test_full_size_properties(handle):
    """size-independent properties at BASELINE config 2 scale: cost decreases, outputs finite, fixed keyframe untouched,
    rejected landmarks keep their position, repeat solve is bit-identical"""
    win = synth.make_window(2, seed=77)
    a = handle.solve_window(win)
    b = handle.solve_window(win)
    assert np.array_equal(a.kf_pose, b.kf_pose) and np.array_equal(a.lm_pos, b.lm_pos)
    assert np.isfinite(a.kf_pose).all() and np.isfinite(a.lm_pos).all()
    assert a.c.final_cost < a.c.initial_cost
    assert np.array_equal(a.kf_pose[0], win.kf_pose[0])
    rej = a.lm_rejected[:win.n_lm].astype(bool)
    assert rej.sum() > 0


@pytest.mark.parametrize("case", ["config2", "config3", "ragged", "short_tracks"])
def test_one_kernel_linearisation_equals_three_kernels(handle, monkeypatch, case):
    """k_linearize (evaluation + landmark blocks + V rows in one kernel, Jacobian in registers, cost at x only at iteration
    zero) against the three materialising kernels it replaces (KBA_LINEARIZE=0): same iterations, same rejections, results equal
    to rounding.  short_tracks: two observations per landmark, i.e. 16 landmarks per warp tile (several components per lane
    in the segment sums); ragged: landmarks without observations between the others."""
    from tests import edge_windows as ew
    if case == "config2":
        win = synth.make_window(2, n_kf=16, n_lm=900, n_obs=9000, seed=9)
    elif case == "config3":
        win = synth.make_window(3, n_kf=12, n_lm=500, n_obs=4000, seed=9, gp_frac=0.2)
    elif case == "ragged":
        win = ew.CASES["ragged"]()
    else:
        win = synth.make_window(2, n_kf=10, n_lm=1500, n_obs=3000, seed=9)
    monkeypatch.setenv("KBA_LINEARIZE", "1")
    a = handle.solve_window(win)
    monkeypatch.setenv("KBA_LINEARIZE", "0")
    b = handle.solve_window(win)
    assert a.c.status == 0 and b.c.status == 0 and a.c.num_solves == b.c.num_solves
    assert [s.num_iterations for s in a.solves] == [s.num_iterations for s in b.solves]
    assert [s.termination for s in a.solves] == [s.termination for s in b.solves]
    assert np.array_equal(a.lm_rejected[:win.n_lm], b.lm_rejected[:win.n_lm])
    assert a.c.final_cost == pytest.approx(b.c.final_cost, rel=1e-10)
    assert np.linalg.norm(a.kf_pose[:, 4:] - b.kf_pose[:, 4:], axis=1).max() <= 1e-8


def test_many_landmarks_host_packed_small_window(handle, oracle):
    """34 000 landmarks with short tracks in a 24-keyframe window: more landmarks than the device-side sort holds (32 768), so the
    window is packed on the host, yet it is a small window (139 reduced rows) and linearised by k_linearize -- its tile builder
    runs with 67 landmarks per chunk, twelve landmarks share a warp tile.  GPU vs oracle."""
    win = synth.make_window(2, n_kf=24, n_lm=34000, n_obs=80000, seed=13)
    assert win.n_lm > 32768
    rg = handle.solve_window(win)
    rc = oracle.solve_window(win, num_threads=8)
    _compare_solves(rg, rc, win, "many landmarks", lm_outliers=17)  # 0.05 % of the landmarks (two-view tracks without parallax)
    dl = np.linalg.norm(rg.lm_pos[:win.n_lm] - rc.lm_pos[:win.n_lm], axis=1)
    assert np.percentile(dl, 99) <= 1e-6


def test_small_batch_does_not_lower_a_live_batch_shared_memory(handle):
    """the opt-in dynamic shared memory of the solve kernels is a per-function attribute: creating a batch with a smaller
    reduced system while a larger one is alive (a persistent window next to one-shot solves) must not break the larger one"""
    from limo_b200 import capi
    big = synth.make_window(2, n_kf=30, n_lm=600, n_obs=6000, seed=3)
    small = synth.make_window(1, seed=4)
    b_big = handle.batch([big])
    ref = handle.solve_window(big)
    handle.solve_window(small)          # 5 keyframes: 64 reduced rows (the big batch uses 192)
    b_big.solve(capi.default_options())
    r = b_big.download()[0]
    assert r.c.status == 0 and np.array_equal(r.kf_pose, ref.kf_pose)
    b_big.close()


def test_bad_arguments(handle):
    """error behaviour of the boundary: fewer than 3 keyframes -> NotEnoughKeyframes (reference cpp:630-632)"""
    from limo_b200 import capi
    win = synth.make_window(1, n_kf=2, n_lm=20, n_obs=40)
    with pytest.raises(capi.KbaError, match="error 3"):
        handle.solve_window(win)


def test_large_window_generic_path_matches_oracle(handle, oracle):
    """BASELINE config 5 scaled to 40 keyframes (234 reduced rows): the panel-based generic Schur kernel and the
    global-memory Cholesky with tensor-core trailing update, GPU vs oracle"""
    win = synth.make_window(5, n_kf=40, n_lm=3000, n_obs=45000)
    rg = handle.solve_window(win)
    rc = oracle.solve_window(win, num_threads=8)
    _compare_solves(rg, rc, win, "config5-small")


def test_config5_full_window_matches_oracle(handle, oracle):
    """BASELINE config 5 at full size (100 keyframes / 20 000 landmarks / ~300 000 observations, 594 reduced rows): the
    split factorisation (k_chol_*) and the generic Schur kernel against the oracle at north_star's tolerances"""
    import os
    win = synth.make_window(5)
    assert (win.n_kf, win.n_lm) == (100, 20000) and win.n_obs > 290000
    rg = handle.solve_window(win)
    rc = oracle.solve_window(win, num_threads=min(32, os.cpu_count() or 8))
    # 20 000 landmarks: the handful seen twice at almost zero parallax (condition > 1e14 along the ray) move by metres with the
    # rounding of the last accepted step -- at most 0.05 % of the landmarks may, 99 % must agree to 1e-6 m
    _compare_solves(rg, rc, win, "config5-full", lm_outliers=10)
    dl = np.linalg.norm(rg.lm_pos[:win.n_lm] - rc.lm_pos[:win.n_lm], axis=1)
    assert np.percentile(dl, 99) <= 1e-6


def test_sharded_solve_with_one_rank_equals_plain_solve(handle):
    """the landmark-sharded multi-GPU path (NCCL exchange points, window-wide trimming) run with a single rank must
    reproduce the plain solve bit for bit; with 2 GPUs it is exercised by scripts/config5_sharded.py"""
    from limo_b200 import capi, parallel
    win = synth.make_window(5, n_kf=40, n_lm=3000, n_obs=45000)
    sub, j0, j1 = parallel.shard_window(win, 0, 1)
    assert (j0, j1) == (0, win.n_lm)
    comm = capi.ShardComm(handle, 0, 1, capi.shard_unique_id())
    batch = handle.batch([sub])
    batch.set_shard(comm, j0, win.n_lm)
    batch.solve(capi.default_options())
    rs = batch.download()[0]
    rp = handle.solve_window(win)
    assert [s.num_iterations for s in rs.solves] == [s.num_iterations for s in rp.solves]
    assert np.array_equal(rs.kf_pose, rp.kf_pose)
    assert np.array_equal(rs.lm_pos[:win.n_lm], rp.lm_pos[:win.n_lm])
    assert np.array_equal(rs.lm_rejected[:win.n_lm], rp.lm_rejected[:win.n_lm])
    batch.close()
    comm.close()


def test_fp32_linearisation_mode(handle, oracle):
    """kba_options.precision = 1 (BASELINE config 3's FP32 setting): residual / Jacobian blocks are evaluated and stored
    in single precision, every accumulation and the cost stay FP64.  Tolerances are single-precision ones, set from
    the measured deviations (scripts/fp32_check.py and scripts/fp32_agreement.py for the blocks; final cost 4e-7 relative, poses
    1.7 mm -- the flat directions of the problem amplify the gradient noise): north_star's 1e-6 m is an FP64 statement."""
    from limo_b200 import capi
    from tests.test_far_windows import check_fp32_blocks
    opt = capi.default_options()
    opt.precision = 1
    win = synth.make_window(2, n_kf=12, n_lm=400, n_obs=3000)
    r, jp, jl, cost, failed = handle.evaluate(win, opt)
    r0, jp0, jl0, cost0, _ = oracle.evaluate(win)
    assert failed == 0 and cost == pytest.approx(cost0, rel=1e-12)  # the cost is evaluated in FP64
    assert np.abs(r - r0).max() <= 2e-3                             # pixels, values up to ~1e3 before the loss
    assert np.abs(jp - jp0).max() <= 3e-5 * np.abs(jp0).max() and np.abs(jl - jl0).max() <= 3e-5 * np.abs(jl0).max()
    # and every column family against kba_eval's FP64 blocks at the bounds tests/test_far_windows.py holds far from the origin
    check_fp32_blocks(win, (r, jp, jl), handle.evaluate(win, capi.default_options()), "config2_slice")
    for cfg, kw in ((2, dict()), (3, dict(seed=41))):
        win = synth.make_window(cfg, **kw)
        rg = handle.solve_window(win, opt)
        rc = oracle.solve_window(win, num_threads=8)
        assert rg.c.status == 0 and rg.c.num_solves == rc.c.num_solves
        assert rg.c.final_cost == pytest.approx(rc.c.final_cost, rel=1e-5)
        assert np.linalg.norm(rg.kf_pose[:, 4:] - rc.kf_pose[:, 4:], axis=1).max() <= 5e-3
        assert (rg.lm_rejected[:win.n_lm] != rc.lm_rejected[:win.n_lm]).mean() <= 0.005


@pytest.mark.parametrize("precision", [0, 1])
def test_eval_landmark_jacobian_is_the_one_the_fused_solve_forms(handle, precision):
    """On the fused path J_l is not stored: the solve forms it in FP64 as (translation columns of J_p) R(keyframe), from the
    FP32 J_p under precision 1.  kba_eval must report that matrix, not a copy rounded to FP32: tests/test_first_step_dense.py
    builds the solve's normal equations from what kba_eval reports."""
    from limo_b200 import capi
    opt = capi.default_options()
    opt.precision = precision
    win = synth.make_window(2, n_kf=12, n_lm=400, n_obs=3000)
    _, jp, jl, _, failed = handle.evaluate(win, opt)
    R = np.stack([g.pose_to_iso(p)[:3, :3] for p in win.kf_pose])[win.obs_kf]
    want = jp[:, :, 3:6] @ R
    free = win.kf_fixed[win.obs_kf] == 0                    # a constant keyframe's J_p is reported as zeros
    assert failed == 0 and free.sum() > 0.8 * win.n_obs
    assert np.abs(jl[free] - want[free]).max() <= 1e-13 * np.abs(want).max()


@pytest.mark.parametrize("case", ["ragged", "all_keyframes_fixed", "evaluation_failure", "tiny"])
def test_edge_case_windows_match_oracle(handle, oracle, case):
    """ragged CSR rows (landmarks with zero / one observation), a window whose keyframes are all constant (no reduced
    system), an evaluation failure at the first iterate (FAILURE termination, then trimming removes the culprit) and a
    window below min_landmarks_for_trimming: same terminations, iterates and results as the oracle"""
    from tests import edge_windows as ew
    win = ew.CASES[case]()
    rg = handle.solve_window(win)
    rc = oracle.solve_window(win)
    # landmarks seen once have a rank-2 block that only the LM damping regularises, and with constant keyframes nothing
    # couples a badly observed landmark to the rest: their positions are flat directions (cost and poses are not)
    tol = {"ragged": dict(lm_p95=1e-4, lm_max=1.0), "all_keyframes_fixed": dict(lm_max=np.inf)}.get(case, {})
    _compare_solves(rg, rc, win, case, **tol)
    if case == "all_keyframes_fixed":
        assert np.array_equal(rg.kf_pose, win.kf_pose)
    if case == "ragged":
        empty = np.diff(win.lm_obs_ptr) == 0
        assert empty.sum() == 4 and np.array_equal(rg.lm_pos[:win.n_lm][empty], win.lm_pos[empty])


def test_device_packing_equals_host_packing(handle, monkeypatch):
    """the packing kernels (kba_pack.cu: landmark sort by (first, last) keyframe, CSR, keyframe-major copy, ground-plane
    mapping, group ranges, caller-order download) against the host packer of round 1 (KBA_DEVICE_PACK=0): the same sorted
    layout, hence bit-identical solves -- mono + depth windows, ground-plane windows, ragged CSR rows, a two-camera rig"""
    from tests import edge_windows as ew
    wins = [synth.make_window(2, n_kf=12, n_lm=700, n_obs=6000, seed=3), synth.make_window(3, seed=41, n_kf=8, n_lm=300, n_obs=1800, gp_frac=0.2),
            ew.CASES["ragged"](), synth.make_window(1, seed=9)]
    dev = handle.solve_batch(wins)
    monkeypatch.setenv("KBA_DEVICE_PACK", "0")
    host = handle.solve_batch(wins)
    for a, b, w in zip(dev, host, wins):
        assert a.c.status == 0 and b.c.status == 0
        assert [s.num_iterations for s in a.solves] == [s.num_iterations for s in b.solves]
        assert np.array_equal(a.kf_pose, b.kf_pose)
        assert np.array_equal(a.lm_pos[:w.n_lm], b.lm_pos[:w.n_lm])
        assert np.array_equal(a.lm_rejected[:w.n_lm], b.lm_rejected[:w.n_lm])
        assert a.c.final_cost == b.c.final_cost
