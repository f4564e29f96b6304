"""The fused small-window Schur kernel (k_schur_fused: 16x8 FP64 MMAs, halves outside a group's exact rows skipped) against
the round-1 path (KBA_FUSED=0: zero-padded global V panels and k_schur_syrk_tma on m8n8k4) on the shapes that exercise its
variants: same iterations, terminations and rejections, results equal to rounding."""
import numpy as np
import pytest

from limo_b200 import geometry as g
from limo_b200 import synth
from limo_b200.capi_types import Window

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


def _gap_over_fixed_keyframe():
    """keyframe 4 is constant as well as keyframe 0: every track through it has a gap in its reduced-system rows, so its
    rows are not one run (per-observation copies instead of one bulk copy per panel column)"""
    win = synth.make_window(2, n_kf=10, n_lm=700, n_obs=6000, seed=17)
    fixed = np.array(win.kf_fixed, dtype=np.uint8)
    fixed[4] = 1
    return Window(kf_pose=win.kf_pose, kf_fixed=fixed, cam_intr=win.cam_intr, cam_pose=win.cam_pose, lm_pos=win.lm_pos,
                  lm_weight=win.lm_weight, lm_obs_ptr=win.lm_obs_ptr, obs_kf=win.obs_kf, obs_u=win.obs_u, obs_v=win.obs_v,
                  obs_d=win.obs_d, obs_cam=win.obs_cam)


def _stereo_rig():
    """two thirds of the landmarks are seen by both cameras of a stereo rig in the same keyframe: rows that add onto
    others (max_rank > 0), the synchronous producer path"""
    win, truth = synth.make_window(2, n_kf=8, n_lm=300, n_obs=1800, seed=31, return_truth=True)
    T0 = g.pose_to_iso(win.cam_pose[0])
    T1 = g.iso(t=[-0.54, 0.0, 0.0]) @ T0
    rng = np.random.default_rng(3)
    okf, ocam, ou, ov, od, ptr = [], [], [], [], [], [0]
    for j in range(win.n_lm):
        for o in range(win.lm_obs_ptr[j], win.lm_obs_ptr[j + 1]):
            k = win.obs_kf[o]
            okf.append(k); ocam.append(0); ou.append(win.obs_u[o]); ov.append(win.obs_v[o]); od.append(win.obs_d[o])
            pc = g.apply(T1 @ g.pose_to_iso(truth["kf_pose"][k]), truth["lm_pos"][j])
            if pc[2] > 0.5 and j % 3 != 0:
                okf.append(k); ocam.append(1)
                ou.append(synth.F * pc[0] / pc[2] + synth.CX + rng.normal(0, 0.5))
                ov.append(synth.F * pc[1] / pc[2] + synth.CY + rng.normal(0, 0.5)); od.append(-1.0)
        ptr.append(len(okf))
    return Window(kf_pose=win.kf_pose, kf_fixed=win.kf_fixed, cam_intr=[win.cam_intr[0]] * 2,
                  cam_pose=[win.cam_pose[0], g.iso_to_pose(T1)], lm_pos=win.lm_pos, lm_weight=win.lm_weight, lm_obs_ptr=ptr,
                  obs_kf=okf, obs_cam=ocam, obs_u=ou, obs_v=ov, obs_d=od, scale_kf0=0, scale_kf1=1,
                  scale_weight=win.scale_weight, scale_value=win.scale_value)


def _window(case):
    from tests import edge_windows as ew
    if case == "config2":
        return synth.make_window(2, n_kf=16, n_lm=900, n_obs=9000, seed=9)
    if case == "short_tracks":   # two observations per landmark
        return synth.make_window(2, n_kf=10, n_lm=1500, n_obs=3000, seed=9)
    if case == "ragged":
        return ew.CASES["ragged"]()
    if case == "gap_over_fixed_keyframe":
        return _gap_over_fixed_keyframe()
    if case == "stereo_rig":
        return _stereo_rig()
    # 30 free keyframes, but 187 rows over all 31 keyframes: the large-window path (k_schur_syrk) with KBA_FUSED=1 as with
    # KBA_FUSED=0, so this case compares that path with itself; the seven-slot variant needs 30 keyframes none of which is fixed
    # (tests/test_first_step_dense.py holds its first step to the dense reference)
    return synth.make_window(2, n_kf=31, n_lm=700, n_obs=7000, seed=5)


@pytest.mark.parametrize("case", ["config2", "short_tracks", "ragged", "gap_over_fixed_keyframe", "stereo_rig",
                                  "free_keyframes_30"])
def test_fused_schur_equals_round_one_schur(handle, monkeypatch, case):
    win = _window(case)
    monkeypatch.setenv("KBA_FUSED", "1")
    a = handle.solve_window(win)
    monkeypatch.setenv("KBA_FUSED", "0")
    b = handle.solve_window(win)
    assert a.c.status == 0 and b.c.status == 0 and a.c.num_solves == b.c.num_solves
    assert [s.num_iterations for s in a.solves] == [s.num_iterations for s in b.solves]
    assert [s.num_successful_steps for s in a.solves] == [s.num_successful_steps for s in b.solves]
    assert [s.termination for s in a.solves] == [s.termination for s in b.solves]
    assert np.array_equal(a.lm_rejected[:win.n_lm], b.lm_rejected[:win.n_lm])
    assert a.c.final_cost == pytest.approx(b.c.final_cost, rel=1e-10)
    assert np.linalg.norm(a.kf_pose[:, 4:] - b.kf_pose[:, 4:], axis=1).max() <= 1e-8
