"""Edge-case windows shared by the CPU (oracle only) and GPU (CUDA vs oracle) tests: ragged CSR rows, fully constant
keyframes, an evaluation failure at the first iterate, and a window too small for trimming."""
import inspect

import numpy as np

from limo_b200 import synth
from limo_b200.capi_types import Window

WINDOW_FIELDS = tuple(inspect.signature(Window.__init__).parameters)[1:]


def copy_window(win, **over):
    """copy of `win` with every field of Window (ground points, plane blocks, scale, plane-chain and speed regularisers
    included) and some of them overridden"""
    args = {k: getattr(win, k) for k in WINDOW_FIELDS}
    args.update(over)
    return Window(**args)


def _rebuild(win, keep_obs=None, **over):
    """copy of `win` with some observations dropped (keep_obs: boolean mask over observations) and fields overridden;
    ground points, plane blocks and the regularisers are not carried over (copy_window keeps them)"""
    ptr = np.asarray(win.lm_obs_ptr)
    keep = np.ones(win.n_obs, dtype=bool) if keep_obs is None else keep_obs
    counts = np.array([keep[ptr[j]:ptr[j + 1]].sum() for j in range(win.n_lm)])
    new_ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    args = dict(kf_pose=win.kf_pose, kf_fixed=win.kf_fixed, cam_intr=win.cam_intr, cam_pose=win.cam_pose,
                lm_pos=win.lm_pos, lm_weight=win.lm_weight, lm_obs_ptr=new_ptr, obs_kf=win.obs_kf[keep],
                obs_u=win.obs_u[keep], obs_v=win.obs_v[keep], obs_d=win.obs_d[keep],
                obs_cam=None if win.obs_cam is None else win.obs_cam[keep])
    args.update(over)
    return Window(**args)


def ragged():
    """landmarks without any observation (empty CSR rows) and landmarks observed exactly once"""
    win = synth.make_window(1, seed=21)
    ptr = np.asarray(win.lm_obs_ptr)
    keep = np.ones(win.n_obs, dtype=bool)
    for j in (0, 7, 8, win.n_lm - 1):          # no observations at all
        keep[ptr[j]:ptr[j + 1]] = False
    for j in (3, 50):                           # a single observation
        keep[ptr[j] + 1:ptr[j + 1]] = False
    return _rebuild(win, keep)


def all_keyframes_fixed():
    """every keyframe constant: only the landmark blocks are in the program (no reduced system at all)"""
    win = synth.make_window(1, seed=22)
    return _rebuild(win, kf_fixed=np.ones(win.n_kf, dtype=np.uint8))


def evaluation_failure():
    """one landmark sits in the |z_cam| < 0.01 band of a keyframe at the initial state: Ceres' "Residual and Jacobian
    evaluation failed" (cost_functors_ceres.hpp:78-83) -> FAILURE termination, state untouched"""
    win = synth.make_window(1, seed=23)
    from limo_b200 import geometry as g
    k = int(win.obs_kf[0])
    T = g.pose_to_iso(win.kf_pose[k])             # keyframe <- origin
    Tc = g.pose_to_iso(win.cam_pose[0]) @ T       # camera <- origin
    p_cam = np.array([0.3, 0.1, 0.001])           # inside the failure band
    p_o = np.linalg.inv(Tc) @ np.append(p_cam, 1.0)
    lm = win.lm_pos.copy()
    lm[0] = p_o[:3]
    return _rebuild(win, lm_pos=lm)


def tiny():
    """3 keyframes / 40 landmarks: below min_landmarks_for_trimming, a single final solve"""
    return synth.make_window(1, seed=24, n_kf=3, n_lm=40, n_obs=100)


CASES = {"ragged": ragged, "all_keyframes_fixed": all_keyframes_fixed, "evaluation_failure": evaluation_failure,
         "tiny": tiny}
