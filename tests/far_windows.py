"""Windows far from the origin.

limo stores a keyframe's pose as keyframe <- origin and its landmarks in the origin's frame, and the origin is where the drive
started: after a KITTI-length drive a window sits hundreds of metres to kilometres from it.  limo_b200/synth.py starts every
trajectory at the identity, so every window it builds lies within about 150 m of the origin.  far(win, G) moves a window to
where a long drive would put it, by moving the origin: the same problem, in other global coordinates.
"""
import numpy as np

from limo_b200 import geometry as g
from tests import edge_windows as ew

YAW = 2.1                                   # rad: about an axis close to, but not, the vertical
AXIS = np.array([0.05, -0.03, 1.0]) / np.linalg.norm([0.05, -0.03, 1.0])
DIRECTION = np.array([0.8, -0.6, 0.05]) / np.linalg.norm([0.8, -0.6, 0.05])

# distance of the window from the new origin, in metres: 1 km, 5 km (the largest distance of a KITTI odometry sequence) and
# 10 km, a stress case
DISTANCES = {"1km": 1e3, "5km": 5e3, "10km": 1e4}


def transform(distance):
    """G = new origin <- old origin: a rotation of YAW about AXIS, then an offset of `distance` metres along DIRECTION"""
    return g.iso(g.angle_axis(YAW, AXIS), distance * DIRECTION)


def far(win, G, skip=()):
    """copy of `win` (every field of Window, edge_windows.copy_window) with the origin moved by the rigid transform G (new origin
    <- old origin).  In exact arithmetic every residual of the window, and so its cost, Jacobian translation columns and trimming
    decisions, stay what they were.

    Moved (they are in the origin's frame, or point to it):
      kf_pose                 keyframe <- origin: T_k G^-1;
      lm_pos                  a point in the origin's frame: G p;
      speed_T_origin_before   origin <- previous frame: G T (speed_reg forms (T_cur T).t, previous frame -> current keyframe,
                              which T_cur G^-1 G T leaves as it was).
    Kept (each is local to a keyframe, a camera or an observation):
      kf_plane                direction and distance of the ground plane in the keyframe's frame: gp_height forms
                              n . (T_k p) + dist, and T_k p is invariant;
      cam_pose, cam_intr      camera <- keyframe and the intrinsics;
      obs_*                   pixels and depths measured in a camera;
      gp_lm, gp_kf, gp_weight indices and weights;
      scale_*                 scale_reg is the length of (T_1 T_0^-1).t, the translation between two keyframes, invariant;
      plane_reg_weight        the plane chain compares directions and distances in keyframe frames, and gp_motion takes
                              (T_0 T_1^-1).t, invariant like the scale's;
      speed_v_before, speed_dt  the previous velocity in the current keyframe's frame, and a time;
      kf_fixed, lm_weight, lm_obs_ptr, obs_kf, obs_cam, landmarks_fixed, plane_dist_fixed, speed_kf, speed_weight: not geometry.
    skip: names among kf_pose, lm_pos and speed_T_origin_before to leave unmoved (a broken transform, for negative controls)."""
    Gi = g.iso_inv(G)
    over = {}
    if "kf_pose" not in skip:
        over["kf_pose"] = np.stack([g.iso_to_pose(g.pose_to_iso(p) @ Gi) for p in win.kf_pose])
    if "lm_pos" not in skip:
        over["lm_pos"] = win.lm_pos @ G[:3, :3].T + G[:3, 3]
    if "speed_T_origin_before" not in skip:
        over["speed_T_origin_before"] = g.iso_to_pose(G @ g.pose_to_iso(np.asarray(win.speed_T_origin_before, dtype=float)))
    return ew.copy_window(win, **over)


def back(pose_or_lm, G, kind):
    """a solved keyframe pose (7) or landmark (3) of far(win, G) in the original window's frame"""
    if kind == "pose":
        return np.stack([g.iso_to_pose(g.pose_to_iso(p) @ G) for p in np.atleast_2d(pose_or_lm)])
    Gi = g.iso_inv(G)
    return np.atleast_2d(pose_or_lm) @ Gi[:3, :3].T + Gi[:3, 3]


def centre_distance(win):
    """distance from the origin of the mean keyframe position (origin <- keyframe translation)"""
    c = np.stack([g.iso_inv(g.pose_to_iso(p))[:3, 3] for p in win.kf_pose])
    return float(np.linalg.norm(c.mean(axis=0)))
