"""A parameter sweep over one synthetic recording, as limo's tuning script runs it (keyframe_bundle_adjustment_ros_tool/res/
tune_parameters_kitti.py): every track of a group replays the same ground-plane drive with its own grid point of depth_thres x
repr_thres and the shrubbery weight 0.9 on the vegetation landmarks of its store.  A step tracks the next frame against the store
(adjust_pose), pushes it as a keyframe and solves the sliding window, which writes the window back into the store.

tests/test_window_options.py drives a few tracks of it as a group and each alone; scripts/sweep_bench.py times it."""
import copy

import numpy as np

from tests.test_track_group import PLANE, _Drive

# the grid of tune_parameters_kitti.py: 10 depth thresholds x 11 reprojection thresholds (1.8 twice), shrubbery weight 0.9
DEPTH_THRES = [round(0.10 + 0.01 * i, 2) for i in range(10)]
REPR_THRES = [1.0, 1.1, 1.2, 1.3, 1.4, 1.5, 1.6, 1.7, 1.8, 1.8, 2.0]
SHRUBBERY_WEIGHT = 0.9


def grid(n=None):
    """(depth_thres, repr_thres) of run i of the tuning script, in its loop order (depth outer); the first n runs"""
    g = [(d, r) for d in DEPTH_THRES for r in REPR_THRES]
    return g if n is None else [g[i % len(g)] for i in range(n)]


def options(points):
    """one kba_options per grid point: limo's defaults with the point's Cauchy scales"""
    from limo_b200 import capi
    out = []
    for d, r in points:
        o = capi.default_options()
        o.depth_thres, o.reprojection_thres = d, r
        out.append(o)
    return out


class SweepDrive:
    """W-keyframe ground-plane windows of one recording; every track keeps its own host mirror of the poses it solved"""

    def __init__(self, W=12, steps=6, n_lm=1500, n_obs=14000, seed=61):
        self.base = _Drive(seed=seed, W=W, n_lm=n_lm, n_obs=n_obs, config=3, ground=True, steps=steps)
        self.W, self.steps = W, steps
        n = self.base.win.n_lm
        self.shrubbery = np.arange(0, n, 4, dtype=np.int32)  # a quarter of the landmarks lie on vegetation

    def make(self, h):
        """a track of the recording (its first W keyframes pushed, shrubbery weights written) and its host mirror"""
        mirror = copy.copy(self.base)
        mirror.poses = self.base.poses.copy()
        t = mirror.make_track(h)
        t.set_landmarks(self.shrubbery, pos=self.base.win.lm_pos[self.shrubbery], weight=np.full(len(self.shrubbery), SHRUBBERY_WEIGHT))
        return t, mirror

    def frame(self, mirror, step):
        """the frame that becomes keyframe W - 1 + step, tracked from the pose of the newest solved keyframe"""
        k = self.W - 1 + step
        lm, u, v, d = self.base.per_kf[k]
        return dict(pose7=mirror.poses[k - 1].copy(), lm_slot=lm, u=u, v=v, d=d)

    def push(self, t, mirror, step, pose7):
        """keyframe W - 1 + step enters the store at the tracked pose"""
        k = self.W - 1 + step
        mirror.poses[k] = pose7
        if k >= self.W + 1:
            t.drop_keyframe(k % (self.W + 1))
        lm, u, v, d, cam = mirror.measurements(k)
        t.push_keyframe(k % (self.W + 1), pose7, lm, u, v, d, cam=cam, plane4=PLANE)
