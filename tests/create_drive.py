"""Seeded drives for push()'s landmark creation (tests/test_track_create.py, scripts/create_landmarks_bench.py).

A drive is a rig of one or two cameras, keyframe poses along x (vehicle <- origin, z up) and, per keyframe, its measurements
(landmark id, camera, u, v, d) in (id, camera) order -- the order of Keyframe::measurements_, which is also the arena order a
caller pushes.  Every push introduces `new_per_push` landmarks.  They cover the cases of the facade's calculateLandmark:
  - a lidar depth on the first keyframe that sees the landmark: on every camera, on the second camera only, or NaN (no depth);
    on a rig also NaN on the first camera and a depth on the second: push() then back-projects the NaN (it skips only d < 0);
  - no depth: two rays or more (a landmark seen by one camera first and by both a keyframe later), or one ray only (never created);
  - parallel rays: the vehicle stands still for one push (two keyframes with the same pose) and some landmarks are measured at
    the same pixel in both; for those at the principal point the host's triangulation divides by an exact zero (inf / NaN).
write() stores a drive in the text format tests/cpp/test_facade_create.cpp reads (doubles as hex floats)."""
import math

import numpy as np

F32 = np.float32


def _quat(yaw, pitch=0.0, roll=0.0):
    cy, sy, cp, sp, cr, sr = (math.cos(yaw / 2), math.sin(yaw / 2), math.cos(pitch / 2), math.sin(pitch / 2), math.cos(roll / 2),
                              math.sin(roll / 2))
    return [cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy]


def _rot(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


class Drive:
    def __init__(self, seed, n_push=30, window=12, rig=True, new_per_push=60, depth=True):
        rng = np.random.default_rng(seed)
        self.window, self.n_push = window, n_push
        self.cam_pose = [np.array([0.5, 0.5, -0.5, 0.5, 0.0, 0.0, 0.0])]  # camera <- vehicle: camera z = vehicle x
        self.cam_intr = [[512.0, 640.0, 192.0]]  # powers of two: the principal point's ray is exactly the optical axis
        if rig:  # a second camera, turned a little, with a quaternion that is not normalised
            self.cam_pose.append(np.array([0.52, 0.48, -0.5, 0.5, 0.3, -0.1, 0.05]))
            self.cam_intr.append([650.0, 610.0, 185.0])
        n_cam = len(self.cam_pose)
        self.stop = n_push // 2  # keyframe stop + 1 has the pose of keyframe stop
        self.kf_pose = []
        for k in range(n_push):
            if k == self.stop + 1:
                self.kf_pose.append(self.kf_pose[-1].copy())
                continue
            q = [1.0, 0.0, 0.0, 0.0] if k == self.stop else _quat(0.01 * k + rng.normal(0, 0.003), rng.normal(0, 0.002), rng.normal(0, 0.002))
            self.kf_pose.append(np.array(q + [-1.5 * k + rng.normal(0, 0.01), rng.normal(0, 0.05), rng.normal(0, 0.02)]))
        self.meas = [dict() for _ in range(n_push)]  # keyframe -> landmark id -> [(camera, u, v, d)] in camera order
        lm = 0
        for k in range(n_push):
            for j in range(new_per_push):
                kind = j % 10
                p = np.array([1.5 * k + rng.uniform(4, 60), rng.uniform(-20, 20), rng.uniform(-2, 5)])
                span = list(range(k, min(n_push, k + int(rng.integers(1, 7)))))
                if kind == 9 and k == self.stop:  # parallel rays: the same pixel in the two keyframes of the stop; at the principal
                    # point the rays are exactly the z axis (the stop's rotation is the identity), sum (I - r r^T) is exactly singular
                    u, v = (F32(640.0), F32(192.0)) if j % 20 == 9 else (F32(rng.uniform(100, 1100)), F32(rng.uniform(50, 330)))
                    self.meas[k][lm] = [(0, u, v, F32(-1.0))]
                    self.meas[k + 1][lm] = [(0, u, v, F32(-1.0))]
                    lm += 1
                    continue
                for i, kk in enumerate(span):
                    if kind == 8:                       # one ray: seen once, by one camera, without a depth
                        if i > 0:
                            break
                        cams = [0]
                    elif kind == 7 and i == 0:          # one camera first, more rays a keyframe later
                        cams = [n_cam - 1]
                    elif kind == 4 and i == 0:          # every camera of the rig (the NaN-then-depth case)
                        cams = list(range(n_cam))
                    else:
                        cams = [c for c in range(n_cam) if rng.random() < 0.7] or [int(rng.integers(0, n_cam))]
                    obs = []
                    for c in cams:
                        Rk, tk = _rot(self.kf_pose[kk][:4]), self.kf_pose[kk][4:]
                        Rc, tc = _rot(self.cam_pose[c][:4] / np.linalg.norm(self.cam_pose[c][:4])), self.cam_pose[c][4:]
                        pc = Rc @ (Rk @ p + tk) + tc
                        f, cx, cy = self.cam_intr[c]
                        if pc[2] > 0.5:
                            u, v = f * pc[0] / pc[2] + cx + rng.normal(0, 0.5), f * pc[1] / pc[2] + cy + rng.normal(0, 0.5)
                        else:
                            u, v = rng.uniform(0, 1200), rng.uniform(0, 380)
                        d = -1.0
                        if depth and i == 0:
                            if kind in (0, 1) or (kind == 2 and c == 1):  # every camera / the second camera only
                                d = pc[2] + rng.normal(0, 0.05)
                            elif kind == 3:
                                d = float("nan")                        # NaN is not a depth
                            elif kind == 4 and n_cam > 1:               # NaN on the first camera, a depth on the second
                                d = float("nan") if c == 0 else pc[2] + rng.normal(0, 0.05)
                        obs.append((c, F32(u), F32(v), F32(d)))
                    self.meas[kk][lm] = obs
                lm += 1
        self.n_lm = lm

    def write(self, path):
        h = lambda x: float(x).hex()  # noqa: E731
        lines = ["cams %d" % len(self.cam_pose)]
        for intr, pose in zip(self.cam_intr, self.cam_pose):
            lines.append(" ".join(h(x) for x in list(intr) + list(pose)))
        lines += ["window %d" % self.window, "landmarks %d" % self.n_lm, "pushes %d" % self.n_push]
        for k in range(self.n_push):
            n = sum(len(o) for o in self.meas[k].values())
            lines.append("kf %d %d %s" % (k, n, " ".join(h(x) for x in self.kf_pose[k])))
            for lid in sorted(self.meas[k]):
                for c, u, v, d in self.meas[k][lid]:
                    lines.append("%d %d %s %s %s" % (lid, c, h(u), h(v), h(d)))
        with open(path, "w") as f:
            f.write("\n".join(lines) + "\n")

    def arena(self, k):
        """keyframe k's measurements as kba_track_push_keyframe takes them: (landmark id, camera, u, v, d) arrays"""
        rows = [(lid, c, u, v, d) for lid in sorted(self.meas[k]) for c, u, v, d in self.meas[k][lid]]
        lm, cam, u, v, d = zip(*rows)
        return (np.array(lm, np.int32), np.array(cam, np.int32), np.array(u, np.float32), np.array(v, np.float32),
                np.array(d, np.float32))
