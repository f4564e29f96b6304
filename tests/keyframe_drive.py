"""Seeded closed-loop drives for keyframe selection (tests/test_track_keyframe.py, scripts/keyframe_flow_bench.py).

A KeyframeDrive is a sequence of frames every 0.1 s from the rig of tests/create_drive.Drive (one or two cameras).  Features are
tracks: a landmark keeps its id from frame to frame while it stays in view and alive, and new tracks replace those that end.  The
selector of limo (flow, pose and time schemes, limo_b200.keyframe_selector) decides on every frame, against the last `window`
selected keyframes, whether it is pushed; the drive is generated in that loop, so that it reaches:
  - a normal speed (enough flow; the time scheme selects every fifth frame) and a standstill and a crawl (too little flow);
  - a rotation burst: a yaw step on the frame after a keyframe, which the pose scheme selects before the time scheme would;
  - a frame that shares no landmark with the newest keyframe: it re-observes landmarks that have slots, but not the newest
    keyframe's, and new ones (no match: NaN, rejected);
  - on a rig, tracks that switch camera: the frame measures a landmark on the camera the newest keyframe did not use;
  - a frame that the time scheme would keep, whose threshold is set to its own flow_sum / n_matched, so that min_median_flow^2
    equals its mean_flow_sq bit for bit (strict >, so rejected).
Landmark slot = landmark id; a landmark has a slot once a selected frame measured it.  write() stores a drive in the text format
tests/cpp/test_facade_keyframe.cpp reads (doubles as hex floats)."""
import numpy as np

from limo_b200.keyframe_selector import (Frame, KeyframeRejectionSchemeFlow, KeyframeSelectionSchemePose, KeyframeSelector,
                                         KeyframeSparsificationSchemeTime, convert_sec, frame_flow, newest)
from tests.create_drive import F32, Drive, _quat, _rot

T0, DT = 1_000_000_000, 100_000_000  # ns


def selector(min_median_flow, critical, time_sec, flow_fn=None):
    """limo's selector (mono_lidar.cpp:447-453): flow rejection, pose selection, time sparsification"""
    s = KeyframeSelector()
    s.addScheme(KeyframeRejectionSchemeFlow(min_median_flow, flow_fn))
    s.addScheme(KeyframeSelectionSchemePose(critical))
    s.addScheme(KeyframeSparsificationSchemeTime(time_sec))
    return s


class KeyframeDrive:
    def __init__(self, seed, n_frames=60, window=12, rig=True, n_feat=300, min_median_flow=5.0, critical=0.03, time_sec=0.4):
        rng = np.random.default_rng(seed)
        rig_of = Drive(seed, n_push=2, rig=rig, new_per_push=0)
        self.cam_pose, self.cam_intr = rig_of.cam_pose, rig_of.cam_intr
        n_cam = len(self.cam_pose)
        self.window, self.n_frames = window, n_frames
        self.min_median_flow, self.critical, self.time_sec = min_median_flow, critical, time_sec
        F = n_frames
        still, crawl, normal = (int(0.25 * F), int(0.4 * F)), (int(0.4 * F), int(0.65 * F)), int(0.65 * F)
        self.blank, self.equal = int(0.8 * F), None
        cams = [(_rot(q[:4] / np.linalg.norm(q[:4])), q[4:]) for q in self.cam_pose]
        tracks = {}  # landmark id -> [point, cameras, frames left]
        n_lm, x, yaw, burst_done = 0, 0.0, 0.0, False
        self.frames, self.thr = [], []
        buffer, slots, sel = {}, set(), []
        for k in range(F):
            speed = 0.0 if still[0] <= k < still[1] else (0.08 if crawl[0] <= k < crawl[1] else 1.0)
            x += speed
            yaw += 0.002 + rng.normal(0, 0.0005) if speed > 0 else 0.0
            if k >= normal and not burst_done and sel and sel[-1]:
                yaw += 0.06  # the rotation burst, on the frame after a keyframe
                burst_done = True
            pose = np.array(_quat(yaw) + [-x, rng.normal(0, 0.02) if speed > 0 else 0.0, 0.0])
            Rk, tk = _rot(pose[:4]), pose[4:]
            meas = {}

            def project(p, c):
                pc = cams[c][0] @ (Rk @ p + tk) + cams[c][1]
                f, cx, cy = self.cam_intr[c]
                if pc[2] < 1.0:
                    return None
                u, v = f * pc[0] / pc[2] + cx + rng.normal(0, 0.3), f * pc[1] / pc[2] + cy + rng.normal(0, 0.3)
                return (F32(u), F32(v)) if 0 <= u < 1280 and 0 <= v < 384 else None

            if k == self.blank:  # no landmark of the newest keyframe: landmarks with slots seen before it, and new ones
                last = newest(buffer)
                old = sorted(slots - set(last.measurements_))
                for lid in rng.choice(old, size=min(len(old), n_feat // 2), replace=False):
                    meas[int(lid)] = {int(rng.integers(0, n_cam)): (F32(rng.uniform(0, 1280)), F32(rng.uniform(0, 384)))}
                for _ in range(n_feat // 2):
                    meas[n_lm] = {0: (F32(rng.uniform(0, 1280)), F32(rng.uniform(0, 384)))}
                    n_lm += 1
            else:
                for lid in sorted(tracks):
                    p, tc, left = tracks[lid]
                    if n_cam > 1 and rng.random() < 0.04:  # the track switches camera
                        tc = [1 - tc[0]] if len(tc) == 1 else [int(rng.integers(0, 2))]
                        tracks[lid][1] = tc
                    obs = {c: uv for c in tc for uv in [project(p, c)] if uv is not None}
                    if left <= 0 or not obs:
                        del tracks[lid]
                        continue
                    tracks[lid][2] = left - 1
                    meas[lid] = obs
                while len(meas) < n_feat:
                    p = np.array([x + rng.uniform(5, 60), rng.uniform(-15, 15), rng.uniform(-2, 4)])
                    tc = sorted({int(rng.integers(0, n_cam)) for _ in range(2)})
                    obs = {c: uv for c in tc for uv in [project(p, c)] if uv is not None}
                    if not obs:
                        continue
                    tracks[n_lm] = [p, tc, int(rng.integers(3, 40))]
                    meas[n_lm] = obs
                    n_lm += 1
            frame = Frame(T0 + k * DT, pose, meas)
            thr = min_median_flow
            if self.equal is None and k >= int(0.88 * F) and frame.timestamp_ - newest(buffer).timestamp_ > convert_sec(time_sec):
                # the first frame there that the time scheme keeps: min_median_flow^2 == mean_flow_sq, the strict > rejects it
                n, s, _ = frame_flow(frame, newest(buffer))
                thr, self.equal = s / n, k
            self.frames.append(frame)
            self.thr.append(thr)
            keep = bool(selector(thr, critical, time_sec).select([frame], buffer))
            sel.append(keep)
            if keep:
                buffer[frame.timestamp_] = frame
                slots |= set(meas)
                while len(buffer) > window:
                    del buffer[min(buffer)]
        self.n_lm, self.selected = n_lm, sel

    def arena(self, k):
        """frame k's measurements in measurements_ order: (landmark id, camera, u, v) arrays"""
        rows = [(lid, c, *uv) for lid in sorted(self.frames[k].measurements_) for c, uv in sorted(self.frames[k].measurements_[lid].items())]
        lm, cam, u, v = zip(*rows)
        return np.array(lm, np.int32), np.array(cam, np.int32), np.array(u, np.float32), np.array(v, np.float32)

    def write(self, path):
        h = lambda x: float(x).hex()  # noqa: E731
        lines = ["cams %d" % len(self.cam_pose)]
        for intr, pose in zip(self.cam_intr, self.cam_pose):
            lines.append(" ".join(h(x) for x in list(intr) + list(pose)))
        lines += ["params %d %s %s" % (self.window, h(self.critical), h(self.time_sec)), "landmarks %d" % self.n_lm, "frames %d" % self.n_frames]
        for k, f in enumerate(self.frames):
            n = sum(len(o) for o in f.measurements_.values())
            lines.append("f %d %d %s %s" % (f.timestamp_, n, " ".join(h(x) for x in f.pose_), h(self.thr[k])))
            lm, cam, u, v = self.arena(k)
            lines += ["%d %d %s %s" % (a, b, h(c), h(d)) for a, b, c, d in zip(lm, cam, u, v)]
        with open(path, "w") as fh:
            fh.write("\n".join(lines) + "\n")
