"""Host-side statement of limo's `KeyframeSelector` and its three keyframe schemes (Python edition).

Same names and rules as the reference (keyframe_bundle_adjustment/include/keyframe_bundle_adjustment/keyframe_selector.hpp,
src/keyframe_selector.cpp:14-133, src/keyframe_{rejection_scheme_flow,selection_scheme_pose,sparsification_scheme_time}.cpp)
and the C++ facade (limo_b200/csrc/facade/keyframe_selector.cpp), double for double: Python floats are IEEE doubles and
nothing here is contracted into a fused multiply-add.

The flow scheme is the one scheme that reads stored measurements.  A track user passes `flow_fn` to take its quantity from the
device-resident store (`capi.Track.frame_flow`, kba_track_frame_flow) instead of walking the newest keyframe on the host; the
early returns and the comparison stay here.  The rotation angle of the pose scheme stays on the host: it goes through atan2,
which the device cannot match bit for bit.
"""
import math

import numpy as np


class Frame:
    """The parts of a Keyframe the schemes read: timestamp_ (unsigned nanoseconds), pose_ (7-vector, quaternion w x y z
    first) and measurements_ ({landmark id: {camera id: (u, v)}}, float32 pixels)."""

    def __init__(self, timestamp, pose, measurements):
        self.timestamp_ = int(timestamp)
        self.pose_ = [float(x) for x in pose]
        self.measurements_ = measurements

    def hasMeasurement(self, lm_id, cam_id):
        return cam_id in self.measurements_.get(lm_id, ())


def convert_sec(ts):
    """convert(TimestampSec): ts * 1e9 truncated to unsigned nanoseconds (definitions.cpp)"""
    return int(float(ts) * 1e9)


def calcQuaternionDiff(p0, p1):
    """the angle of AngleAxisd(q1.inverse() * q0), in the facade's operation order (mini_eigen.hpp)"""
    w0, x0, y0, z0 = p0[:4]
    w1, x1, y1, z1 = p1[:4]
    n = w1 * w1 + x1 * x1 + y1 * y1 + z1 * z1
    aw, ax, ay, az = w1 / n, -x1 / n, -y1 / n, -z1 / n
    qw = aw * w0 - ax * x0 - ay * y0 - az * z0
    qx = aw * x0 + ax * w0 + ay * z0 - az * y0
    qy = aw * y0 - ax * z0 + ay * w0 + az * x0
    qz = aw * z0 + ax * y0 - ay * x0 + az * w0
    s = math.sqrt(qx * qx + qy * qy + qz * qz)
    return 2.0 * math.atan2(s, abs(qw)) if s != 0.0 else 0.0


def newest(last_frames):
    """the frame with the largest time stamp, the first of equal ones in key order (std::max_element)"""
    best = None
    for k in sorted(last_frames):
        if best is None or best.timestamp_ < last_frames[k].timestamp_:
            best = last_frames[k]
    return best


def frame_flow(new_frame, last_keyframe):
    """KeyframeRejectionSchemeFlow's quantity: (n_matched, flow_sum, mean_flow_sq) over the (landmark, camera) pairs of new_frame
    that last_keyframe also measures, summed in measurements_ order; mean_flow_sq is NaN without a match"""
    n, s = 0, 0.0
    for lm in sorted(new_frame.measurements_):
        for cam in sorted(new_frame.measurements_[lm]):
            if not last_keyframe.hasMeasurement(lm, cam):
                continue
            u, v = new_frame.measurements_[lm][cam]
            lu, lv = last_keyframe.measurements_[lm][cam]
            dx, dy = float(np.float32(u)) - float(np.float32(lu)), float(np.float32(v)) - float(np.float32(lv))
            s += math.sqrt(dx * dx + dy * dy)
            n += 1
    with np.errstate(invalid="ignore"):
        m = np.float64(s) / np.float64(n)  # 0 / 0 gives the CPU's NaN, as in the facade
    return n, s, float(m * m)


class KeyframeRejectionSchemeFlow:
    """reject a frame whose pixels moved too little against the newest selected keyframe (the squared mean flow, which the
    reference calls the median).  flow_fn(new_frame, last_keyframe) -> (n_matched, flow_sum, mean_flow_sq) replaces the host
    walk, e.g. by capi.Track.frame_flow on the store."""

    def __init__(self, min_median_flow, flow_fn=None):
        self.min_median_flow_squared_ = float(min_median_flow) * float(min_median_flow)
        self.flow_fn = flow_fn or frame_flow

    def isUsable(self, new_frame, last_frames):
        if not last_frames:
            return True
        if not new_frame.measurements_:
            return False
        return self.flow_fn(new_frame, newest(last_frames))[2] > self.min_median_flow_squared_


class KeyframeSelectionSchemePose:
    """select a frame whose rotation differs by more than critical_quaternion_difference (radians) from the newest keyframe's"""

    def __init__(self, critical_quaternion_difference):
        self.critical_quaternion_diff_ = float(critical_quaternion_difference)

    def isUsable(self, new_frame, last_frames):
        if not last_frames:  # an empty buffer would otherwise take every frame
            return False
        return calcQuaternionDiff(new_frame.pose_, newest(last_frames).pose_) > self.critical_quaternion_diff_


class KeyframeSparsificationSchemeTime:
    """keep a frame only when more than time_difference_sec have passed since the newest keyframe; the difference is unsigned
    64-bit arithmetic, so a frame older than the newest keyframe wraps around and is usable"""

    def __init__(self, time_difference_sec):
        self.time_difference_nano_sec_ = convert_sec(time_difference_sec)

    def isUsable(self, new_frame, last_frames):
        if not last_frames:
            return True
        return (new_frame.timestamp_ - newest(last_frames).timestamp_) % 2**64 > self.time_difference_nano_sec_


def _pass_all(frames, buffer, schemes):
    """applyRejectionScheme (cpp:33-56): the frames no scheme turns down, numbered 0, 1, ..., each tested against the buffer
    and against the frames this pass accepted before it"""
    out = {}
    for f in frames:
        if not any(not s.isUsable(f, buffer) or not s.isUsable(f, out) for s in schemes):
            out[len(out)] = f
    return out


def _pass_any(frames, buffer, schemes):
    """applySelectionScheme (cpp:66-84): the frames some scheme takes, against the buffer or the frames taken before"""
    out = {}
    for f in frames:
        if any(s.isUsable(f, buffer) or s.isUsable(f, out) for s in schemes):
            out[len(out)] = f
    return out


def eraseRejected(cur, kept):
    """cpp:85-104: drop the entries of cur whose KEY (a pass's own counter, not a frame) is not a key of kept.  The entry after
    an erased one is skipped, as the reference's loop advances past the iterator erase() returns; where that iterator is the
    end, the reference's advance is undefined and this stops."""
    if not kept:
        cur.clear()
    if not cur:
        return
    keys = sorted(cur)
    i = 0
    while i < len(keys):
        if keys[i] not in kept:
            del cur[keys[i]]
            if i + 1 == len(keys):
                break
            i += 1  # erase() returned the next entry, which the loop's increment then skips
        i += 1


class KeyframeSelector:
    """KeyframeSelector: rejection, selection and sparsification schemes composed as select() composes them.  frames is a list
    here and is walked in the caller's order (the reference walks a std::set of pointers, by address; limo passes one frame)."""

    def __init__(self):
        self.selection_schemes_, self.rejection_schemes_, self.sparsification_schemes_ = [], [], []

    def addScheme(self, scheme):
        if isinstance(scheme, KeyframeSelectionSchemePose):
            self.selection_schemes_.append(scheme)
        elif isinstance(scheme, KeyframeRejectionSchemeFlow):
            self.rejection_schemes_.append(scheme)
        elif isinstance(scheme, KeyframeSparsificationSchemeTime):
            self.sparsification_schemes_.append(scheme)
        else:
            raise TypeError("not a keyframe scheme: %r" % (scheme,))

    def select(self, frames, buffer_selected_frames):
        """the frames to keep, in the order of frames"""
        kept = _pass_all(frames, buffer_selected_frames, self.rejection_schemes_)
        selected = _pass_any(frames, buffer_selected_frames, self.selection_schemes_)
        eraseRejected(selected, kept)
        sparse = _pass_all(frames, buffer_selected_frames, self.sparsification_schemes_)
        eraseRejected(sparse, kept)
        ids = {id(f) for f in list(selected.values()) + list(sparse.values())}
        return [f for f in frames if id(f) in ids]
