"""ctypes mirror of the POD structs in include/kba_b200.h, plus a numpy-backed window container.

Only data layout lives here (no compute): both the product binding (limo_b200.capi) and the test-only oracle
binding (oracle/oracle.py) build their arguments from these types so that they see identical inputs.
"""
import ctypes as C

import numpy as np

KBA_MAX_SOLVES = 8

c_double_p = C.POINTER(C.c_double)
c_float_p = C.POINTER(C.c_float)
c_int32_p = C.POINTER(C.c_int32)
c_uint8_p = C.POINTER(C.c_uint8)


class KbaWindow(C.Structure):
    _fields_ = [
        ("n_kf", C.c_int32), ("n_cam", C.c_int32), ("n_lm", C.c_int32), ("n_obs", C.c_int32), ("n_gp", C.c_int32),
        ("kf_pose", c_double_p), ("kf_fixed", c_uint8_p), ("kf_plane", c_double_p),
        ("cam_intr", c_double_p), ("cam_pose", c_double_p),
        ("lm_pos", c_double_p), ("lm_weight", c_double_p), ("lm_obs_ptr", c_int32_p),
        ("obs_kf", c_int32_p), ("obs_cam", c_int32_p), ("obs_u", c_float_p), ("obs_v", c_float_p), ("obs_d", c_float_p),
        ("gp_lm", c_int32_p), ("gp_kf", c_int32_p), ("gp_weight", c_double_p),
        ("scale_kf0", C.c_int32), ("scale_kf1", C.c_int32), ("scale_weight", C.c_double), ("scale_value", C.c_double),
        ("plane_reg_weight", C.c_double), ("plane_dist_fixed", C.c_uint8), ("landmarks_fixed", C.c_uint8),
        ("reserved_", C.c_uint8 * 6),
        ("speed_kf", C.c_int32), ("reserved2_", C.c_int32), ("speed_weight", C.c_double), ("speed_dt", C.c_double),
        ("speed_v_before", C.c_double * 3), ("speed_T_origin_before", C.c_double * 7),
    ]


class KbaTrackCaps(C.Structure):
    _fields_ = [("max_keyframes", C.c_int32), ("max_landmarks", C.c_int32), ("max_measurements", C.c_int32),
                ("win_keyframes", C.c_int32), ("win_landmarks", C.c_int32), ("win_observations", C.c_int32),
                ("win_ground", C.c_int32), ("win_rows", C.c_int32)]


class KbaTrackRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("kf_slot", c_int32_p), ("kf_fixed", c_uint8_p), ("n_lm", C.c_int32), ("lm_slot", c_int32_p),
                ("sel", C.POINTER(KbaWindow))]


class KbaEvaluateOut(C.Structure):
    _fields_ = [("obs_capacity", C.c_int32), ("n_obs", C.c_int32), ("n_gp", C.c_int32), ("failed", C.c_int32), ("cost", C.c_double * 6),
                ("obs_lm", c_int32_p), ("obs_kf", c_int32_p), ("obs_cam", c_int32_p), ("residual", c_double_p), ("rho", c_double_p),
                ("trim_repr", c_double_p), ("trim_depth", c_double_p), ("rejected_repr", c_uint8_p), ("rejected_depth", c_uint8_p),
                ("gp_lm", c_int32_p), ("gp_kf", c_int32_p), ("gp_weight", c_double_p), ("gp_residual", c_double_p)]


class KbaSelectParams(C.Structure):
    _fields_ = [("voxel_size", C.c_double * 3), ("roi_far", C.c_double), ("roi_middle", C.c_double)]


class KbaSelectOut(C.Structure):
    _fields_ = [("cheiral", C.POINTER(C.c_uint8)), ("bin", C.POINTER(C.c_int8)), ("near_order", c_int32_p), ("n_near", c_int32_p),
                ("flow", c_double_p), ("seen", c_int32_p)]


class KbaSelectRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_cand", C.c_int32), ("kf_slot", c_int32_p), ("lm_slot", c_int32_p),
                ("params", C.POINTER(KbaSelectParams))]


class KbaCreateRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("kf_new", C.c_int32), ("n_new", C.c_int32), ("reserved_", C.c_int32), ("kf_slot", c_int32_p),
                ("lm_slot", c_int32_p)]


class KbaCreateOut(C.Structure):
    _fields_ = [("pos", c_double_p), ("flags", C.POINTER(C.c_uint8))]


class KbaDeactivateRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_lm", C.c_int32), ("min_connecting", C.c_int32), ("min_window", C.c_int32),
                ("max_window", C.c_int32), ("reserved_", C.c_int32), ("kf_slot", c_int32_p), ("lm_slot", c_int32_p)]


class KbaDeactivateOut(C.Structure):
    _fields_ = [("kf_active", C.POINTER(C.c_uint8)), ("kf_common", c_int32_p), ("lm_active", C.POINTER(C.c_uint8))]


class KbaDepthRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_elig", C.c_int32), ("cap", C.c_int32), ("reserved_", C.c_int32), ("kf_slot", c_int32_p),
                ("lm_slot", c_int32_p)]


class KbaDepthOut(C.Structure):
    _fields_ = [("off", c_int32_p), ("cand", c_int32_p), ("cost", c_double_p)]


class KbaFlowRequest(C.Structure):
    _fields_ = [("kf_last", C.c_int32), ("n_meas", C.c_int32), ("lm_slot", c_int32_p), ("cam", c_int32_p), ("u", c_float_p), ("v", c_float_p),
                ("min_median_flow", C.c_double)]


class KbaFlowOut(C.Structure):
    _fields_ = [("n_matched", C.c_int32), ("usable", C.c_uint8), ("reserved_", C.c_uint8 * 3), ("flow_sum", C.c_double),
                ("mean_flow_sq", C.c_double), ("match", c_int32_p)]


class KbaReclaimRequest(C.Structure):
    _fields_ = [("lo", C.c_int32), ("hi", C.c_int32)]


class KbaReclaimOut(C.Structure):
    _fields_ = [("n_free", C.c_int32), ("reserved_", C.c_int32), ("free_slot", c_int32_p), ("pos", c_double_p), ("weight", c_double_p)]


class KbaPushRequest(C.Structure):
    _fields_ = [("kf_slot", C.c_int32), ("n_meas", C.c_int32), ("pose7", c_double_p), ("plane4", c_double_p), ("lm_slot", c_int32_p),
                ("cam", c_int32_p), ("u", c_float_p), ("v", c_float_p), ("d", c_float_p)]


class KbaLandmarkWrite(C.Structure):
    _fields_ = [("n", C.c_int32), ("reserved_", C.c_int32), ("lm_slot", c_int32_p), ("pos3", c_double_p), ("weight", c_double_p)]


class KbaPoseWrite(C.Structure):
    _fields_ = [("n", C.c_int32), ("reserved_", C.c_int32), ("kf_slot", c_int32_p), ("pose7s", c_double_p), ("plane4s", c_double_p)]


# ---- snapshots of a track's store (kba_track_save, include/kba_b200.h) ----------------------------------------------------------
SNAPSHOT_MAGIC = 0x504E534B    # the bytes "KSNP"
SNAPSHOT_VERSION = 1


class KbaSnapshotHeader(C.Structure):
    _fields_ = [("magic", C.c_uint32), ("format_version", C.c_uint32), ("writer_version", C.c_int32), ("n_cam", C.c_int32),
                ("caps", KbaTrackCaps), ("n_keyframes", C.c_int32), ("n_entries", C.c_int32), ("lm_cap", C.c_int32),
                ("reserved_", C.c_int32), ("cam_offset", C.c_int64), ("cam_bytes", C.c_int64), ("kf_offset", C.c_int64),
                ("kf_bytes", C.c_int64), ("meas_offset", C.c_int64), ("meas_bytes", C.c_int64), ("lm_offset", C.c_int64),
                ("lm_bytes", C.c_int64)]


def _align8(b):
    return (b + 7) & ~7


def _snapshot_layout(n_cam, K, M, L):
    """byte offset of every array of a snapshot with these counts, and its end (the layout of include/kba_b200.h)"""
    o = dict(cam_intr=C.sizeof(KbaSnapshotHeader))
    o["cam_pose"] = o["cam_intr"] + 24 * n_cam
    o["slot"] = o["cam_pose"] + 56 * n_cam
    o["count"] = o["slot"] + _align8(4 * K)
    o["pose"] = o["count"] + _align8(4 * K)
    o["plane"] = o["pose"] + 56 * K
    col = _align8(4 * M)
    for i, name in enumerate(("lm", "cam", "u", "v", "d")):
        o[name] = o["plane"] + 32 * K + i * col
    o["pos"] = o["lm"] + 5 * col
    o["weight"] = o["pos"] + 24 * L
    o["end"] = o["weight"] + 8 * L
    return o


def parse_snapshot(data):
    """The contents of a track snapshot (kba_track_save, Track.snapshot) as numpy views of `data`, after the checks kba_track_load
    makes.  Returns a dict: header (the KbaSnapshotHeader), cam_intr [n_cam, 3], cam_pose [n_cam, 7]; the live keyframes in ascending
    slot order: slot, count, pose [K, 7], plane [K, 4]; their measurements in that order: lm, cam, u, v, d [M]; the landmark values
    of every slot: pos [lm_cap, 3], weight [lm_cap].  A malformed snapshot raises ValueError naming the field.  Needs no GPU."""
    buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data.view(np.uint8).ravel()
    if len(buf) < C.sizeof(KbaSnapshotHeader):
        raise ValueError("truncated snapshot: shorter than the header")
    hd = KbaSnapshotHeader.from_buffer_copy(buf[:C.sizeof(KbaSnapshotHeader)].tobytes())
    checks = [("magic", hd.magic == SNAPSHOT_MAGIC), ("format_version", hd.format_version == SNAPSHOT_VERSION),
              ("reserved_", hd.reserved_ == 0), ("n_cam", 1 <= hd.n_cam <= len(buf) // 80),
              ("lm_cap", 1 <= hd.lm_cap == hd.caps.max_landmarks), ("n_keyframes", 0 <= hd.n_keyframes <= hd.caps.max_keyframes),
              ("n_entries", 0 <= hd.n_entries <= hd.caps.max_measurements)]
    for name, ok in checks:
        if not ok:
            raise ValueError("snapshot header: %s" % name)
    K, M, L = hd.n_keyframes, hd.n_entries, hd.lm_cap
    o = _snapshot_layout(hd.n_cam, K, M, L)
    want = dict(cam_offset=o["cam_intr"], cam_bytes=o["slot"] - o["cam_intr"], kf_offset=o["slot"], kf_bytes=o["lm"] - o["slot"],
                meas_offset=o["lm"], meas_bytes=o["pos"] - o["lm"], lm_offset=o["pos"], lm_bytes=o["end"] - o["pos"])
    for name, v in want.items():
        if getattr(hd, name) != v:
            raise ValueError("snapshot header: %s %d, the counts give %d" % (name, getattr(hd, name), v))
    if o["end"] > len(buf):
        raise ValueError("truncated snapshot: %d bytes, the sections end at %d" % (len(buf), o["end"]))

    def arr(name, dtype, n, *shape):
        a = buf[o[name]:o[name] + n * np.dtype(dtype).itemsize].view(dtype)
        return a.reshape(shape) if shape else a
    out = dict(header=hd, cam_intr=arr("cam_intr", np.float64, 3 * hd.n_cam, -1, 3), cam_pose=arr("cam_pose", np.float64, 7 * hd.n_cam, -1, 7),
               slot=arr("slot", np.int32, K), count=arr("count", np.int32, K), pose=arr("pose", np.float64, 7 * K, -1, 7),
               plane=arr("plane", np.float64, 4 * K, -1, 4), lm=arr("lm", np.int32, M), cam=arr("cam", np.int32, M), u=arr("u", np.float32, M),
               v=arr("v", np.float32, M), d=arr("d", np.float32, M), pos=arr("pos", np.float64, 3 * L, -1, 3), weight=arr("weight", np.float64, L))
    s = out["slot"]
    if K and (s.min() < 0 or s.max() >= hd.caps.max_keyframes or np.any(np.diff(s) <= 0)):
        raise ValueError("keyframe slots: not ascending in [0, caps.max_keyframes)")
    if np.any(out["count"] < 0) or int(out["count"].astype(np.int64).sum()) != M:
        raise ValueError("keyframe counts: negative, or their sum is not n_entries = %d" % M)
    if M and (out["lm"].min() < 0 or out["lm"].max() >= L):
        raise ValueError("measurement landmark slot out of [0, lm_cap)")
    if M and (out["cam"].min() < 0 or out["cam"].max() >= hd.n_cam):
        raise ValueError("measurement camera out of [0, n_cam)")
    return out


class KbaDepthEntry(C.Structure):
    _fields_ = [("ind", C.c_int32), ("wanted", C.c_int32)]


# int32_t (*draw)(void* ctx, int32_t n, int32_t* out) of kba_rank_request
KbaDrawFn = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_int32, c_int32_p)


class KbaRankRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_cand", C.c_int32), ("kf_slot", c_int32_p), ("lm_slot", c_int32_p), ("elig", c_uint8_p),
                ("params", C.c_void_p), ("max_near", C.c_int32), ("max_middle", C.c_int32), ("max_far", C.c_int32), ("n_depth", C.c_int32),
                ("depth", C.POINTER(KbaDepthEntry)), ("draw", KbaDrawFn), ("draw_ctx", C.c_void_p)]


class KbaRankOut(C.Structure):
    _fields_ = [("n_sel", C.c_int32), ("n_ground", C.c_int32), ("n_draws", C.c_int32), ("reserved_", C.c_int32), ("cand", c_int32_p),
                ("category", C.POINTER(C.c_int8))]


class KbaRankedRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("reserved_", C.c_int32), ("kf_slot", c_int32_p), ("kf_fixed", c_uint8_p), ("sel", C.c_void_p)]


# kba_label_class.classes bits
LABEL_OUTLIER, LABEL_SHRUBBERY, LABEL_GROUND = 1, 2, 4


class KbaLabelClass(C.Structure):
    _fields_ = [("label", C.c_int32), ("classes", C.c_int32)]


class KbaTracklet(C.Structure):
    _fields_ = [("lm_slot", C.c_int32), ("label", C.c_int32), ("is_outlier", C.c_uint8), ("reserved_", C.c_uint8 * 3)]


class KbaKfsolveRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_lm", C.c_int32), ("min_connecting", C.c_int32), ("min_window", C.c_int32),
                ("max_window", C.c_int32), ("n_trk", C.c_int32), ("kf_slot", c_int32_p), ("lm_slot", c_int32_p), ("lm_ground", c_uint8_p),
                ("trk", C.POINTER(KbaTracklet)), ("classes", C.POINTER(KbaLabelClass)), ("n_class", C.c_int32), ("n_outlier", C.c_int32),
                ("outlier_slot", c_int32_p), ("shrubbery_weight", C.c_double), ("params", C.c_void_p), ("max_near", C.c_int32),
                ("max_middle", C.c_int32), ("max_far", C.c_int32), ("n_depth", C.c_int32), ("depth", C.POINTER(KbaDepthEntry)),
                ("draw", KbaDrawFn), ("draw_ctx", C.c_void_p), ("sel", C.c_void_p)]


class KbaKfsolveOut(C.Structure):
    _fields_ = [("kf_active", c_uint8_p), ("kf_common", c_int32_p), ("lm_active", c_uint8_p), ("lm_outlier", c_uint8_p),
                ("lm_ground", c_uint8_p), ("trk_outlier", c_uint8_p), ("rank", KbaRankOut)]


class KbaTrackFrame(C.Structure):
    _fields_ = [("n_meas", C.c_int32), ("reserved_", C.c_int32), ("pose7", c_double_p), ("lm_slot", c_int32_p), ("cam", c_int32_p),
                ("u", c_float_p), ("v", c_float_p), ("d", c_float_p), ("speed_weight", C.c_double), ("speed_dt", C.c_double),
                ("speed_v_before", C.c_double * 3), ("speed_T_origin_before", C.c_double * 7)]


class KbaFrameStepRequest(C.Structure):
    _fields_ = [("n_kf", C.c_int32), ("n_meas", C.c_int32), ("kf_slot", c_int32_p), ("lm_slot", c_int32_p), ("cam", c_int32_p),
                ("u", c_float_p), ("v", c_float_p), ("d", c_float_p), ("run_sel", c_uint8_p), ("n_new", C.c_int32), ("kf_new", C.c_int32),
                ("new_slot", c_int32_p), ("pose7", c_double_p), ("plane4", c_double_p), ("speed_weight", C.c_double),
                ("speed_dt", C.c_double), ("speed_v_before", C.c_double * 3), ("speed_T_origin_before", C.c_double * 7),
                ("min_median_flow", C.c_double), ("critical_quaternion_diff", C.c_double), ("time_difference_ns", C.c_uint64),
                ("stamp", C.c_uint64), ("stamp_last", C.c_uint64), ("adjust", C.c_uint8), ("reserved_", C.c_uint8 * 7)]


class KbaFrameStepOut(C.Structure):
    _fields_ = [("n_matched", C.c_int32), ("usable_flow", C.c_uint8), ("usable_pose", C.c_uint8), ("usable_time", C.c_uint8),
                ("selected", C.c_uint8), ("flow_sum", C.c_double), ("mean_flow_sq", C.c_double), ("angle", C.c_double),
                ("match", c_int32_p), ("pos", c_double_p), ("flags", c_uint8_p)]


class KbaOptions(C.Structure):
    _fields_ = [
        ("depth_thres", C.c_double), ("reprojection_thres", C.c_double),
        ("depth_quantile", C.c_double), ("reprojection_quantile", C.c_double),
        ("gp_quantile", C.c_double), ("gp_huber", C.c_double),
        ("num_trim_rounds", C.c_int32), ("trim_solver_iterations", C.c_int32),
        ("final_solver_iterations", C.c_int32), ("min_landmarks_for_trimming", C.c_int32),
        ("min_residual_groups", C.c_int32), ("num_rounds_option", C.c_int32),
        ("solver_time_sec", C.c_double),
        ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double),
        ("initial_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
        ("min_trust_region_radius", C.c_double), ("min_relative_decrease", C.c_double),
        ("min_lm_diagonal", C.c_double), ("max_lm_diagonal", C.c_double),
        ("max_consecutive_invalid_steps", C.c_int32), ("precision", C.c_int32),
    ]


class KbaIteration(C.Structure):
    _fields_ = [
        ("cost", C.c_double), ("cost_change", C.c_double), ("gradient_max_norm", C.c_double),
        ("step_norm", C.c_double), ("relative_decrease", C.c_double), ("trust_region_radius", C.c_double),
        ("iteration", C.c_int32), ("solve_index", C.c_int32),
        ("step_is_valid", C.c_int32), ("step_is_successful", C.c_int32),
    ]


class KbaSolveSummary(C.Structure):
    _fields_ = [
        ("initial_cost", C.c_double), ("final_cost", C.c_double),
        ("num_iterations", C.c_int32), ("num_successful_steps", C.c_int32), ("termination", C.c_int32),
        ("num_landmarks", C.c_int32), ("num_residual_blocks", C.c_int32), ("reserved_", C.c_int32),
    ]


class KbaResult(C.Structure):
    _fields_ = [
        ("kf_pose", c_double_p), ("kf_plane", c_double_p), ("lm_pos", c_double_p), ("lm_rejected", c_uint8_p),
        ("iterations", C.POINTER(KbaIteration)), ("iterations_capacity", C.c_int32),
        ("num_iteration_records", C.c_int32), ("num_solves", C.c_int32), ("status", C.c_int32),
        ("solves", KbaSolveSummary * KBA_MAX_SOLVES),
        ("initial_cost", C.c_double), ("final_cost", C.c_double), ("time_sec", C.c_double),
    ]


class KbaEvalOut(C.Structure):
    _fields_ = [
        ("residual", c_double_p), ("jac_pose", c_double_p), ("jac_lm", c_double_p), ("cost", c_double_p),
        ("failed", c_int32_p),
    ]


class KbaCounters(C.Structure):
    _fields_ = [
        ("launches_total", C.c_int64),
        ("launches_jacobian", C.c_int64), ("launches_prep", C.c_int64), ("launches_schur", C.c_int64),
        ("launches_solve", C.c_int64), ("launches_backsub", C.c_int64), ("launches_cost", C.c_int64),
        ("launches_update", C.c_int64), ("launches_trim", C.c_int64),
        ("ms_jacobian", C.c_double), ("jacobian_obs", C.c_int64),
    ]


class KbaLidarOptions(C.Structure):
    _fields_ = [
        ("image_width", C.c_int32), ("image_height", C.c_int32),
        ("rect_width", C.c_double), ("rect_height", C.c_double), ("rect_offset_x", C.c_double), ("rect_offset_y", C.c_double),
        ("hist_bin_width", C.c_double), ("hist_min_count", C.c_int32), ("min_points", C.c_int32),
        ("depth_min", C.c_double), ("depth_max", C.c_double), ("local_rel_tolerance", C.c_double),
        ("triangle_crossnorm_min", C.c_double), ("viewray_plane_min", C.c_double),
    ]


class KbaLidarCloud(C.Structure):
    _fields_ = [("points", c_float_p), ("n_points", C.c_int32), ("stride", C.c_int32)]


class KbaLidarView(C.Structure):
    _fields_ = [
        ("cloud", C.c_int32), ("n_features", C.c_int32), ("T_cam_lidar", c_double_p), ("intr", c_double_p),
        ("features_uv", c_float_p), ("depth_out", c_float_p),
    ]


class KbaFrameLidar(C.Structure):
    _fields_ = [
        ("points", c_float_p), ("n_points", C.c_int32), ("stride", C.c_int32), ("T_cam_lidar", c_double_p),
        ("opt", C.POINTER(KbaLidarOptions)), ("depth_out", c_float_p),
    ]


STEP_SOLVE = {"never": 0, "always": 1, "if_selected": 2}  # KBA_STEP_SOLVE_*


class KbaCameraStepRequest(C.Structure):
    _fields_ = [("step", KbaFrameStepRequest), ("solve", C.c_uint8), ("reserved_", C.c_uint8 * 3), ("n_cand", C.c_int32),
                ("min_connecting", C.c_int32), ("min_window", C.c_int32), ("max_window", C.c_int32), ("n_trk", C.c_int32),
                ("lm_slot", c_int32_p), ("lm_new", c_int32_p), ("lm_ground", c_uint8_p), ("trk", C.POINTER(KbaTracklet)),
                ("classes", C.POINTER(KbaLabelClass)), ("n_class", C.c_int32), ("n_outlier", C.c_int32), ("outlier_slot", c_int32_p),
                ("shrubbery_weight", C.c_double), ("params", C.c_void_p), ("max_near", C.c_int32), ("max_middle", C.c_int32),
                ("max_far", C.c_int32), ("n_depth", C.c_int32), ("depth", C.POINTER(KbaDepthEntry)), ("draw", KbaDrawFn),
                ("draw_ctx", C.c_void_p), ("sel", C.c_void_p)]


class KbaCameraStepOut(C.Structure):
    _fields_ = [("step", KbaFrameStepOut), ("solved", C.c_uint8), ("reserved_", C.c_uint8 * 3), ("n_lm", C.c_int32),
                ("lm_index", c_int32_p), ("solve", KbaKfsolveOut)]


def _ptr(a, ctype):
    if a is None:
        return C.cast(None, C.POINTER(ctype))
    return a.ctypes.data_as(C.POINTER(ctype))


class Window:
    """numpy-backed optimisation window; `.c` is the KbaWindow struct that points into the arrays."""

    def __init__(self, kf_pose, kf_fixed, cam_intr, cam_pose, lm_pos, lm_weight, lm_obs_ptr, obs_kf, obs_u, obs_v,
                 obs_d, obs_cam=None, kf_plane=None, gp_lm=None, gp_kf=None, gp_weight=None, scale_kf0=0,
                 scale_kf1=1, scale_weight=0.0, scale_value=0.0, plane_reg_weight=0.0, plane_dist_fixed=False,
                 landmarks_fixed=False, speed_kf=0, speed_weight=0.0, speed_dt=1.0, speed_v_before=(0, 0, 0),
                 speed_T_origin_before=(1, 0, 0, 0, 0, 0, 0)):
        f64 = lambda a, shape: np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(shape))
        self.kf_pose = f64(kf_pose, (-1, 7))
        self.n_kf = self.kf_pose.shape[0]
        self.kf_fixed = np.ascontiguousarray(np.asarray(kf_fixed, dtype=np.uint8).reshape(self.n_kf))
        self.kf_plane = None if kf_plane is None else f64(kf_plane, (self.n_kf, 4))
        self.cam_intr = f64(cam_intr, (-1, 3))
        self.n_cam = self.cam_intr.shape[0]
        self.cam_pose = f64(cam_pose, (self.n_cam, 7))
        self.lm_pos = f64(lm_pos, (-1, 3))
        self.n_lm = self.lm_pos.shape[0]
        self.lm_weight = f64(lm_weight, (self.n_lm,))
        self.lm_obs_ptr = np.ascontiguousarray(np.asarray(lm_obs_ptr, dtype=np.int32).reshape(self.n_lm + 1))
        self.obs_kf = np.ascontiguousarray(np.asarray(obs_kf, dtype=np.int32).reshape(-1))
        self.n_obs = self.obs_kf.shape[0]
        assert self.n_obs == int(self.lm_obs_ptr[-1]) if self.n_lm else self.n_obs == 0
        self.obs_cam = None if obs_cam is None else np.ascontiguousarray(np.asarray(obs_cam, dtype=np.int32).reshape(self.n_obs))
        f32 = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(self.n_obs))
        self.obs_u, self.obs_v, self.obs_d = f32(obs_u), f32(obs_v), f32(obs_d)
        self.gp_lm = None if gp_lm is None else np.ascontiguousarray(np.asarray(gp_lm, dtype=np.int32).reshape(-1))
        self.n_gp = 0 if self.gp_lm is None else self.gp_lm.shape[0]
        self.gp_kf = None if gp_kf is None else np.ascontiguousarray(np.asarray(gp_kf, dtype=np.int32).reshape(self.n_gp))
        self.gp_weight = None if gp_weight is None else f64(gp_weight, (self.n_gp,))
        self.scale_kf0, self.scale_kf1 = int(scale_kf0), int(scale_kf1)
        self.scale_weight, self.scale_value = float(scale_weight), float(scale_value)
        self.plane_reg_weight = float(plane_reg_weight)
        self.plane_dist_fixed = bool(plane_dist_fixed)
        self.landmarks_fixed = bool(landmarks_fixed)
        self.speed_kf, self.speed_weight, self.speed_dt = int(speed_kf), float(speed_weight), float(speed_dt)
        self.speed_v_before = tuple(float(x) for x in speed_v_before)
        self.speed_T_origin_before = tuple(float(x) for x in speed_T_origin_before)
        self.c = self._make_struct()

    def _make_struct(self):
        w = KbaWindow()
        w.n_kf, w.n_cam, w.n_lm, w.n_obs, w.n_gp = self.n_kf, self.n_cam, self.n_lm, self.n_obs, self.n_gp
        w.kf_pose = _ptr(self.kf_pose, C.c_double)
        w.kf_fixed = _ptr(self.kf_fixed, C.c_uint8)
        w.kf_plane = _ptr(self.kf_plane, C.c_double)
        w.cam_intr = _ptr(self.cam_intr, C.c_double)
        w.cam_pose = _ptr(self.cam_pose, C.c_double)
        w.lm_pos = _ptr(self.lm_pos, C.c_double)
        w.lm_weight = _ptr(self.lm_weight, C.c_double)
        w.lm_obs_ptr = _ptr(self.lm_obs_ptr, C.c_int32)
        w.obs_kf = _ptr(self.obs_kf, C.c_int32)
        w.obs_cam = _ptr(self.obs_cam, C.c_int32)
        w.obs_u = _ptr(self.obs_u, C.c_float)
        w.obs_v = _ptr(self.obs_v, C.c_float)
        w.obs_d = _ptr(self.obs_d, C.c_float)
        w.gp_lm = _ptr(self.gp_lm, C.c_int32)
        w.gp_kf = _ptr(self.gp_kf, C.c_int32)
        w.gp_weight = _ptr(self.gp_weight, C.c_double)
        w.scale_kf0, w.scale_kf1 = self.scale_kf0, self.scale_kf1
        w.scale_weight, w.scale_value = self.scale_weight, self.scale_value
        w.plane_reg_weight = self.plane_reg_weight
        w.plane_dist_fixed = 1 if self.plane_dist_fixed else 0
        w.landmarks_fixed = 1 if self.landmarks_fixed else 0
        w.speed_kf, w.speed_weight, w.speed_dt = self.speed_kf, self.speed_weight, self.speed_dt
        w.speed_v_before = (C.c_double * 3)(*self.speed_v_before)
        w.speed_T_origin_before = (C.c_double * 7)(*self.speed_T_origin_before)
        return w


class Result:
    """Caller-side result buffers for one window."""

    def __init__(self, win, iterations_capacity=256):
        self.kf_pose = np.zeros((win.n_kf, 7))
        self.kf_plane = np.zeros((win.n_kf, 4))
        self.lm_pos = np.zeros((max(win.n_lm, 1), 3))
        self.lm_rejected = np.zeros(max(win.n_lm, 1), dtype=np.uint8)
        self._iters = (KbaIteration * iterations_capacity)()
        r = KbaResult()
        r.kf_pose = _ptr(self.kf_pose, C.c_double)
        r.kf_plane = _ptr(self.kf_plane, C.c_double)
        r.lm_pos = _ptr(self.lm_pos, C.c_double)
        r.lm_rejected = _ptr(self.lm_rejected, C.c_uint8)
        r.iterations = C.cast(self._iters, C.POINTER(KbaIteration))
        r.iterations_capacity = iterations_capacity
        self.c = r
        self.n_lm = win.n_lm

    @property
    def iterations(self):
        return [self._iters[i] for i in range(min(self.c.num_iteration_records, self.c.iterations_capacity))]

    @property
    def solves(self):
        return [self.c.solves[i] for i in range(self.c.num_solves)]
