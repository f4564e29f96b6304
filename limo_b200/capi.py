"""ctypes binding of the CUDA library limo_b200/libkba_b200.so (C ABI: include/kba_b200.h).

The product path: there is no CPU fallback.  Importing works without a GPU (symbols can be inspected), but every
computing call fails with KBA_ERR_CUDA when no sm_90 (H100) device is present.
"""
import ctypes as C
import functools
import inspect
import itertools
import os

import numpy as np

from .capi_types import (KbaCameraStepOut, KbaCameraStepRequest, STEP_SOLVE, KbaCounters, KbaCreateOut, KbaCreateRequest, KbaDeactivateOut, KbaDeactivateRequest, KbaDepthEntry, KbaDepthOut, KbaDepthRequest, KbaDrawFn, KbaEvalOut, KbaEvaluateOut, KbaFlowOut, KbaFlowRequest, KbaFrameLidar, KbaFrameStepOut, KbaFrameStepRequest, KbaKfsolveOut, KbaKfsolveRequest, KbaLabelClass, KbaLandmarkWrite, KbaLidarCloud, KbaLidarOptions, KbaLidarView, KbaOptions, KbaPoseWrite, KbaPushRequest, KbaRankedRequest, KbaRankOut, KbaRankRequest, KbaReclaimOut, KbaReclaimRequest, KbaResult, KbaSelectOut, KbaSelectParams, KbaSelectRequest, KbaTracklet,
                         KbaSnapshotHeader, KbaTrackCaps, KbaTrackFrame, KbaTrackRequest, KbaWindow, Result, Window, c_double_p, c_float_p, c_int32_p,
                         c_uint8_p)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KBA_LIB_PATH") or os.path.join(_HERE, "libkba_b200.so")  # KBA_LIB_PATH: instrumented builds
_lib = None

SYMBOLS = ["kba_version", "kba_last_error", "kba_default_options", "kba_create", "kba_destroy", "kba_set_stream",
           "kba_solve_window", "kba_solve_batch", "kba_eval", "kba_batch_create", "kba_batch_upload",
           "kba_batch_solve", "kba_batch_download", "kba_batch_transfer_bytes", "kba_batch_jacobian_pass", "kba_batch_destroy",
           "kba_get_counters", "kba_enable_kernel_timing", "kba_lidar_default_options", "kba_lidar_depth",
           "kba_shard_unique_id", "kba_shard_comm_create", "kba_shard_comm_create_local", "kba_shard_comm_destroy",
           "kba_batch_set_shard",
           "kba_init_landmarks", "kba_track_create", "kba_track_destroy", "kba_track_push_keyframe", "kba_track_drop_keyframe",
           "kba_track_set_landmarks", "kba_track_set_keyframe_pose", "kba_track_set_keyframe_poses", "kba_track_solve", "kba_track_transfer_bytes",
           "kba_track_group_create", "kba_track_group_destroy", "kba_track_group_solve", "kba_track_group_transfer_bytes",
           "kba_track_adjust_pose", "kba_track_group_adjust_pose", "kba_track_select_landmarks", "kba_track_group_select_landmarks",
           "kba_track_create_landmarks", "kba_track_group_create_landmarks", "kba_track_deactivate_keyframes",
           "kba_track_group_deactivate_keyframes", "kba_track_depth_costs", "kba_track_group_depth_costs", "kba_track_frame_flow",
           "kba_track_group_frame_flow", "kba_track_reclaim_landmarks", "kba_track_group_reclaim_landmarks",
           "kba_track_rank_landmarks", "kba_track_group_rank_landmarks", "kba_track_solve_ranked", "kba_track_group_solve_ranked",
           "kba_solve_batch_opts", "kba_batch_solve_opts", "kba_track_group_solve_opts", "kba_track_group_solve_ranked_opts",
           "kba_track_group_adjust_pose_opts", "kba_track_group_push_keyframes", "kba_track_group_drop_keyframes",
           "kba_track_group_set_landmarks", "kba_track_group_set_keyframe_poses", "kba_lidar_depth_batch",
           "kba_lidar_depth_batch_opts", "kba_track_snapshot_size", "kba_track_save", "kba_track_load", "kba_track_clone",
           "kba_track_group_snapshot_sizes", "kba_track_group_save", "kba_track_evaluate", "kba_track_group_evaluate",
           "kba_track_group_evaluate_opts", "kba_track_keyframe_solve", "kba_track_group_keyframe_solve",
           "kba_track_group_keyframe_solve_opts", "kba_track_frame_step", "kba_track_group_frame_step", "kba_track_group_frame_step_opts",
           "kba_track_frame_step_lidar", "kba_track_group_frame_step_lidar", "kba_track_group_frame_step_lidar_opts",
           "kba_track_camera_step", "kba_track_group_camera_step", "kba_track_group_camera_step_opts"]


class KbaError(RuntimeError):
    pass


# LandmarkSparsificationSchemeVoxel::Parameters' bin caps: the defaults of a ranking request
RANK_DEFAULTS = dict(max_near=300, max_middle=300, max_far=300)


def _draw_source(draws):
    """the kba_rank_request draw function of `draws`: a callable n -> n ints, an array consumed from its start, or None (no
    function: a request that needs draws fails)"""
    if draws is None:
        return KbaDrawFn()
    if callable(draws):
        take = draws
    else:
        src = np.ascontiguousarray(draws, dtype=np.int64).ravel()

        def take(n):
            if n > len(src):
                raise ValueError("%d draws asked, %d given" % (n, len(src)))
            return src[:n]

    def fn(_ctx, n, out):
        try:
            v = np.ascontiguousarray(np.asarray(take(int(n)), dtype=np.int64).ravel().astype(np.int32))  # alive until the copy
            if len(v) != n:
                return 1
            C.memmove(out, v.ctypes.data, 4 * int(n))
            return 0
        except Exception:  # a failing source fails the call (KBA_ERR_BAD_ARG), it must not unwind through C
            return 1
    return KbaDrawFn(fn)


# LandmarkSparsificationSchemeVoxel::Parameters' values: the defaults of a selection request
SELECT_DEFAULTS = dict(voxel_size=(1.0, 1.0, 0.5), roi_far=50.0, roi_middle=25.0)


@functools.lru_cache(maxsize=None)
def _records(struct):
    """numpy dtype with the layout of a ctypes mirror, pointers as addresses: arrays of structs filled by numpy"""
    fmt = lambda t: np.uint64 if issubclass(t, (C._Pointer, C.c_void_p)) else np.dtype(t)  # noqa: E731
    return np.dtype(dict(names=[f for f, _ in struct._fields_], formats=[fmt(t) for _, t in struct._fields_],
                         offsets=[getattr(struct, f).offset for f, _ in struct._fields_], itemsize=C.sizeof(struct)))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise KbaError("CUDA library %s is missing: build it with `make -C limo_b200/csrc` (there is no CPU "
                           "fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        vp = C.c_void_p
        L.kba_version.restype = C.c_int
        L.kba_last_error.restype = C.c_char_p
        L.kba_default_options.argtypes = [C.POINTER(KbaOptions)]
        L.kba_create.argtypes = [C.POINTER(vp), C.c_int]
        L.kba_destroy.argtypes = [vp]
        L.kba_destroy.restype = None
        L.kba_set_stream.argtypes = [vp, vp]
        L.kba_solve_window.argtypes = [vp, C.POINTER(KbaWindow), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_solve_batch.argtypes = [vp, C.c_int32, C.POINTER(KbaWindow), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_eval.argtypes = [vp, C.POINTER(KbaWindow), C.POINTER(KbaOptions), C.POINTER(KbaEvalOut)]
        L.kba_batch_create.argtypes = [vp, C.c_int32, C.POINTER(KbaWindow), C.POINTER(vp)]
        L.kba_batch_upload.argtypes = [vp, C.c_int32, C.POINTER(KbaWindow)]
        L.kba_batch_solve.argtypes = [vp, C.POINTER(KbaOptions)]
        L.kba_batch_download.argtypes = [vp, C.POINTER(KbaResult)]
        L.kba_batch_jacobian_pass.argtypes = [vp, C.POINTER(KbaOptions), C.c_int32, C.POINTER(C.c_float)]
        L.kba_batch_transfer_bytes.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.kba_batch_destroy.argtypes = [vp]
        L.kba_batch_destroy.restype = None
        L.kba_get_counters.argtypes = [vp, C.POINTER(KbaCounters), C.c_int]
        L.kba_enable_kernel_timing.argtypes = [vp, C.c_int]
        L.kba_shard_unique_id.argtypes = [C.c_char_p]
        L.kba_shard_comm_create.argtypes = [vp, C.c_int32, C.c_int32, C.c_char_p, C.POINTER(vp)]
        L.kba_shard_comm_create_local.argtypes = [C.POINTER(vp), C.c_int32, C.POINTER(vp)]
        L.kba_shard_comm_destroy.argtypes = [vp]
        L.kba_shard_comm_destroy.restype = None
        L.kba_batch_set_shard.argtypes = [vp, vp, C.c_int32, C.c_int32]
        L.kba_init_landmarks.argtypes = [vp, C.POINTER(KbaWindow), c_double_p, C.POINTER(C.c_uint8), C.POINTER(C.c_float)]
        ip, u8p = C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
        L.kba_track_create.argtypes = [vp, C.POINTER(KbaTrackCaps), C.c_int32, c_double_p, c_double_p, C.POINTER(vp)]
        L.kba_track_destroy.argtypes = [vp]
        L.kba_track_destroy.restype = None
        L.kba_track_push_keyframe.argtypes = [vp, C.c_int32, c_double_p, c_double_p, C.c_int32, ip, ip, C.POINTER(C.c_float),
                                              C.POINTER(C.c_float), C.POINTER(C.c_float)]
        L.kba_track_drop_keyframe.argtypes = [vp, C.c_int32]
        L.kba_track_set_landmarks.argtypes = [vp, C.c_int32, ip, c_double_p, c_double_p]
        L.kba_track_set_keyframe_pose.argtypes = [vp, C.c_int32, c_double_p, c_double_p]
        L.kba_track_set_keyframe_poses.argtypes = [vp, C.c_int32, ip, c_double_p, c_double_p]
        L.kba_track_solve.argtypes = [vp, C.c_int32, ip, u8p, C.c_int32, ip, C.POINTER(KbaWindow), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_track_transfer_bytes.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.kba_track_group_create.argtypes = [vp, C.c_int32, C.POINTER(vp), C.POINTER(vp)]
        L.kba_track_group_destroy.argtypes = [vp]
        L.kba_track_group_destroy.restype = None
        L.kba_track_group_solve.argtypes = [vp, C.POINTER(KbaTrackRequest), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_track_group_transfer_bytes.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.kba_track_adjust_pose.argtypes = [vp, C.POINTER(KbaTrackFrame), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_track_group_adjust_pose.argtypes = [vp, C.POINTER(KbaTrackFrame), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_track_select_landmarks.argtypes = [vp, C.c_int32, ip, C.c_int32, ip, C.POINTER(KbaSelectParams), C.POINTER(KbaSelectOut)]
        L.kba_track_group_select_landmarks.argtypes = [vp, C.POINTER(KbaSelectRequest), C.POINTER(KbaSelectOut)]
        L.kba_track_create_landmarks.argtypes = [vp, C.POINTER(KbaCreateRequest), C.POINTER(KbaCreateOut)]
        L.kba_track_group_create_landmarks.argtypes = [vp, C.POINTER(KbaCreateRequest), C.POINTER(KbaCreateOut)]
        L.kba_track_deactivate_keyframes.argtypes = [vp, C.POINTER(KbaDeactivateRequest), C.POINTER(KbaDeactivateOut)]
        L.kba_track_group_deactivate_keyframes.argtypes = [vp, C.POINTER(KbaDeactivateRequest), C.POINTER(KbaDeactivateOut)]
        L.kba_track_depth_costs.argtypes = [vp, C.POINTER(KbaDepthRequest), C.POINTER(KbaDepthOut)]
        L.kba_track_group_depth_costs.argtypes = [vp, C.POINTER(KbaDepthRequest), C.POINTER(KbaDepthOut)]
        L.kba_track_frame_flow.argtypes = [vp, C.POINTER(KbaFlowRequest), C.POINTER(KbaFlowOut)]
        L.kba_track_group_frame_flow.argtypes = [vp, C.POINTER(KbaFlowRequest), C.POINTER(KbaFlowOut)]
        L.kba_track_reclaim_landmarks.argtypes = [vp, C.POINTER(KbaReclaimRequest), C.POINTER(KbaReclaimOut)]
        L.kba_track_group_reclaim_landmarks.argtypes = [vp, C.POINTER(KbaReclaimRequest), C.POINTER(KbaReclaimOut)]
        L.kba_track_rank_landmarks.argtypes = [vp, C.POINTER(KbaRankRequest), C.POINTER(KbaRankOut)]
        L.kba_track_group_rank_landmarks.argtypes = [vp, C.POINTER(KbaRankRequest), C.POINTER(KbaRankOut)]
        L.kba_track_solve_ranked.argtypes = [vp, C.c_int32, ip, u8p, C.POINTER(KbaWindow), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_track_group_solve_ranked.argtypes = [vp, C.POINTER(KbaRankedRequest), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_solve_batch_opts.argtypes = [vp, C.c_int32, C.POINTER(KbaWindow), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_batch_solve_opts.argtypes = [vp, C.POINTER(KbaOptions)]
        L.kba_track_group_solve_opts.argtypes = [vp, C.POINTER(KbaTrackRequest), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_track_group_solve_ranked_opts.argtypes = [vp, C.POINTER(KbaRankedRequest), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_track_group_adjust_pose_opts.argtypes = [vp, C.POINTER(KbaTrackFrame), C.POINTER(KbaOptions), C.POINTER(KbaResult)]
        L.kba_track_group_push_keyframes.argtypes = [vp, C.POINTER(KbaPushRequest)]
        L.kba_track_group_drop_keyframes.argtypes = [vp, ip]
        L.kba_track_group_set_landmarks.argtypes = [vp, C.POINTER(KbaLandmarkWrite)]
        L.kba_track_group_set_keyframe_poses.argtypes = [vp, C.POINTER(KbaPoseWrite)]
        i64p = C.POINTER(C.c_int64)
        L.kba_track_snapshot_size.argtypes = [vp, i64p]
        L.kba_track_save.argtypes = [vp, vp, C.c_int64]
        L.kba_track_load.argtypes = [vp, vp, C.c_int64, C.POINTER(KbaTrackCaps), C.POINTER(vp)]
        L.kba_track_clone.argtypes = [vp, vp, C.POINTER(KbaTrackCaps), C.POINTER(vp)]
        L.kba_track_group_snapshot_sizes.argtypes = [vp, i64p]
        L.kba_track_group_save.argtypes = [vp, C.POINTER(vp), i64p]
        L.kba_track_evaluate.argtypes = [vp, C.POINTER(KbaTrackRequest), C.POINTER(KbaOptions), C.POINTER(KbaEvaluateOut)]
        for f in (L.kba_track_group_evaluate, L.kba_track_group_evaluate_opts):
            f.argtypes = [vp, C.POINTER(KbaTrackRequest), C.POINTER(KbaOptions), C.POINTER(KbaEvaluateOut)]
        for f in (L.kba_track_keyframe_solve, L.kba_track_group_keyframe_solve, L.kba_track_group_keyframe_solve_opts):
            f.argtypes = [vp, C.POINTER(KbaKfsolveRequest), C.POINTER(KbaOptions), C.POINTER(KbaKfsolveOut), C.POINTER(KbaResult)]
        for f in (L.kba_track_frame_step, L.kba_track_group_frame_step, L.kba_track_group_frame_step_opts):
            f.argtypes = [vp, C.POINTER(KbaFrameStepRequest), C.POINTER(KbaOptions), C.POINTER(KbaFrameStepOut), C.POINTER(KbaResult)]
        for f in (L.kba_track_frame_step_lidar, L.kba_track_group_frame_step_lidar, L.kba_track_group_frame_step_lidar_opts):
            f.argtypes = [vp, C.POINTER(KbaFrameStepRequest), C.POINTER(KbaFrameLidar), C.POINTER(KbaOptions), C.POINTER(KbaFrameStepOut),
                          C.POINTER(KbaResult)]
        for f in (L.kba_track_camera_step, L.kba_track_group_camera_step, L.kba_track_group_camera_step_opts):
            f.argtypes = [vp, C.POINTER(KbaCameraStepRequest), C.POINTER(KbaFrameLidar), C.POINTER(KbaOptions), C.POINTER(KbaOptions),
                          C.POINTER(KbaCameraStepOut), C.POINTER(KbaResult), C.POINTER(KbaResult)]
        L.kba_lidar_default_options.argtypes = [C.POINTER(KbaLidarOptions)]
        L.kba_lidar_default_options.restype = None
        fp = C.POINTER(C.c_float)
        L.kba_lidar_depth.argtypes = [vp, fp, C.c_int32, C.c_int32, c_double_p, c_double_p, fp, C.c_int32,
                                      C.POINTER(KbaLidarOptions), fp, fp]
        for f in (L.kba_lidar_depth_batch, L.kba_lidar_depth_batch_opts):
            f.argtypes = [vp, C.c_int32, C.POINTER(KbaLidarCloud), C.c_int32, C.POINTER(KbaLidarView), C.POINTER(KbaLidarOptions), fp]
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise KbaError("kba_b200 error %d: %s" % (rc, lib().kba_last_error().decode()))


def default_options():
    o = KbaOptions()
    lib().kba_default_options(C.byref(o))
    return o


def _options(opt, n, single, per_unit):
    """(C function, options argument) of a call over n windows, tracks or frames: opt None or one KbaOptions -> the single-options
    function; a sequence with one KbaOptions (or None: the defaults) per unit -> its per-unit form.  A wrong length raises before
    any C call."""
    if opt is None or isinstance(opt, KbaOptions):
        return single, C.byref(opt or default_options())
    opts = list(opt)
    if len(opts) != n:
        raise ValueError("%d option sets for %d windows / tracks" % (len(opts), n))
    return per_unit, (KbaOptions * n)(*[o or default_options() for o in opts])


def lidar_default_options():
    o = KbaLidarOptions()
    lib().kba_lidar_default_options(C.byref(o))
    return o


def _lidar_batch_request(clouds, views, opt):
    """the arguments of kba_lidar_depth_batch(_opts) for Handle.lidar_depth_batch: (C function, clouds array, views array,
    options argument, one depth array per view, the arrays the structs point into).  opt None or one KbaLidarOptions -> the
    single-options function; a sequence with one KbaLidarOptions (or None: the defaults) per view -> the _opts form.  A view
    naming a missing cloud, or an opt sequence of the wrong length, raises before any C call."""
    cl = [np.ascontiguousarray(c, dtype=np.float32) for c in clouds]
    for i, c in enumerate(cl):
        if c.ndim != 2:
            raise ValueError("cloud %d: an [n, stride] array expected, got shape %s" % (i, c.shape))
    carr = (KbaLidarCloud * len(cl))()
    for c, a in zip(carr, cl):
        c.points, c.n_points, c.stride = a.ctypes.data_as(c_float_p), a.shape[0], a.shape[1]
    views = list(views)
    varr = (KbaLidarView * len(views))()
    keep, outs = list(cl), []
    for i, (v, (ci, T, K, uv)) in enumerate(zip(varr, views)):
        if not 0 <= int(ci) < len(cl):
            raise IndexError("view %d names cloud %d, there are %d clouds" % (i, int(ci), len(cl)))
        T = np.ascontiguousarray(T, dtype=np.float64).ravel(); K = np.ascontiguousarray(K, dtype=np.float64).ravel()
        uv = np.ascontiguousarray(uv, dtype=np.float32).reshape(-1, 2)
        if T.size != 7 or K.size != 3:
            raise ValueError("view %d: T_cam_lidar has 7 entries and intr 3, got %d and %d" % (i, T.size, K.size))
        out = np.full(len(uv), -1.0, dtype=np.float32)
        keep += [T, K, uv]
        outs.append(out)
        v.cloud, v.n_features = int(ci), len(uv)
        v.T_cam_lidar, v.intr, v.features_uv = T.ctypes.data_as(c_double_p), K.ctypes.data_as(c_double_p), uv.ctypes.data_as(c_float_p)
        v.depth_out = out.ctypes.data_as(c_float_p) if len(uv) else None  # a view without features sits out
    if opt is None or isinstance(opt, KbaLidarOptions):
        return lib().kba_lidar_depth_batch, carr, varr, C.byref(opt or lidar_default_options()), outs, keep
    opts = list(opt)
    if len(opts) != len(views):
        raise ValueError("%d option sets for %d views" % (len(opts), len(views)))
    return (lib().kba_lidar_depth_batch_opts, carr, varr,
            (KbaLidarOptions * len(opts))(*[o or lidar_default_options() for o in opts]), outs, keep)


class Batch:
    """Windows resident in HBM (kba_batch_*)."""

    def __init__(self, handle, windows):
        self.handle, self.windows = handle, list(windows)
        self._arr = (KbaWindow * len(self.windows))(*[w.c for w in self.windows])
        self._p = C.c_void_p()
        _check(lib().kba_batch_create(handle._p, len(self.windows), self._arr, C.byref(self._p)))

    def upload(self):
        _check(lib().kba_batch_upload(self._p, len(self.windows), self._arr))

    def solve(self, opt=None):
        """opt: one KbaOptions for every window, or a sequence of one per window (kba_batch_solve_opts)"""
        fn, o = _options(opt, len(self.windows), lib().kba_batch_solve, lib().kba_batch_solve_opts)
        _check(fn(self._p, o))

    def download(self, iterations_capacity=0, results=None):
        """results: reuse the buffers of an earlier download (avoids re-allocating numpy arrays every step)"""
        if results is None:
            results = [Result(w, max(iterations_capacity, 1)) for w in self.windows]
            self._res_arr = (KbaResult * len(results))(*[r.c for r in results])
        arr = self._res_arr
        _check(lib().kba_batch_download(self._p, arr))
        for r, c in zip(results, arr):
            r.c = c
        return results

    def set_shard(self, comm, lm_begin, lm_total):
        """this batch holds one rank's shard of a window split by landmark blocks; solve() becomes a collective call"""
        _check(lib().kba_batch_set_shard(self._p, comm._p, int(lm_begin), int(lm_total)))
        self._comm = comm

    def transfer_bytes(self):
        """(host->device bytes of the last upload, device->host bytes of the last download)"""
        a, b = C.c_int64(), C.c_int64()
        _check(lib().kba_batch_transfer_bytes(self._p, C.byref(a), C.byref(b)))
        return a.value, b.value

    def jacobian_pass(self, opt=None, repeats=1):
        ms = C.c_float()
        _check(lib().kba_batch_jacobian_pass(self._p, C.byref(opt or default_options()), repeats, C.byref(ms)))
        return ms.value

    def close(self):
        if self._p:
            lib().kba_batch_destroy(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _arr(a, dtype, *shape):
    """a as a contiguous array of dtype (reshaped to shape, if given); None stays None (a NULL pointer to the C call)"""
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=dtype)
    return a.reshape(shape) if shape else a


_c_int8_p, _depth_p = C.POINTER(C.c_int8), C.POINTER(KbaDepthEntry)


def _p(a, ptype):
    """a's data as the pointer type ptype, for a struct field or an argument; None stays None (NULL)"""
    return None if a is None else a.ctypes.data_as(ptype)


_I7 = [1.0, 0, 0, 0, 0, 0, 0]


def _sel_window(n_kf, n_lm, kf_fixed=None, **scalars):
    """the `sel` window of a solve of the store: it carries the sizes, the scalars and the ground-plane lists, and sizes the
    solve's Result"""
    return Window(np.tile(_I7, (n_kf, 1)), np.zeros(n_kf, np.uint8) if kf_fixed is None else kf_fixed, [[1.0, 0, 0]], [_I7],
                  np.zeros((n_lm, 3)), np.ones(n_lm), np.zeros(n_lm + 1, dtype=np.int32), [], [], [], [], **scalars)


def _filled(res):
    """the result function of a solve into Result res: c is the KbaResult the call filled (res.c, or a group's array entry)"""
    def done(c):
        res.c = c
        return res
    return done


def _idle(Req, n_kf):
    """the entry of a track that sits a group solve (n_kf = 0) or pose-only call (n_kf = 1: its one pose) out: a zeroed request
    and an idle Result"""
    res = Result(_sel_window(n_kf, 0), 1)
    return Req(), res.c, (), _filled(res)


def _select_args(kf_slots, lm_slots, voxel_size=SELECT_DEFAULTS["voxel_size"], roi_far=SELECT_DEFAULTS["roi_far"],
                 roi_middle=SELECT_DEFAULTS["roi_middle"]):
    """a selection's lists and its kba_select_params as 5 doubles (voxel size xyz, roi_far, roi_middle), the struct's layout"""
    vs = np.asarray(voxel_size, np.float64)
    if vs.shape != (3,):
        raise ValueError("voxel_size must have 3 entries")
    prm = np.empty(5, np.float64)
    prm[:3], prm[3], prm[4] = vs, roi_far, roi_middle
    return _arr(kf_slots, np.int32, -1), _arr(lm_slots, np.int32, -1), prm


def _select_outputs(n_cand):
    """the output buffers of a selection over requests of n_cand[i] candidates, shared by the call (a call that succeeds writes
    every entry), each request's offset co[i] in them and its n_near entry, and result(i) -> request i's dict of views"""
    co = [0, *itertools.accumulate(n_cand)]
    N = co[-1]
    bufs = dict(cheiral=np.empty(N + 1, np.uint8), bin=np.empty(N + 1, np.int8), near_order=np.empty(N + 1, np.int32),
                flow=np.empty(N + 1, np.float64), seen=np.empty(N + 1, np.int32))
    n_near = np.zeros(len(n_cand), np.int32)

    def result(i):
        a, b = co[i], co[i + 1]
        return dict(cheiral=bufs["cheiral"][a:b], bin=bufs["bin"][a:b], near_order=bufs["near_order"][a:a + int(n_near[i])],
                    flow=bufs["flow"][a:b], seen=bufs["seen"][a:b])
    return bufs, co, n_near, result


COST_PARTS = ("reprojection", "depth", "ground_plane", "scale", "plane_chain", "total")


def _evaluate_outputs(n_lm, obs_cap, gp_cap):
    """the output struct of an evaluation of n_lm landmarks with room for obs_cap observations and gp_cap ground-plane residuals,
    its arrays, and the function of the filled struct that gives the evaluation's dict of numpy arrays"""
    b = dict(obs_lm=np.empty(obs_cap, np.int32), obs_kf=np.empty(obs_cap, np.int32), obs_cam=np.empty(obs_cap, np.int32),
             residual=np.empty((obs_cap, 3)), rho=np.empty((obs_cap, 2)), trim_repr=np.empty(n_lm), trim_depth=np.empty(n_lm),
             rejected_repr=np.empty(n_lm, np.uint8), rejected_depth=np.empty(n_lm, np.uint8), gp_lm=np.empty(gp_cap, np.int32),
             gp_kf=np.empty(gp_cap, np.int32), gp_weight=np.empty(gp_cap), gp_residual=np.empty(gp_cap))
    o = KbaEvaluateOut(obs_capacity=obs_cap)
    ptr = dict(KbaEvaluateOut._fields_)
    for k, a in b.items():
        setattr(o, k, a.ctypes.data_as(ptr[k]))

    def done(c):
        n, g = c.n_obs, c.n_gp
        r = {k: (a[:n] if k.startswith("obs_") or k in ("residual", "rho") else a[:g] if k.startswith("gp_") else a)
             for k, a in b.items()}
        r.update(n_obs=n, n_gp=g, failed=bool(c.failed), cost=np.array(c.cost[:]))
        r.update(rejected_repr=r["rejected_repr"].astype(bool), rejected_depth=r["rejected_depth"].astype(bool))
        return r
    return o, tuple(b.values()), done


def _frame_lidar_args(cloud, T_cam_lidar, lidar_opt, depths):
    """the lidar part of a frame step request: its cloud, one pose per camera and one KbaLidarOptions per camera (lidar_opt None
    or one KbaLidarOptions: the same for every camera; a sequence: one per camera, None entries the defaults)"""
    cl = np.ascontiguousarray(cloud, dtype=np.float32)
    if cl.ndim != 2 or cl.shape[1] < 3:
        raise ValueError("cloud: an [n, stride >= 3] array expected, got shape %s" % (cl.shape,))
    if T_cam_lidar is None:
        raise ValueError("a cloud needs T_cam_lidar, one 7-vector per camera")
    T = np.ascontiguousarray(T_cam_lidar, dtype=np.float64)
    if T.size == 0 or T.size % 7:
        raise ValueError("T_cam_lidar: one 7-vector per camera, got %d entries" % T.size)
    T = T.reshape(-1, 7)
    if lidar_opt is None or isinstance(lidar_opt, KbaLidarOptions):
        opts = [lidar_opt] * len(T)
    else:
        opts = list(lidar_opt)
        if len(opts) != len(T):
            raise ValueError("%d lidar option sets for %d cameras" % (len(opts), len(T)))
    return dict(cloud=cl, T=T, opts=(KbaLidarOptions * len(T))(*[o or lidar_default_options() for o in opts]), depths=bool(depths))


def _frame_step_args(kf_slots, lm_slot, u, v, run_sel, kf_new, pose7, stamp, stamp_last, critical_quaternion_diff,
                     time_difference_ns, d=None, cam=None, new_slots=(), plane4=None, adjust=True, speed=None, min_median_flow=5.0,
                     cloud=None, T_cam_lidar=None, lidar_opt=None, depths=False):
    """one frame step request's arrays and scalars, checked where the C call would read past an array.  With a cloud the depths
    come from it (the lidar form) and d is not taken."""
    kf, lm, cm, new = _arr(kf_slots, np.int32, -1), _arr(lm_slot, np.int32, -1), _arr(cam, np.int32, -1), _arr(new_slots, np.int32, -1)
    if (d is None) == (cloud is None):
        raise ValueError("a request takes d (the depths) or a lidar cloud, not both")
    lid = None if cloud is None else _frame_lidar_args(cloud, T_cam_lidar, lidar_opt, depths)
    uu, vv, dd = (_arr(x, np.float32, -1) for x in (u, v, d))
    rs = np.ascontiguousarray(np.asarray(run_sel, dtype=bool).ravel().astype(np.uint8))
    n_runs = int(1 + np.count_nonzero(lm[1:] != lm[:-1])) if len(lm) else 0
    if len(rs) != n_runs:
        raise ValueError("run_sel has %d flags for %d runs" % (len(rs), n_runs))
    if any(a is not None and len(a) != len(lm) for a in (cm, uu, vv, dd)):
        raise ValueError("cam, u, v, d must have one entry per measurement")
    pose, pl = _arr(pose7, np.float64, 7), _arr(plane4, np.float64, 4)
    sp = dict(speed_weight=0.0, speed_dt=1.0, speed_v_before=np.zeros(3), speed_T_origin_before=np.zeros(7))
    if speed:
        sp.update(speed_weight=float(speed["weight"]), speed_dt=float(speed["dt"]), speed_v_before=np.asarray(speed["v_before"], np.float64),
                  speed_T_origin_before=np.asarray(speed["T_origin_before"], np.float64))
    return dict(kf=kf, lm=lm, cam=cm, new=new, u=uu, v=vv, d=dd, lidar=lid, run_sel=rs, pose=pose, plane=pl, kf_new=int(kf_new),
                n_sel_runs=int(rs.sum()), adjust=int(bool(adjust)), min_median_flow=float(min_median_flow),
                critical_quaternion_diff=float(critical_quaternion_diff), time_difference_ns=int(time_difference_ns), stamp=int(stamp),
                stamp_last=int(stamp_last), **sp)


def _frame_step_records(fn, requests, capacity, lidar=False, n_cam=None):
    """the request and output arrays of a frame step over requests (None: the track sits out) as numpy records, the KbaResult
    array, the buffers they point into, and result(i, filled KbaResult array) -> request i's dict.  No ctypes object per track
    but its Result.  lidar: every request carries a cloud (the _lidar forms): the kba_frame_lidar records are returned sixth.
    n_cam: the tracks' camera counts, which each request's T_cam_lidar must match (None: not checked)."""
    n = len(requests)
    act = [i for i, r in enumerate(requests) if r is not None]
    args = [_built(fn, i, requests[i], _frame_step_args) for i in act]
    for i, a in zip(act, args):
        if len(a["kf"]) == 0:  # n_kf = 0 would sit the track out: a request without keyframes is an error, as for one track
            raise KbaError("%s: track %d: no keyframes or a negative size" % (fn.__name__, i))
        if (a["lidar"] is not None) != lidar:
            raise ValueError("%s: request %d: %s" % (fn.__name__, i, "no cloud in a lidar call" if lidar else "a cloud in a call without lidar"))
        if lidar and n_cam is not None and len(a["lidar"]["T"]) != n_cam[i]:
            raise ValueError("%s: request %d: T_cam_lidar has %d poses for %d cameras" % (fn.__name__, i, len(a["lidar"]["T"]), n_cam[i]))
    req, out = np.zeros(n, _records(KbaFrameStepRequest)), np.zeros(n, _records(KbaFrameStepOut))
    nk, nm, nn = (np.array([len(a[k]) for a in args], np.int64) for k in ("kf", "lm", "new"))
    has_cam = np.array([a["cam"] is not None for a in args], bool)
    ints = np.concatenate([a["kf"] for a in args] + [a["lm"] for a in args] + [a["cam"] for a in args if a["cam"] is not None] +
                          [a["new"] for a in args] + [np.zeros(1, np.int32)])
    cols = ("u", "v") if lidar else ("u", "v", "d")  # the lidar form reads no d column
    flts = np.concatenate([a[k] for k in cols for a in args] + [np.zeros(1, np.float32)])
    flags = np.concatenate([a["run_sel"] for a in args] + [np.zeros(1, np.uint8)])
    poses = np.concatenate([a["pose"] for a in args] + [np.zeros(0)])
    planes = np.concatenate([a["plane"] for a in args if a["plane"] is not None] + [np.zeros(0)])
    ex = lambda c: np.concatenate(([0], np.cumsum(c)[:-1])).astype(np.int64)  # noqa: E731  exclusive sums
    M, K = int(nm.sum()), int(nk.sum())
    cam_off = K + M + ex(np.where(has_cam, nm, 0))
    req["n_kf"][act], req["n_meas"][act], req["n_new"][act] = nk, nm, nn
    req["kf_slot"][act] = ints.ctypes.data + 4 * ex(nk)
    req["lm_slot"][act] = ints.ctypes.data + 4 * (K + ex(nm))
    req["cam"][act] = np.where(has_cam, ints.ctypes.data + 4 * cam_off, 0)
    req["new_slot"][act] = ints.ctypes.data + 4 * (K + M + int(nm[has_cam].sum()) + ex(nn))
    for j, k in enumerate(cols):
        req[k][act] = flts.ctypes.data + 4 * (j * M + ex(nm))
    req["run_sel"][act] = flags.ctypes.data + ex([len(a["run_sel"]) for a in args])
    req["pose7"][act] = poses.ctypes.data + 56 * np.arange(len(act))
    has_plane = np.array([a["plane"] is not None for a in args], bool)
    req["plane4"][act] = np.where(has_plane, planes.ctypes.data + 32 * ex(has_plane), 0)
    for k in ("kf_new", "adjust", "min_median_flow", "critical_quaternion_diff", "time_difference_ns", "stamp", "stamp_last",
              "speed_weight", "speed_dt", "speed_v_before", "speed_T_origin_before"):
        req[k][act] = [a[k] for a in args]
    match = np.zeros(M + 1, np.int32)
    pos, cflags = np.full((int(nn.sum()) + 1, 3), np.nan), np.zeros(int(nn.sum()) + 1, np.uint8)
    out["match"][act] = match.ctypes.data + 4 * ex(nm)
    out["pos"][act] = pos.ctypes.data + 24 * ex(nn)
    out["flags"][act] = cflags.ctypes.data + ex(nn)
    depth = np.full(M + 1, -1.0, np.float32)
    lid, lkeep = None, ()
    if lidar:
        lid = np.zeros(n, _records(KbaFrameLidar))
        la = [a["lidar"] for a in args]
        lid["points"][act] = [x["cloud"].ctypes.data for x in la]
        lid["n_points"][act] = [x["cloud"].shape[0] for x in la]
        lid["stride"][act] = [x["cloud"].shape[1] for x in la]
        lid["T_cam_lidar"][act] = [x["T"].ctypes.data for x in la]
        lid["opt"][act] = [C.addressof(x["opts"]) for x in la]
        lid["depth_out"][act] = np.where([x["depths"] for x in la], depth.ctypes.data + 4 * ex(nm), 0)
        lkeep = (depth, la)
    ress = (KbaResult * n)()
    results = {}
    for j, i in enumerate(act):
        results[i] = Result(_sel_window(1, args[j]["n_sel_runs"]), capacity)
        ress[i] = results[i].c
    row = dict(zip(act, range(len(act))))
    mo, no = dict(zip(act, ex(nm))), dict(zip(act, ex(nn)))

    def result(i, filled):
        o, j = out[i], row[i]
        res = results[i]
        res.c = filled[i]
        m0, n0 = int(mo[i]), int(no[i])
        picked = bool(o["selected"])
        return dict(n_matched=int(o["n_matched"]), flow_sum=float(o["flow_sum"]), mean_flow_sq=float(o["mean_flow_sq"]),
                    match=match[m0:m0 + nm[j]].copy(), angle=float(o["angle"]), usable_flow=bool(o["usable_flow"]),
                    usable_pose=bool(o["usable_pose"]), usable_time=bool(o["usable_time"]), selected=picked,
                    pos=pos[n0:n0 + nn[j]].copy() if picked else None, flags=cflags[n0:n0 + nn[j]].copy() if picked else None,
                    depth=depth[m0:m0 + nm[j]].copy() if lidar and args[j]["lidar"]["depths"] else None, result=res)
    keep = (ints, flts, flags, poses, planes, match, pos, cflags, lkeep, results)
    return (req, out, ress, keep, result, lid) if lidar else (req, out, ress, keep, result)


class Track:
    """Persistent, device-resident sliding window (kba_track_*): keyframes are uploaded once when pushed, a solve sends only
    the lists of active keyframe slots and selected landmark slots.

    Each store call turns its keywords into C structs in one builder (Track._push_request, ._landmark_write, ._solve_request,
    ...), which TrackGroup also calls, with a group request's keywords.  A builder returns (the request in the group ABI's
    struct, the output struct or None, the arrays both point into -- outputs first -- which must stay alive during the call,
    the function of the filled output struct that gives the call's result, or None).  The selection shares _select_args and
    _select_outputs instead: its group call fills numpy records."""

    def __init__(self, handle, cam_intr, cam_pose, max_keyframes, max_landmarks, max_measurements, win_keyframes,
                 win_landmarks, win_observations, win_ground=0, win_rows=0):
        """win_rows: largest reduced system a solve may need (6 rows per keyframe, 10 with plane blocks, plus one); 0 keeps the
        fused path's limits (30 keyframes, 18 with plane blocks), beyond 184 the track also owns a large-window solver"""
        self.handle = handle
        self._n_sel = None  # size of the track's last ranking (rank_landmarks, alone or in a group): what solve_ranked returns
        self.caps = caps = KbaTrackCaps(max_keyframes, max_landmarks, max_measurements, win_keyframes, win_landmarks, win_observations,
                                        win_ground, win_rows)
        intr = np.ascontiguousarray(cam_intr, dtype=np.float64).reshape(-1, 3)
        pose = np.ascontiguousarray(cam_pose, dtype=np.float64).reshape(-1, 7)
        self.n_cam = len(intr)
        self._p = C.c_void_p()
        _check(lib().kba_track_create(handle._p, C.byref(caps), len(intr), intr.ctypes.data_as(c_double_p),
                                      pose.ctypes.data_as(c_double_p), C.byref(self._p)))

    def _push_request(self, slot, pose7, lm_slot, u, v, d, cam=None, plane4=None):
        pose, pl, lm, cm = _arr(pose7, np.float64), _arr(plane4, np.float64), _arr(lm_slot, np.int32, -1), _arr(cam, np.int32, -1)
        uu, vv, dd = (_arr(x, np.float32) for x in (u, v, d))
        q = KbaPushRequest(int(slot), len(lm), _p(pose, c_double_p), _p(pl, c_double_p), _p(lm, c_int32_p), _p(cm, c_int32_p),
                           _p(uu, c_float_p), _p(vv, c_float_p), _p(dd, c_float_p))
        return q, None, (pose, pl, lm, cm, uu, vv, dd), None

    def push_keyframe(self, slot, pose7, lm_slot, u, v, d, cam=None, plane4=None):
        q, _, _keep, _ = self._push_request(slot, pose7, lm_slot, u, v, d, cam, plane4)
        _check(lib().kba_track_push_keyframe(self._p, q.kf_slot, q.pose7, q.plane4, q.n_meas, q.lm_slot, q.cam, q.u, q.v, q.d))

    def drop_keyframe(self, slot):
        _check(lib().kba_track_drop_keyframe(self._p, int(slot)))

    def _landmark_write(self, lm_slot, pos=None, weight=None):
        lm, p, w = _arr(lm_slot, np.int32, -1), _arr(pos, np.float64, -1, 3), _arr(weight, np.float64)
        q = KbaLandmarkWrite(n=len(lm), lm_slot=_p(lm, c_int32_p), pos3=_p(p, c_double_p), weight=_p(w, c_double_p))
        return q, None, (lm, p, w), None

    def set_landmarks(self, lm_slot, pos=None, weight=None):
        q, _, _keep, _ = self._landmark_write(lm_slot, pos, weight)
        _check(lib().kba_track_set_landmarks(self._p, q.n, q.lm_slot, q.pos3, q.weight))

    def _pose_write(self, kf_slots, pose7s, plane4s=None):
        kf, p, pl = _arr(kf_slots, np.int32, -1), _arr(pose7s, np.float64, -1, 7), _arr(plane4s, np.float64, -1, 4)
        q = KbaPoseWrite(n=len(kf), kf_slot=_p(kf, c_int32_p), pose7s=_p(p, c_double_p), plane4s=_p(pl, c_double_p))
        return q, None, (kf, p, pl), None

    def set_keyframe_poses(self, kf_slots, pose7s, plane4s=None):
        q, _, _keep, _ = self._pose_write(kf_slots, pose7s, plane4s)
        _check(lib().kba_track_set_keyframe_poses(self._p, q.n, q.kf_slot, q.pose7s, q.plane4s))

    def _solve_request(self, capacity, kf_slots, kf_fixed, lm_slots, **scalars):
        """capacity: the Result's iteration records"""
        kf, fx, lm = _arr(kf_slots, np.int32, -1), _arr(kf_fixed, np.uint8), _arr(lm_slots, np.int32, -1)
        sel = _sel_window(len(kf), len(lm), fx, **scalars)
        res = Result(sel, capacity)
        q = KbaTrackRequest(len(kf), _p(kf, c_int32_p), _p(fx, c_uint8_p), len(lm), _p(lm, c_int32_p), C.pointer(sel.c))
        return q, res.c, (kf, fx, lm, sel), _filled(res)

    def solve(self, kf_slots, kf_fixed, lm_slots, opt=None, **scalars):
        """scalars: scale_kf0, scale_kf1, scale_weight, scale_value, plane_reg_weight, plane_dist_fixed, gp_lm, gp_kf, gp_weight.
        gp_lm without gp_kf / gp_weight: candidate ground landmarks (ascending indices into lm_slots), attached on the device
        (kba_track_solve); plane_reg_weight < 0: 10 iff a ground-plane residual is in the window."""
        q, o, _keep, done = self._solve_request(256, kf_slots, kf_fixed, lm_slots, **scalars)
        _check(lib().kba_track_solve(self._p, q.n_kf, q.kf_slot, q.kf_fixed, q.n_lm, q.lm_slot, q.sel, C.byref(opt or default_options()),
                                     C.byref(o)))
        return done(o)

    def _evaluate_request(self, kf_slots, kf_fixed, lm_slots, obs_capacity=None, **scalars):
        """the solve's request (_solve_request) and the outputs of an evaluation of it: obs_capacity observations (default: the
        track's win_observations, which holds any window), win_ground ground-plane residuals"""
        q, _, keep, _ = self._solve_request(1, kf_slots, kf_fixed, lm_slots, **scalars)
        cap = self.caps.win_observations if obs_capacity is None else int(obs_capacity)
        o, bufs, done = _evaluate_outputs(q.n_lm, cap, self.caps.win_ground)
        return q, o, (*bufs, *keep), done

    def evaluate(self, kf_slots, kf_fixed, lm_slots, opt=None, obs_capacity=None, **scalars):
        """residuals, losses, trimming values and decisions and the cost parts of the window Track.solve would build for these
        arguments, at the store's state, without changing it (kba_track_evaluate).  Returns a dict: n_obs, obs_lm, obs_kf, obs_cam,
        residual [n_obs, 3] (u, v, depth before any loss), rho [n_obs, 2] (scaled Cauchy losses), trim_repr, trim_depth,
        rejected_repr, rejected_depth [n_lm], n_gp, gp_lm, gp_kf, gp_weight, gp_residual [n_gp], cost [6] (COST_PARTS), failed."""
        q, o, _keep, done = self._evaluate_request(kf_slots, kf_fixed, lm_slots, obs_capacity, **scalars)
        _check(lib().kba_track_evaluate(self._p, C.byref(q), C.byref(opt or default_options()), C.byref(o)))
        return done(o)

    def _frame_request(self, capacity, pose7, lm_slot, u, v, d, cam=None, speed=None):
        """speed: None or a dict weight, dt, v_before (3), T_origin_before (7) -- the speed_* fields of a window.  The Result
        (capacity iteration records) has one landmark per run of lm_slot."""
        pose, lm, cm = _arr(pose7, np.float64, 7), _arr(lm_slot, np.int32, -1), _arr(cam, np.int32, -1)
        uu, vv, dd = (_arr(x, np.float32) for x in (u, v, d))
        fr = KbaTrackFrame(n_meas=len(lm), pose7=_p(pose, c_double_p), lm_slot=_p(lm, c_int32_p), cam=_p(cm, c_int32_p),
                           u=_p(uu, c_float_p), v=_p(vv, c_float_p), d=_p(dd, c_float_p), speed_weight=0.0, speed_dt=1.0)
        if speed:
            fr.speed_weight, fr.speed_dt = float(speed["weight"]), float(speed["dt"])
            fr.speed_v_before = (C.c_double * 3)(*[float(x) for x in speed["v_before"]])
            fr.speed_T_origin_before = (C.c_double * 7)(*[float(x) for x in speed["T_origin_before"]])
        n_runs = int(1 + np.count_nonzero(lm[1:] != lm[:-1])) if len(lm) else 0
        res = Result(_sel_window(1, n_runs), capacity)
        return fr, res.c, (pose, lm, uu, vv, dd, cm), _filled(res)

    def adjust_pose(self, pose7, lm_slot, u, v, d, cam=None, speed=None, opt=None, iterations_capacity=256):
        """adjustPoseOnly of one frame against this track's store (kba_track_adjust_pose): one free pose, landmarks read by slot
        (lm_slot: one contiguous run per landmark, in the caller's landmark order).  Returns a Result: kf_pose [1, 7],
        lm_rejected [runs], summaries and iterations; the store is not modified."""
        q, o, _keep, done = self._frame_request(iterations_capacity, pose7, lm_slot, u, v, d, cam, speed)
        _check(lib().kba_track_adjust_pose(self._p, C.byref(q), C.byref(opt or default_options()), C.byref(o)))
        return done(o)

    def select_landmarks(self, kf_slots, lm_slots, voxel_size=SELECT_DEFAULTS["voxel_size"], roi_far=SELECT_DEFAULTS["roi_far"],
                         roi_middle=SELECT_DEFAULTS["roi_middle"]):
        """per-landmark quantities of limo's selection chain on this track's store (kba_track_select_landmarks).
        kf_slots: active keyframes in ascending timestamp order; lm_slots: candidates in ascending landmark id order.  The
        defaults are LandmarkSparsificationSchemeVoxel::Parameters'.  Returns a dict of numpy arrays over the candidates:
        cheiral (uint8), bin (int8: 0 near, 1 middle, 2 far, -1 dropped), near_order (int32 candidate indices in ascending voxel
        index), flow (float64, NaN without a value), seen (int32)."""
        kf, lm, prm = _select_args(kf_slots, lm_slots, voxel_size, roi_far, roi_middle)
        b, _co, n_near, result = _select_outputs([len(lm)])
        o = KbaSelectOut(_p(b["cheiral"], c_uint8_p), _p(b["bin"], _c_int8_p), _p(b["near_order"], c_int32_p), _p(n_near, c_int32_p),
                         _p(b["flow"], c_double_p), _p(b["seen"], c_int32_p))
        _check(lib().kba_track_select_landmarks(self._p, len(kf), _p(kf, c_int32_p), len(lm), _p(lm, c_int32_p),
                                                prm.ctypes.data_as(C.POINTER(KbaSelectParams)), C.byref(o)))
        res = result(0)
        res["near_order"] = res["near_order"].copy()
        return res

    def _create_request(self, kf_slots, kf_new, lm_slots):
        kf, lm = _arr(kf_slots, np.int32, -1), _arr(lm_slots, np.int32, -1)
        pos, flags = np.zeros((len(lm), 3), np.float64), np.zeros(len(lm), np.uint8)
        q = KbaCreateRequest(n_kf=len(kf), kf_new=int(kf_new), n_new=len(lm), kf_slot=_p(kf, c_int32_p), lm_slot=_p(lm, c_int32_p))
        return q, KbaCreateOut(_p(pos, c_double_p), _p(flags, c_uint8_p)), (pos, flags, kf, lm), lambda o: (pos, flags)

    def create_landmarks(self, kf_slots, kf_new, lm_slots):
        """push()'s landmark creation on this track's store (kba_track_create_landmarks): kf_slots the active keyframes in
        ascending id order, kf_new the index in kf_slots of the keyframe just pushed, lm_slots the landmarks it measures that do
        not exist yet.  Returns (pos [n, 3] float64, NaN where not created; flags [n] uint8: bit 0 created, bit 1 has depth);
        created landmarks are written into the store with weight 1."""
        q, o, _keep, done = self._create_request(kf_slots, kf_new, lm_slots)
        _check(lib().kba_track_create_landmarks(self._p, C.byref(q), C.byref(o)))
        return done(o)

    def _deactivate_request(self, kf_slots, lm_slots, min_connecting=3, min_window=4, max_window=20):
        kf, lm = _arr(kf_slots, np.int32, -1), _arr(lm_slots, np.int32, -1)
        res = (np.zeros(len(kf), np.uint8), np.zeros(len(kf), np.int32), np.zeros(len(lm), np.uint8))
        q = KbaDeactivateRequest(n_kf=len(kf), n_lm=len(lm), min_connecting=int(min_connecting), min_window=int(min_window),
                                 max_window=int(max_window), kf_slot=_p(kf, c_int32_p), lm_slot=_p(lm, c_int32_p))
        o = KbaDeactivateOut(_p(res[0], c_uint8_p), _p(res[1], c_int32_p), _p(res[2], c_uint8_p))
        return q, o, (*res, kf, lm), lambda o: res

    def deactivate_keyframes(self, kf_slots, lm_slots, min_connecting=3, min_window=4, max_window=20):
        """deactivateKeyframes() on this track's store (kba_track_deactivate_keyframes): kf_slots the active keyframes in ascending
        id order (the last one the newest), lm_slots the active landmarks.  Returns (kf_active [n_kf] uint8, kf_common [n_kf] int32:
        distinct landmarks shared with the newest keyframe, lm_active [n_lm] uint8: measured by a keyframe that stays active)."""
        q, o, _keep, done = self._deactivate_request(kf_slots, lm_slots, min_connecting, min_window, max_window)
        _check(lib().kba_track_deactivate_keyframes(self._p, C.byref(q), C.byref(o)))
        return done(o)

    def _depth_request(self, kf_slots, lm_slots, cap=None):
        kf, lm = _arr(kf_slots, np.int32, -1), _arr(lm_slots, np.int32, -1)
        cap = min(len(kf) * len(lm), 2**31 - 1) if cap is None else int(cap)  # len(kf) * len(lm) bounds the pairs
        off, cand, cost = np.zeros(len(kf) + 1, np.int32), np.zeros(max(cap, 0), np.int32), np.zeros(max(cap, 0), np.float64)
        q = KbaDepthRequest(n_kf=len(kf), n_elig=len(lm), cap=cap, kf_slot=_p(kf, c_int32_p), lm_slot=_p(lm, c_int32_p))
        o = KbaDepthOut(_p(off, c_int32_p), _p(cand, c_int32_p), _p(cost, c_double_p))
        return q, o, (off, cand, cost, kf, lm), lambda o: (off, cand[:off[-1]].copy(), cost[:off[-1]].copy())

    def depth_costs(self, kf_slots, lm_slots, cap=None):
        """The AddDepth scheme's costs on this track's store (kba_track_depth_costs) for limo's sorter: kf_slots the active keyframes
        in ascending id order (FrameIndex i = kf_slots[i]), lm_slots the eligible landmarks in ascending id order.  Returns (off
        [n_kf + 1], cand, cost): keyframe k's eligible landmarks (indices into lm_slots, arena order) and costs at off[k] ..
        off[k + 1).  cap: output capacity (default n_kf * n_elig)."""
        q, o, _keep, done = self._depth_request(kf_slots, lm_slots, cap)
        _check(lib().kba_track_depth_costs(self._p, C.byref(q), C.byref(o)))
        return done(o)

    def _flow_request(self, kf_last, lm_slot, u, v, cam=None, min_median_flow=5.0):
        lm, cm, uu, vv = _arr(lm_slot, np.int32, -1), _arr(cam, np.int32, -1), _arr(u, np.float32), _arr(v, np.float32)
        match = np.zeros(len(lm), np.int32)
        q = KbaFlowRequest(kf_last=int(kf_last), n_meas=len(lm), lm_slot=_p(lm, c_int32_p), cam=_p(cm, c_int32_p),
                           u=_p(uu, c_float_p), v=_p(vv, c_float_p), min_median_flow=float(min_median_flow))

        def done(o):
            return dict(n_matched=o.n_matched, flow_sum=o.flow_sum, mean_flow_sq=o.mean_flow_sq, usable=bool(o.usable), match=match)
        return q, KbaFlowOut(match=_p(match, c_int32_p)), (match, lm, cm, uu, vv), done

    def frame_flow(self, kf_last, lm_slot, u, v, cam=None, min_median_flow=5.0):
        """KeyframeRejectionSchemeFlow's quantity of a new frame against the stored keyframe kf_last, the newest active one
        (kba_track_frame_flow): the frame's measurements whose landmark has a slot, in Keyframe::measurements_ order (runs by
        landmark, ascending id, cameras ascending inside a run).  Returns a dict: n_matched, flow_sum, mean_flow_sq (NaN without a
        match), usable (mean_flow_sq > min_median_flow ** 2) and match [n_meas] (index into kf_last's measurements, -1: none).
        min_median_flow defaults to limo's launch files' 5 px."""
        q, o, _keep, done = self._flow_request(kf_last, lm_slot, u, v, cam, min_median_flow)
        _check(lib().kba_track_frame_flow(self._p, C.byref(q), C.byref(o)))
        return done(o)

    def _reclaim_request(self, lo, hi, evict=False):
        n = max(int(hi) - int(lo), 0)
        slot = np.zeros(n, np.int32)
        pos, weight = (np.zeros((n, 3), np.float64), np.zeros(n, np.float64)) if evict else (None, None)
        o = KbaReclaimOut(free_slot=_p(slot, c_int32_p), pos=_p(pos, c_double_p), weight=_p(weight, c_double_p))

        def done(o):
            k = o.n_free
            return (slot[:k].copy(), pos[:k].copy(), weight[:k].copy()) if evict else slot[:k].copy()
        return KbaReclaimRequest(lo=int(lo), hi=int(hi)), o, (slot, pos, weight), done

    def reclaim_landmarks(self, lo, hi, evict=False):
        """The landmark slots in [lo, hi) that no live keyframe (pushed and not dropped) measures, ascending
        (kba_track_reclaim_landmarks).  Returns the slots, or with evict=True (slots, pos [n, 3], weight [n]): the store's current
        values of those slots, for a caller that restores an evicted landmark later with set_landmarks.  The store is not written:
        a slot handed out again must be written (create_landmarks or set_landmarks) before a call reads it."""
        q, o, _keep, done = self._reclaim_request(lo, hi, evict)
        _check(lib().kba_track_reclaim_landmarks(self._p, C.byref(q), C.byref(o)))
        return done(o)

    def _rank_request(self, kf_slots, lm_slots, elig=None, voxel_size=SELECT_DEFAULTS["voxel_size"], roi_far=SELECT_DEFAULTS["roi_far"],
                      roi_middle=SELECT_DEFAULTS["roi_middle"], max_near=RANK_DEFAULTS["max_near"], max_middle=RANK_DEFAULTS["max_middle"],
                      max_far=RANK_DEFAULTS["max_far"], depth=(), draws=None):
        """its result function keeps the size of the ranking for solve_ranked"""
        kf, lm, prm = _select_args(kf_slots, lm_slots, voxel_size, roi_far, roi_middle)
        n = len(lm)
        el = _arr(elig, np.uint8, n)
        dp = np.ascontiguousarray(np.asarray(depth, dtype=np.int32).reshape(-1, 2))
        cand, cat = np.zeros(n, np.int32), np.zeros(n, np.int8)
        fn = _draw_source(draws)
        q = KbaRankRequest(n_kf=len(kf), n_cand=n, kf_slot=_p(kf, c_int32_p), lm_slot=_p(lm, c_int32_p), elig=_p(el, c_uint8_p),
                           params=prm.ctypes.data, max_near=int(max_near), max_middle=int(max_middle), max_far=int(max_far),
                           n_depth=len(dp), depth=_p(dp, _depth_p), draw=fn)

        def done(o):
            self._n_sel = o.n_sel
            return dict(cand=cand[:o.n_sel].copy(), category=cat[:o.n_sel].copy(), n_ground=o.n_ground, n_draws=o.n_draws)
        return q, KbaRankOut(cand=_p(cand, c_int32_p), category=_p(cat, _c_int8_p)), (cand, cat, kf, lm, el, dp, prm, fn), done

    def rank_landmarks(self, kf_slots, lm_slots, elig=None, draws=None, **kw):
        """The ranked selection of limo's chain on this track's store (kba_track_rank_landmarks): the arguments of select_landmarks,
        elig [n_cand] (the AddDepth comparator per candidate, None: none), the caps max_near / max_middle / max_far, depth: the
        AddDepth (FrameIndex, NumberLandmarks) entries, draws: the middle bin's random source -- a callable n -> n ints, or an
        array whose first n entries are taken (too short: the call fails), or None when no draw can be needed.  Returns a dict:
        cand (ascending candidate indices), category (0 near, 1 middle, 2 far, 3 AddDepth only), n_ground, n_draws.  The track
        keeps the ranking for solve_ranked."""
        q, o, _keep, done = self._rank_request(kf_slots, lm_slots, elig=elig, draws=draws, **kw)
        _check(lib().kba_track_rank_landmarks(self._p, C.byref(q), C.byref(o)))
        return done(o)

    def _ranked_request(self, capacity, kf_slots, kf_fixed, ground=False, **scalars):
        """a solve of this track's last ranking, its Result (capacity iteration records) sized for that ranking"""
        if self._n_sel is None:
            raise KbaError("solve_ranked: the track has no ranking to solve (rank_landmarks)")
        kf, fx = _arr(kf_slots, np.int32, -1), _arr(kf_fixed, np.uint8)
        sel = _sel_window(len(kf), self._n_sel, fx, **scalars)
        if ground:  # the ranking's ground candidates, attached on the device: n_gp > 0 with no lists
            sel.c.n_gp = 1
        res = Result(sel, capacity)
        q = KbaRankedRequest(n_kf=len(kf), kf_slot=_p(kf, c_int32_p), kf_fixed=_p(fx, c_uint8_p), sel=C.addressof(sel.c))
        return q, res.c, (kf, fx, sel), _filled(res)

    def solve_ranked(self, kf_slots, kf_fixed, opt=None, ground=False, **scalars):
        """solve() on this track's last ranking (kba_track_solve_ranked), made by rank_landmarks of this track or of a TrackGroup:
        ground=True attaches its ground candidates on the device; the other scalars as for solve (gp_* lists index the ranking).
        Results come in ranked order, sized for the ranking."""
        q, o, _keep, done = self._ranked_request(256, kf_slots, kf_fixed, ground, **scalars)
        _check(lib().kba_track_solve_ranked(self._p, q.n_kf, q.kf_slot, q.kf_fixed, C.cast(q.sel, C.POINTER(KbaWindow)),
                                            C.byref(opt or default_options()), C.byref(o)))
        return done(o)

    def _keyframe_solve_request(self, capacity, kf_slots, lm_slots, min_connecting=3, min_window=4, max_window=20, lm_ground=None,
                                tracklets=(), label_classes=None, outliers=(), shrubbery_weight=1.0, voxel_size=SELECT_DEFAULTS["voxel_size"],
                                roi_far=SELECT_DEFAULTS["roi_far"], roi_middle=SELECT_DEFAULTS["roi_middle"], max_near=RANK_DEFAULTS["max_near"],
                                max_middle=RANK_DEFAULTS["max_middle"], max_far=RANK_DEFAULTS["max_far"], depth=(), draws=None, ground=False,
                                **scalars):
        """the deactivation's lists, updateLabels' inputs, the ranking's and the solve's keywords.  Returns a builder's four values
        and the KbaResult the call fills (the call has two outputs); the result function takes a group call's filled KbaResult as
        its second argument and keeps the size of the ranking for solve_ranked."""
        kf, lm, prm = _select_args(kf_slots, lm_slots, voxel_size, roi_far, roi_middle)
        K, L = len(kf), len(lm)
        gr = _arr(lm_ground, np.uint8, L)
        # a kba_tracklet is three little-endian int32 words: slot, label, is_outlier (the byte) with its three zero bytes
        trk = np.ascontiguousarray(np.asarray(tracklets, dtype=np.int64).reshape(-1, 3).astype(np.int32))
        if trk.size and (trk[:, 2].min() < 0 or trk[:, 2].max() > 1):
            raise ValueError("tracklet is_outlier must be 0 or 1")
        cls = np.ascontiguousarray(np.array(sorted((label_classes or {}).items()), dtype=np.int32).reshape(-1, 2))
        out_slots = _arr(outliers, np.int32, -1)
        dp = np.ascontiguousarray(np.asarray(depth, dtype=np.int32).reshape(-1, 2))
        fn = _draw_source(draws)
        sel = _sel_window(K, L, **scalars)
        if ground:  # the ranking's ground candidates, attached on the device: n_gp > 0 with no lists
            sel.c.n_gp = 1
        res = Result(sel, capacity)
        bufs = dict(kf_active=np.zeros(K, np.uint8), kf_common=np.zeros(K, np.int32), lm_active=np.zeros(L, np.uint8),
                    lm_outlier=np.zeros(L, np.uint8), lm_ground=np.zeros(L, np.uint8), trk_outlier=np.zeros(len(trk), np.uint8),
                    cand=np.zeros(L, np.int32), category=np.zeros(L, np.int8))
        q = KbaKfsolveRequest(n_kf=K, n_lm=L, min_connecting=int(min_connecting), min_window=int(min_window), max_window=int(max_window),
                              n_trk=len(trk), kf_slot=_p(kf, c_int32_p), lm_slot=_p(lm, c_int32_p), lm_ground=_p(gr, c_uint8_p),
                              trk=_p(trk, C.POINTER(KbaTracklet)), classes=_p(cls, C.POINTER(KbaLabelClass)), n_class=len(cls),
                              n_outlier=len(out_slots), outlier_slot=_p(out_slots, c_int32_p), shrubbery_weight=float(shrubbery_weight),
                              params=prm.ctypes.data, max_near=int(max_near), max_middle=int(max_middle), max_far=int(max_far),
                              n_depth=len(dp), depth=_p(dp, _depth_p), draw=fn, sel=C.addressof(sel.c))
        o = KbaKfsolveOut(kf_active=_p(bufs["kf_active"], c_uint8_p), kf_common=_p(bufs["kf_common"], c_int32_p),
                          lm_active=_p(bufs["lm_active"], c_uint8_p), lm_outlier=_p(bufs["lm_outlier"], c_uint8_p),
                          lm_ground=_p(bufs["lm_ground"], c_uint8_p), trk_outlier=_p(bufs["trk_outlier"], c_uint8_p),
                          rank=KbaRankOut(cand=_p(bufs["cand"], c_int32_p), category=_p(bufs["category"], _c_int8_p)))

        def done(o, c=None):  # c: the KbaResult a group call filled (a single call fills res.c itself)
            r = o.rank
            self._n_sel = r.n_sel
            if c is not None:
                res.c = c
            n_kept = int(bufs["kf_active"].sum())
            res.kf_pose, res.kf_plane = res.kf_pose[:n_kept], res.kf_plane[:n_kept]
            res.lm_pos, res.lm_rejected, res.n_lm = res.lm_pos[:max(r.n_sel, 1)], res.lm_rejected[:max(r.n_sel, 1)], r.n_sel
            out = {k: bufs[k] for k in ("kf_active", "kf_common", "lm_active", "lm_outlier", "lm_ground", "trk_outlier")}
            out.update(cand=bufs["cand"][:r.n_sel].copy(), category=bufs["category"][:r.n_sel].copy(), n_ground=r.n_ground,
                       n_draws=r.n_draws, result=res)
            return out
        return q, o, (*bufs.values(), kf, lm, gr, trk, cls, out_slots, dp, prm, fn, sel, res), done, res.c

    def keyframe_solve(self, kf_slots, lm_slots, opt=None, iterations_capacity=256, **kw):
        """limo's solve block -- deactivateKeyframes, updateLabels and solve() -- as one call (kba_track_keyframe_solve): kf_slots /
        lm_slots the active keyframes and landmarks in ascending id order with the keywords of deactivate_keyframes; lm_ground
        [n_lm] the landmarks' ground flags before the call (None: none); tracklets [(slot or -1, label, is_outlier)];
        label_classes {label: LABEL_* bits}; outliers: the current outlier set's slots; shrubbery_weight; the ranking's keywords
        of rank_landmarks (without lists or elig); ground and the scalar keywords of solve_ranked.  Returns one dict: the
        deactivation's kf_active, kf_common, lm_active; lm_outlier, lm_ground, trk_outlier after the labels; the ranking's cand
        (indices into the still-active, non-outlier landmarks in list order), category, n_ground, n_draws; and result, the ranked
        solve's Result (keyframe arrays for the kept keyframes, landmark arrays in ranked order)."""
        q, o, _keep, done, rc = self._keyframe_solve_request(iterations_capacity, kf_slots, lm_slots, **kw)
        _check(lib().kba_track_keyframe_solve(self._p, C.byref(q), C.byref(opt or default_options()), C.byref(o), C.byref(rc)))
        return done(o)

    def frame_step(self, opt=None, iterations_capacity=256, **kw):
        """limo's frame step -- adjustPoseOnly, KeyframeSelector::select and push() with its new landmarks -- as one call
        (kba_track_frame_step).  Keywords: kf_slots (the active keyframes in ascending id order, the newest last), the frame's
        measurements lm_slot, u, v, d and cam (every run's landmark with a slot; runs as for adjust_pose), run_sel (one flag per
        run: the landmark is in the last selection), kf_new (the free slot the frame is pushed into if selected), new_slots (the
        landmarks to create then), pose7, plane4, adjust (False: the pose is taken as given), speed (as for adjust_pose),
        min_median_flow, critical_quaternion_diff (radians), time_difference_ns, stamp and stamp_last (ns).
        mono-lidar (kba_track_frame_step_lidar): cloud ([n, stride >= 3] float32, xyz first) instead of d, with T_cam_lidar (one
        7-vector per camera, camera <- lidar), lidar_opt (None, one KbaLidarOptions, or one per camera) and depths (True: return
        the depth each measurement got): the measurements' depths come from the cloud on the device.  Returns a dict: the
        flow's n_matched, flow_sum, mean_flow_sq, match; angle; usable_flow, usable_pose, usable_time, selected; pos, flags (the
        creation's, None when not selected); depth (the lidar depths when asked for, else None); result, the adjustment's
        Result."""
        return _frame_step_call(self._p, lib().kba_track_frame_step, lib().kba_track_frame_step_lidar, [kw],
                                C.byref(opt or default_options()), iterations_capacity, [self.n_cam])[0]

    def camera_step(self, opt_adjust=None, opt_solve=None, iterations_capacity=256, **kw):
        """limo's camera callback -- the frame step and, when due, the solve block on the landmarks the push leaves active -- as one
        call (kba_track_camera_step).  Keywords: those of frame_step (d or a cloud), solve ("never", "always", "if_selected"),
        cand_slots / cand_tags / cand_ground (the solve's candidate list: ascending landmark id; tag -2 active before the frame,
        -1 measured by it, k >= 0 new_slots[k]) and the keywords of keyframe_solve but its lists.  opt_adjust, opt_solve: the
        adjustment's and the solve's options.  Returns a dict: step (frame_step's dict), solved, and when solved n_lm, lm_index
        (each candidate's position in the solve's list, or -1) and solve (keyframe_solve's dict, its landmark arrays for the list)."""
        return _camera_step_call(self._p, lib().kba_track_camera_step, [kw], [self], C.byref(opt_adjust or default_options()),
                                 C.byref(opt_solve or default_options()), iterations_capacity)[0]

    def transfer_bytes(self):
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        _check(lib().kba_track_transfer_bytes(self._p, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def snapshot(self):
        """the store as a snapshot (kba_track_save): a numpy uint8 array, read by capi_types.parse_snapshot and Track.load"""
        n = C.c_int64()
        _check(lib().kba_track_snapshot_size(self._p, C.byref(n)))
        buf = np.empty(n.value, np.uint8)
        _check(lib().kba_track_save(self._p, buf.ctypes.data, n.value))
        return buf

    @staticmethod
    def _caps(saved, kw):
        """saved caps (a KbaTrackCaps) with the keyword caps kw changed, or None (the saved caps) without keywords"""
        if not kw:
            return None
        c = KbaTrackCaps.from_buffer_copy(saved)
        for k, v in kw.items():
            if not hasattr(c, k):
                raise TypeError("unknown track cap %r" % k)
            setattr(c, k, int(v))
        return c

    @classmethod
    def _adopt(cls, handle, p, caps, n_cam):
        t = cls.__new__(cls)
        t.handle, t._n_sel, t._p, t.caps, t.n_cam = handle, None, p, caps, n_cam
        return t

    @classmethod
    def load(cls, handle, data, caps=None):
        """A track on handle whose store is the snapshot data (kba_track_load).  caps: None (the saved caps) or a dict of keyword
        caps (max_keyframes, ..., win_rows) that replace the saved ones, e.g. dict(win_keyframes=20) to grow the window."""
        buf = np.ascontiguousarray(np.frombuffer(data, np.uint8) if not isinstance(data, np.ndarray) else data.view(np.uint8).ravel())
        hd = KbaSnapshotHeader.from_buffer_copy(buf[:C.sizeof(KbaSnapshotHeader)].tobytes()) \
            if len(buf) >= C.sizeof(KbaSnapshotHeader) else None
        saved = hd.caps if hd is not None else KbaTrackCaps()
        c = cls._caps(saved, caps or {})
        p = C.c_void_p()
        _check(lib().kba_track_load(handle._p, buf.ctypes.data, len(buf), C.byref(c) if c else None, C.byref(p)))
        return cls._adopt(handle, p, c or KbaTrackCaps.from_buffer_copy(saved), hd.n_cam)  # a snapshot that loads has a header

    def clone(self, handle=None, **caps):
        """a copy of this track on handle (default: this track's handle) with the keyword caps changed (kba_track_clone); on the
        same device the store is copied without a host round trip"""
        h = handle or self.handle
        c = self._caps(self.caps, caps)
        p = C.c_void_p()
        _check(lib().kba_track_clone(self._p, h._p, C.byref(c) if c else None, C.byref(p)))
        return self._adopt(h, p, c or KbaTrackCaps.from_buffer_copy(self.caps), self.n_cam)

    def close(self):
        if self._p:
            lib().kba_track_destroy(self._p)
            self._p = C.c_void_p()


def _built(fn, i, r, build, *args):
    """build(*args, **r): the structs of request r, the i-th of the group call fn.  A key the single call does not take, or a
    malformed argument, raises naming the request."""
    try:
        return build(*args, **r)
    except (TypeError, ValueError) as e:
        raise type(e)("%s: request %d: %s" % (fn.__name__, i, e)) from None


def _frame_step_call(p, fn, fn_lidar, requests, o, capacity, n_cam):
    """a frame step of the track or group p through fn, or through fn_lidar when the requests carry clouds: one result dict per
    request, None for a track that sits out"""
    lidar = any(r is not None and "cloud" in r for r in requests)
    f = fn_lidar if lidar else fn
    req, out, ress, _keep, result, *lid = _frame_step_records(f, requests, capacity, lidar, n_cam)
    args = [req.ctypes.data_as(C.POINTER(KbaFrameStepRequest))] + [x.ctypes.data_as(C.POINTER(KbaFrameLidar)) for x in lid]
    _check(f(p, *args, o, out.ctypes.data_as(C.POINTER(KbaFrameStepOut)), ress))
    return [None if r is None else result(i, ress) for i, r in enumerate(requests)]


_STEP_KEYS = frozenset(inspect.signature(_frame_step_args).parameters)


def _camera_step_solve(track, capacity, kf_slots, kf_new, solve="never", cand_slots=(), cand_tags=(), cand_ground=None, **kw):
    """the solve block's part of one camera step request of track: solve ("never", "always", "if_selected"), the candidates of
    the solve's landmark list (cand_slots in ascending landmark id, cand_tags: -2 active before the frame, -1 measured by it,
    k >= 0 new_slots[k]; cand_ground their is_ground_plane) and the other keywords of Track.keyframe_solve, over the keyframes
    kf_slots followed by kf_new.  Returns (request with its step part zero, output with its step part zero, the KbaResult the
    solve fills, keep, result(out, res_solve) -> (n_lm, lm_index, keyframe_solve's dict))."""
    if solve not in STEP_SOLVE:
        raise ValueError("solve must be one of %s, got %r" % (sorted(STEP_SOLVE), solve))
    if solve == "never":
        return KbaCameraStepRequest(), KbaCameraStepOut(), KbaResult(), (), None
    kf = list(_arr(kf_slots, np.int32, -1)) + [int(kf_new)]
    q, o, kkeep, kdone, krc = track._keyframe_solve_request(capacity, kf, cand_slots, lm_ground=cand_ground, **kw)
    tags = _arr(cand_tags, np.int32, -1)
    if len(tags) != q.n_lm:
        raise ValueError("cand_tags has %d tags for %d candidates" % (len(tags), q.n_lm))
    index = np.full(q.n_lm, -1, np.int32)
    r = KbaCameraStepRequest(solve=STEP_SOLVE[solve], n_cand=q.n_lm, lm_new=_p(tags, c_int32_p))
    for f, _ in KbaKfsolveRequest._fields_:
        if f not in ("n_kf", "n_lm", "kf_slot"):
            setattr(r, f, getattr(q, f))
    out = KbaCameraStepOut(lm_index=_p(index, c_int32_p), solve=o)

    def result(c, res_solve):
        d = kdone(c.solve, res_solve)
        for k in ("lm_active", "lm_outlier", "lm_ground"):
            d[k] = d[k][:c.n_lm].copy()
        return c.n_lm, index.copy(), d
    return r, out, krc, (kkeep, tags, index), result


def _camera_step_call(p, fn, requests, tracks, o_adjust, o_solve, capacity):
    """a camera step of the track or group p through fn: the frame step's records of every request built at once (as for
    frame_step), the solve block's part per request that may solve.  One result dict per request, None for a track that sits
    out.  Every request carries a cloud or none does (the lidar form is the call with lid, the other one without)."""
    n = len(requests)
    steps = [None if r is None else {k: v for k, v in r.items() if k in _STEP_KEYS} for r in requests]
    lidars = {"cloud" in r for r in steps if r is not None}
    if len(lidars) > 1:
        raise ValueError("%s: a call's requests all carry a cloud or none does" % fn.__name__)
    lidar = lidars == {True}
    freq, fout, fress, fkeep, fresult, *flid = _frame_step_records(fn, steps, capacity, lidar, [t.n_cam for t in tracks])
    reqs, outs, rs = (KbaCameraStepRequest * n)(), (KbaCameraStepOut * n)(), (KbaResult * n)()
    keep, done = [], {}
    sq, so = C.sizeof(KbaFrameStepRequest), C.sizeof(KbaFrameStepOut)
    for i, r in enumerate(requests):
        if r is None:
            continue
        rest = {k: v for k, v in r.items() if k not in _STEP_KEYS}
        q, ob, rc, k, d = _built(fn, i, rest, _camera_step_solve, tracks[i], capacity, r.get("kf_slots", ()), r.get("kf_new", 0))
        reqs[i], outs[i], rs[i] = q, ob, rc
        C.memmove(C.addressof(reqs[i]), freq.ctypes.data + sq * i, sq)  # the step part, at offset 0 of both structs
        C.memmove(C.addressof(outs[i]), fout.ctypes.data + so * i, so)
        keep.append(k)
        done[i] = d
    lid = flid[0].ctypes.data_as(C.POINTER(KbaFrameLidar)) if lidar else None
    _check(fn(p, reqs, lid, o_adjust, o_solve, outs, fress, rs))
    results = [None] * n
    for i, r in enumerate(requests):
        if r is None:
            continue
        C.memmove(fout.ctypes.data + so * i, C.addressof(outs[i]), so)
        res = dict(step=fresult(i, fress), solved=bool(outs[i].solved), n_lm=None, lm_index=None, solve=None)
        if outs[i].solved:
            res["n_lm"], res["lm_index"], res["solve"] = done[i](outs[i], rs[i])
        results[i] = res
    del keep, fkeep
    return results


def _no_keyframes(q):  # n_kf = 0 would sit the track out: a request without keyframes is an error, as for one track
    return q.n_kf == 0


class TrackGroup:
    """Several persistent windows solved as one batch (kba_track_group_*): one launch for a window of every track."""

    def __init__(self, handle, tracks):
        self.handle, self.tracks = handle, list(tracks)
        arr = (C.c_void_p * len(self.tracks))(*[t._p.value for t in self.tracks])
        self._p = C.c_void_p()
        _check(lib().kba_track_group_create(handle._p, len(self.tracks), arr, C.byref(self._p)))

    def _call(self, fn, requests, build, Req, Out=None, idle=None, sits_out=None, why=None, opt=()):
        """The group call fn(group, requests, *opt, outputs) with one entry per track, and its results (None for a track that
        sat out).  requests[i] None sits track i out: idle() gives its entry, else it is a zeroed request.  Otherwise requests[i]
        holds the keywords of the single call, and build (a Track builder) makes its entry.  A request that the group call would
        read as a sit-out (sits_out(request)) fails with why, as the single call fails, or without why its result is the one of
        an untouched output, as the single call answers it."""
        assert len(requests) == len(self.tracks)
        n = len(requests)
        reqs, outs = (Req * n)(), (Out * n)() if Out else None
        keep, results, done = [], [None] * n, []  # keep: the arrays the entries point into, alive until the call returns
        for i, r in enumerate(requests):
            if r is None:
                if idle is None:
                    continue
                q, o, k, d = idle()
            else:
                q, o, k, d = _built(fn, i, r, build, self.tracks[i])
                if sits_out is not None and sits_out(q):
                    if why:
                        raise KbaError("%s: track %d: %s" % (fn.__name__, i, why))
                    results[i] = d(Out())
                    continue
            reqs[i] = q
            if Out:
                outs[i] = o
            keep.append(k)
            if d:
                done.append((i, d))
        _check(fn(self._p, reqs, *opt, *([outs] if Out else [])))
        for i, d in done:
            results[i] = d(outs[i])
        return results

    def solve(self, requests, opt=None, iterations_capacity=256):
        """requests: one per track, None (the track sits this solve out) or a dict with the arguments of Track.solve
        (kf_slots, kf_fixed, lm_slots and the scalar keywords).  opt: one KbaOptions, or one per track
        (kba_track_group_solve_opts).  Returns one Result per track."""
        fn, o = _options(opt, len(self.tracks), lib().kba_track_group_solve, lib().kba_track_group_solve_opts)
        return self._call(fn, requests, lambda t, **r: t._solve_request(iterations_capacity, **r), KbaTrackRequest, KbaResult,
                          idle=lambda: _idle(KbaTrackRequest, 0), opt=(o,))

    def evaluate(self, requests, opt=None):
        """one evaluation per track in one launch sequence (kba_track_group_evaluate): requests as for TrackGroup.solve, with the
        keywords of Track.evaluate; opt: one KbaOptions, or one per track (kba_track_group_evaluate_opts).  Returns one dict per
        track (Track.evaluate's), None for a track that sat out."""
        fn, o = _options(opt, len(self.tracks), lib().kba_track_group_evaluate, lib().kba_track_group_evaluate_opts)
        return self._call(fn, requests, lambda t, **r: t._evaluate_request(**r), KbaTrackRequest, KbaEvaluateOut,
                          sits_out=_no_keyframes, why="fewer than 3 keyframes (kba_track_evaluate refuses it with error 3)", opt=(o,))

    def adjust_pose(self, frames, opt=None, iterations_capacity=256):
        """one frame per track in one launch (kba_track_group_adjust_pose): each entry None (the track sits the call out) or a
        dict with the arguments of Track.adjust_pose (pose7, lm_slot, u, v, d, cam, speed).  opt: one KbaOptions, or one per
        track (kba_track_group_adjust_pose_opts).  Returns one Result per track."""
        fn, o = _options(opt, len(self.tracks), lib().kba_track_group_adjust_pose, lib().kba_track_group_adjust_pose_opts)
        return self._call(fn, frames, lambda t, **r: t._frame_request(iterations_capacity, **r), KbaTrackFrame, KbaResult,
                          idle=lambda: _idle(KbaTrackFrame, 1), opt=(o,))

    def select_landmarks(self, requests):
        """the selection quantities of every track in one launch sequence (kba_track_group_select_landmarks): each entry None
        (the track sits the call out) or a dict with the arguments of Track.select_landmarks (kf_slots, lm_slots, voxel_size,
        roi_far, roi_middle).  Returns one dict per track as Track.select_landmarks returns it (its arrays are views of buffers
        shared by the call), None for a track that sat out."""
        # Not _call: the outputs share buffers sized by every request, and the request and output structs are numpy records,
        # filled without a ctypes object per track.  With one KbaSelectRequest and KbaSelectOut per track instead, a group
        # call of 132 tracks took 7.4-8.4 ms against 2.0-2.6 ms at 12 keyframes / 1.1k landmarks, and 14.3-14.7 ms against
        # 19.3-26.3 ms at 20 keyframes / 8k landmarks, a difference not broken down yet (scripts/group_select_bench.py,
        # medians of 30 calls over several runs, NVIDIA H100 80GB HBM3 at a 700 W power limit).
        assert len(requests) == len(self.tracks)
        fn = lib().kba_track_group_select_landmarks
        act = [i for i, r in enumerate(requests) if r is not None]
        args = [_built(fn, i, requests[i], _select_args) for i in act]
        for i, (kf, _lm, _prm) in zip(act, args):
            if len(kf) == 0:  # n_kf = 0 would sit the track out: a request without keyframes is an error, as for one track
                raise KbaError("%s: track %d: no keyframes or a negative size" % (fn.__name__, i))
        n_cand = [0] * len(requests)
        for i, (_kf, lm, _prm) in zip(act, args):
            n_cand[i] = len(lm)
        bufs, co, n_near, result = _select_outputs(n_cand)
        co = np.array(co[:-1], np.int64)[act]  # the candidate offset of each request that runs
        out = np.zeros(len(requests), _records(KbaSelectOut))
        out["n_near"] = n_near.ctypes.data + 4 * np.arange(len(requests))
        for name, a in bufs.items():
            out[name][act] = a.ctypes.data + a.itemsize * co
        nk = np.array([len(kf) for kf, _lm, _prm in args], np.int64)
        lists = np.concatenate([a[0] for a in args] + [a[1] for a in args] + [np.zeros(1, np.int32)])
        prm = np.concatenate([a[2] for a in args] + [np.zeros(0)])
        req = np.zeros(len(requests), _records(KbaSelectRequest))
        req["n_kf"][act], req["n_cand"][act] = nk, [len(lm) for _kf, lm, _prm in args]
        req["kf_slot"][act] = lists.ctypes.data + 4 * np.concatenate(([0], np.cumsum(nk)[:-1]))
        req["lm_slot"][act] = lists.ctypes.data + 4 * (nk.sum() + co)
        req["params"][act] = prm.ctypes.data + C.sizeof(KbaSelectParams) * np.arange(len(act))
        _check(fn(self._p, req.ctypes.data_as(C.POINTER(KbaSelectRequest)), out.ctypes.data_as(C.POINTER(KbaSelectOut))))
        return [None if r is None else result(i) for i, r in enumerate(requests)]

    def create_landmarks(self, requests):
        """push()'s landmark creation for every track in one launch sequence (kba_track_group_create_landmarks): each entry None
        (the track sits the call out) or a dict with the arguments of Track.create_landmarks (kf_slots, kf_new, lm_slots).
        Returns one (pos, flags) per track as Track.create_landmarks returns it, None for a track that sat out."""
        return self._call(lib().kba_track_group_create_landmarks, requests, Track._create_request, KbaCreateRequest, KbaCreateOut,
                          sits_out=_no_keyframes, why="no keyframes or a negative size")

    def deactivate_keyframes(self, requests):
        """deactivateKeyframes() for every track in one launch sequence (kba_track_group_deactivate_keyframes): each entry None (the
        track sits the call out) or a dict with the arguments of Track.deactivate_keyframes.  Returns one (kf_active, kf_common,
        lm_active) per track, None for a track that sat out."""
        return self._call(lib().kba_track_group_deactivate_keyframes, requests, Track._deactivate_request, KbaDeactivateRequest,
                          KbaDeactivateOut, sits_out=_no_keyframes, why="no keyframes or a negative size")

    def depth_costs(self, requests):
        """The AddDepth costs for every track in one launch sequence (kba_track_group_depth_costs): each entry None or a dict with
        the arguments of Track.depth_costs.  Returns one (off, cand, cost) per track, None for a track that sat out."""
        return self._call(lib().kba_track_group_depth_costs, requests, Track._depth_request, KbaDepthRequest, KbaDepthOut,
                          sits_out=_no_keyframes, why="no keyframes or a negative size")

    def frame_flow(self, requests):
        """The flow scheme's quantity for one frame of every track in one launch sequence (kba_track_group_frame_flow): each entry
        None (the track sits the call out) or a dict with the arguments of Track.frame_flow.  Returns one result dict per track,
        None for a track that sat out."""
        return self._call(lib().kba_track_group_frame_flow, requests, Track._flow_request, KbaFlowRequest, KbaFlowOut,
                          idle=lambda: (KbaFlowRequest(kf_last=-1), KbaFlowOut(), (), None), sits_out=lambda q: q.kf_last < 0,
                          why="kf_last not pushed")

    def reclaim_landmarks(self, requests):
        """The free landmark slots of every track in one launch sequence (kba_track_group_reclaim_landmarks): each entry None (the
        track sits the call out) or a dict with the arguments of Track.reclaim_landmarks (lo, hi, evict).  Returns one result per
        track as Track.reclaim_landmarks returns it, None for a track that sat out."""
        # an empty range would sit the track out: its result is the empty one of a single call
        return self._call(lib().kba_track_group_reclaim_landmarks, requests, Track._reclaim_request, KbaReclaimRequest, KbaReclaimOut,
                          sits_out=lambda q: q.hi == q.lo)

    def rank_landmarks(self, requests):
        """The ranked selection of every track in one launch sequence (kba_track_group_rank_landmarks): each entry None (the track
        sits the call out, its ranking kept) or a dict with the arguments of Track.rank_landmarks.  Returns one result dict per
        track, None for a track that sat out."""
        return self._call(lib().kba_track_group_rank_landmarks, requests, Track._rank_request, KbaRankRequest, KbaRankOut,
                          sits_out=_no_keyframes, why="no keyframes or a negative size")

    def solve_ranked(self, requests, opt=None, iterations_capacity=256):
        """solve_ranked for every track as one batch (kba_track_group_solve_ranked): each entry None (the track sits this solve out)
        or a dict with the arguments of Track.solve_ranked (kf_slots, kf_fixed, ground and the scalar keywords).  Returns one
        Result per track, sized for its ranking.  opt: one KbaOptions, or one per track (kba_track_group_solve_ranked_opts)."""
        fn, o = _options(opt, len(self.tracks), lib().kba_track_group_solve_ranked, lib().kba_track_group_solve_ranked_opts)
        return self._call(fn, requests, lambda t, **r: t._ranked_request(iterations_capacity, **r), KbaRankedRequest, KbaResult,
                          idle=lambda: _idle(KbaRankedRequest, 0), opt=(o,))

    def keyframe_solve(self, requests, opt=None, iterations_capacity=256):
        """limo's solve block for every track (kba_track_group_keyframe_solve): each entry None (the track sits the call out) or
        a dict with the arguments of Track.keyframe_solve.  opt: one KbaOptions, or one per track
        (kba_track_group_keyframe_solve_opts).  Returns one result dict per track (Track.keyframe_solve's), None for a track that
        sat out."""
        # Not _call: the call has two output arrays, the dicts and the solve results
        n = len(self.tracks)
        assert len(requests) == n
        fn, o = _options(opt, n, lib().kba_track_group_keyframe_solve, lib().kba_track_group_keyframe_solve_opts)
        reqs, outs, ress = (KbaKfsolveRequest * n)(), (KbaKfsolveOut * n)(), (KbaResult * n)()
        keep, done = [], []
        for i, r in enumerate(requests):
            if r is None:
                continue
            q, ob, k, d, rc = _built(fn, i, r, lambda t, **kw: t._keyframe_solve_request(iterations_capacity, **kw), self.tracks[i])
            if _no_keyframes(q):
                raise KbaError("%s: track %d: no keyframes or a negative size" % (fn.__name__, i))
            reqs[i], outs[i], ress[i] = q, ob, rc
            keep.append(k)
            done.append((i, d))
        _check(fn(self._p, reqs, o, outs, ress))
        results = [None] * n
        for i, d in done:
            results[i] = d(outs[i], ress[i])
        return results

    def frame_step(self, requests, opt=None, iterations_capacity=256):
        """limo's frame step for every track (kba_track_group_frame_step): each entry None (the track sits the call out) or a dict
        with the keywords of Track.frame_step.  opt: one KbaOptions, or one per track (kba_track_group_frame_step_opts).  Returns
        one result dict per track (Track.frame_step's), None for a track that sat out."""
        # Not _call: the request and output structs are numpy records, filled without a ctypes object per track
        assert len(requests) == len(self.tracks)
        L = lib()
        fn, o = _options(opt, len(self.tracks), L.kba_track_group_frame_step, L.kba_track_group_frame_step_opts)
        fn_lidar, _ = _options(opt, len(self.tracks), L.kba_track_group_frame_step_lidar, L.kba_track_group_frame_step_lidar_opts)
        return _frame_step_call(self._p, fn, fn_lidar, requests, o, iterations_capacity, [t.n_cam for t in self.tracks])

    def camera_step(self, requests, opt_adjust=None, opt_solve=None, iterations_capacity=256):
        """limo's camera callback for every track (kba_track_group_camera_step): each entry None (the track sits the call out) or
        a dict with the keywords of Track.camera_step.  opt_adjust, opt_solve: one KbaOptions each, or one per track (both lists:
        kba_track_group_camera_step_opts).  Returns one result dict per track (Track.camera_step's), None for a track that sat
        out."""
        assert len(requests) == len(self.tracks)
        L, n = lib(), len(self.tracks)
        per_track = not (opt_adjust is None or isinstance(opt_adjust, KbaOptions)) or \
            not (opt_solve is None or isinstance(opt_solve, KbaOptions))
        fn = L.kba_track_group_camera_step_opts if per_track else L.kba_track_group_camera_step
        if per_track:
            oa = [opt_adjust] * n if opt_adjust is None or isinstance(opt_adjust, KbaOptions) else opt_adjust
            os_ = [opt_solve] * n if opt_solve is None or isinstance(opt_solve, KbaOptions) else opt_solve
            _, o_adjust = _options(list(oa), n, None, fn)
            _, o_solve = _options(list(os_), n, None, fn)
        else:
            o_adjust, o_solve = C.byref(opt_adjust or default_options()), C.byref(opt_solve or default_options())
        return _camera_step_call(self._p, fn, requests, self.tracks, o_adjust, o_solve, iterations_capacity)

    def push_keyframes(self, requests):
        """one keyframe into every track's store in one call (kba_track_group_push_keyframes): each entry None (the track sits the
        call out) or a dict with the arguments of Track.push_keyframe (slot, pose7, lm_slot, u, v, d and optionally cam, plane4)"""
        self._call(lib().kba_track_group_push_keyframes, requests, Track._push_request, KbaPushRequest,
                   idle=lambda: (KbaPushRequest(kf_slot=-1), None, (), None), sits_out=lambda q: q.kf_slot < 0,
                   why="keyframe slot out of range")

    def drop_keyframes(self, slots):
        """one keyframe slot per track out of its window (kba_track_group_drop_keyframes): None or a negative slot sits out"""
        assert len(slots) == len(self.tracks)
        arr = np.array([-1 if s is None else int(s) for s in slots], dtype=np.int32)
        _check(lib().kba_track_group_drop_keyframes(self._p, arr.ctypes.data_as(c_int32_p)))

    def set_landmarks(self, requests):
        """landmark positions and weights of every track in one call (kba_track_group_set_landmarks): each entry None (the track
        sits the call out) or a dict with the arguments of Track.set_landmarks (lm_slot, and optionally pos, weight)"""
        self._call(lib().kba_track_group_set_landmarks, requests, Track._landmark_write, KbaLandmarkWrite)

    def set_keyframe_poses(self, requests):
        """keyframe poses (and planes) of every track in one call (kba_track_group_set_keyframe_poses): each entry None (the track
        sits the call out) or a dict with the arguments of Track.set_keyframe_poses (kf_slots, pose7s, and optionally plane4s)"""
        self._call(lib().kba_track_group_set_keyframe_poses, requests, Track._pose_write, KbaPoseWrite)

    def snapshot(self, which=None):
        """the snapshots of the tracks in `which` (indices; None: every track) in one call (kba_track_group_save): a list with one
        numpy uint8 array per track, None for a track that sat out"""
        n = len(self.tracks)
        sizes = np.zeros(n, np.int64)
        _check(lib().kba_track_group_snapshot_sizes(self._p, sizes.ctypes.data_as(C.POINTER(C.c_int64))))
        take = set(range(n)) if which is None else {int(i) for i in which}
        out = [np.empty(sizes[i], np.uint8) if i in take else None for i in range(n)]
        bufs = (C.c_void_p * n)(*[None if b is None else b.ctypes.data for b in out])
        _check(lib().kba_track_group_save(self._p, bufs, sizes.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def transfer_bytes(self):
        """(host->device bytes, device->host bytes) of the last group solve, pose-only call, selection, creation, upkeep, flow
        call or store write"""
        a, b = C.c_int64(), C.c_int64()
        _check(lib().kba_track_group_transfer_bytes(self._p, C.byref(a), C.byref(b)))
        return a.value, b.value

    def close(self):
        if self._p:
            lib().kba_track_group_destroy(self._p)
            self._p = C.c_void_p()


SHARD_ID_BYTES = 128


def shard_unique_id():
    """NCCL unique id (bytes) -- create on rank 0 and broadcast to the other ranks"""
    buf = C.create_string_buffer(SHARD_ID_BYTES)
    _check(lib().kba_shard_unique_id(buf))
    return bytes(buf.raw)


class ShardComm:
    """Communicator of the sharded window solve: NCCL, one process per GPU (kba_shard_comm_create is collective over all
    ranks), or in process (ShardComm.local)"""

    def __init__(self, handle, rank, world, unique_id):
        assert len(unique_id) == SHARD_ID_BYTES
        self._p = C.c_void_p()
        self.rank, self.world = rank, world
        _check(lib().kba_shard_comm_create(handle._p, rank, world, C.c_char_p(unique_id), C.byref(self._p)))

    @classmethod
    def local(cls, handles):
        """one communicator per handle, connecting W handles of this process on one device (kba_shard_comm_create_local):
        rank r's batch is solved by handles[r] from its own thread (parallel.solve_sharded_local)"""
        world = len(handles)
        hs = (C.c_void_p * world)(*[h._p.value for h in handles])
        out = (C.c_void_p * world)()
        _check(lib().kba_shard_comm_create_local(hs, world, out))
        comms = []
        for r in range(world):
            c = cls.__new__(cls)
            c._p, c.rank, c.world = C.c_void_p(out[r]), r, world
            comms.append(c)
        return comms

    def close(self):
        if self._p:
            lib().kba_shard_comm_destroy(self._p)
            self._p = C.c_void_p()


class Handle:
    """One solver handle per host thread / GPU (kba_create)."""

    def __init__(self, device=0, stream=None):
        self._p = C.c_void_p()
        _check(lib().kba_create(C.byref(self._p), device))
        if stream is not None:
            _check(lib().kba_set_stream(self._p, C.c_void_p(stream)))

    def default_options(self):
        return default_options()

    def solve_window(self, win, opt=None, iterations_capacity=256):
        res = Result(win, iterations_capacity)
        _check(lib().kba_solve_window(self._p, C.byref(win.c), C.byref(opt or default_options()), C.byref(res.c)))
        return res

    def solve_batch(self, windows, opt=None, iterations_capacity=1):
        """opt: one KbaOptions for every window, or a sequence of one per window (kba_solve_batch_opts)"""
        fn, o = _options(opt, len(windows), lib().kba_solve_batch, lib().kba_solve_batch_opts)
        results = [Result(w, iterations_capacity) for w in windows]
        warr = (KbaWindow * len(windows))(*[w.c for w in windows])
        rarr = (KbaResult * len(windows))(*[r.c for r in results])
        _check(fn(self._p, len(windows), warr, o, rarr))
        for r, c in zip(results, rarr):
            r.c = c
        self._keep = rarr
        return results

    def evaluate(self, win, opt=None):
        n = max(win.n_obs, 1)
        r = np.zeros((n, 3)); jp = np.zeros((n, 3, 6)); jl = np.zeros((n, 3, 3)); cost = np.zeros(1)
        failed = np.zeros(1, dtype=np.int32)
        out = KbaEvalOut()
        out.residual = r.ctypes.data_as(c_double_p); out.jac_pose = jp.ctypes.data_as(c_double_p)
        out.jac_lm = jl.ctypes.data_as(c_double_p); out.cost = cost.ctypes.data_as(c_double_p)
        out.failed = failed.ctypes.data_as(c_int32_p)
        _check(lib().kba_eval(self._p, C.byref(win.c), C.byref(opt or default_options()), C.byref(out)))
        return r[:win.n_obs], jp[:win.n_obs], jl[:win.n_obs], float(cost[0]), int(failed[0])

    def batch(self, windows):
        return Batch(self, windows)

    def init_landmarks(self, win):
        """push() landmark initialisation for every landmark of `win` on the device: (positions, flags, device ms);
        flags bit 0 = created, bit 1 = in front of every observing camera"""
        pos = np.zeros((max(win.n_lm, 1), 3))
        flags = np.zeros(max(win.n_lm, 1), dtype=np.uint8)
        ms = C.c_float()
        _check(lib().kba_init_landmarks(self._p, C.byref(win.c), pos.ctypes.data_as(c_double_p),
                                        flags.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(ms)))
        return pos[:win.n_lm], flags[:win.n_lm], ms.value

    def lidar_depth(self, cloud, T_cam_lidar, intr, features_uv, opt=None):
        """cloud [n, stride>=3] float32, features_uv [m, 2] float32 -> (depth [m] float32 (-1 = none), device ms)"""
        cloud = np.ascontiguousarray(cloud, dtype=np.float32)
        feats = np.ascontiguousarray(features_uv, dtype=np.float32).reshape(-1, 2)
        T = np.ascontiguousarray(T_cam_lidar, dtype=np.float64); K = np.ascontiguousarray(intr, dtype=np.float64)
        out = np.zeros(max(len(feats), 1), dtype=np.float32)
        ms = C.c_float()
        fp = C.POINTER(C.c_float)
        _check(lib().kba_lidar_depth(self._p, cloud.ctypes.data_as(fp), cloud.shape[0], cloud.shape[1],
                                     T.ctypes.data_as(c_double_p), K.ctypes.data_as(c_double_p), feats.ctypes.data_as(fp),
                                     len(feats), C.byref(opt or lidar_default_options()), out.ctypes.data_as(fp),
                                     C.byref(ms)))
        return out[:len(feats)], ms.value

    def lidar_depth_batch(self, clouds, views, opt=None):
        """depths of many views in one call (kba_lidar_depth_batch).  clouds: float32 [n, stride>=3] arrays; views:
        (cloud index, T_cam_lidar, intr, features_uv [m, 2]) each; opt: None, one KbaLidarOptions, or one per view.  ->
        (one float32 depth array [m] per view (-1 = none), device ms)"""
        fn, carr, varr, o, outs, _keep = _lidar_batch_request(clouds, views, opt)
        ms = C.c_float()
        _check(fn(self._p, len(carr), carr, len(varr), varr, o, C.byref(ms)))
        return outs, ms.value

    def counters(self, reset=False):
        c = KbaCounters()
        _check(lib().kba_get_counters(self._p, C.byref(c), 1 if reset else 0))
        return c

    def enable_kernel_timing(self, on=True):
        _check(lib().kba_enable_kernel_timing(self._p, 1 if on else 0))

    def close(self):
        if self._p:
            lib().kba_destroy(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
