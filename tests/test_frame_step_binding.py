"""The frame step's request builder of the Python binding without a GPU: the numpy records of TrackGroup.frame_step and
Track.frame_step point at the request's arrays, field by field, with NULL for what a request leaves out, and a malformed
request is refused before any C call."""
import ctypes as C

import numpy as np
import pytest

from limo_b200 import capi

I7 = [1.0, 0, 0, 0, 0, 0, 0]


def _req(**kw):
    r = dict(kf_slots=[0, 1], lm_slot=[3, 3, 5, 9], cam=[0, 1, 0, 1], u=[1, 2, 3, 4], v=[5, 6, 7, 8], d=[-1, 2, 3, 4], run_sel=[1, 0, 1],
             kf_new=2, new_slots=[9], pose7=[0.5, 0.5, 0.5, 0.5, 1, 2, 3], stamp=7_000, stamp_last=5_000, critical_quaternion_diff=0.03,
             time_difference_ns=400, speed=dict(weight=2.0, dt=0.1, v_before=[1, 2, 3], T_origin_before=I7), min_median_flow=4.0)
    r.update(kw)
    return r


def _ints(addr, n, t=C.c_int32):
    return list((t * n).from_address(int(addr))) if n else []


def test_group_records_point_at_every_array():
    fn = capi.lib().kba_track_group_frame_step
    reqs = [_req(), None, _req(kf_slots=[4], lm_slot=[1, 2], cam=None, u=[9, 8], v=[7, 6], d=[1, 1], run_sel=[0, 0], new_slots=[],
                               plane4=[0, 0, 1, 2], adjust=False, speed=None, kf_new=0)]
    req, out, ress, keep, _result = capi._frame_step_records(fn, reqs, 8)
    assert req.dtype.itemsize == C.sizeof(capi.KbaFrameStepRequest) and out.dtype.itemsize == C.sizeof(capi.KbaFrameStepOut)
    assert list(req["n_kf"]) == [2, 0, 1] and list(req["n_meas"]) == [4, 0, 2] and list(req["n_new"]) == [1, 0, 0]
    assert req[1].tobytes() == bytes(req.dtype.itemsize) and out[1].tobytes() == bytes(out.dtype.itemsize)  # sits out
    r0, r2 = req[0], req[2]
    assert _ints(r0["kf_slot"], 2) == [0, 1] and _ints(r0["lm_slot"], 4) == [3, 3, 5, 9] and _ints(r0["cam"], 4) == [0, 1, 0, 1]
    assert _ints(r0["new_slot"], 1) == [9] and _ints(r0["run_sel"], 3, C.c_uint8) == [1, 0, 1]
    assert _ints(r0["u"], 4, C.c_float) == [1, 2, 3, 4] and _ints(r0["d"], 4, C.c_float) == [-1, 2, 3, 4]
    assert _ints(r0["pose7"], 7, C.c_double) == [0.5, 0.5, 0.5, 0.5, 1, 2, 3] and r0["plane4"] == 0
    assert (r0["kf_new"], r0["adjust"], r0["stamp"], r0["stamp_last"], r0["time_difference_ns"]) == (2, 1, 7000, 5000, 400)
    assert (r0["min_median_flow"], r0["critical_quaternion_diff"], r0["speed_weight"], r0["speed_dt"]) == (4.0, 0.03, 2.0, 0.1)
    assert list(r0["speed_v_before"]) == [1, 2, 3] and list(r0["speed_T_origin_before"]) == I7
    assert _ints(r2["kf_slot"], 1) == [4] and _ints(r2["lm_slot"], 2) == [1, 2] and r2["cam"] == 0
    assert _ints(r2["v"], 2, C.c_float) == [7, 6] and _ints(r2["plane4"], 4, C.c_double) == [0, 0, 1, 2]
    assert (r2["adjust"], r2["speed_weight"]) == (0, 0.0)
    # outputs: the match indices, positions and flags of each request, one Result per request sized for its selected runs
    assert out[0]["match"] != 0 and out[2]["match"] == out[0]["match"] + 16 and out[0]["pos"] != 0 and out[0]["flags"] != 0
    assert ress[0].iterations_capacity == 8 and ress[1].iterations_capacity == 0
    assert keep[-1][0].lm_rejected.shape == (2,) and keep[-1][2].lm_rejected.shape == (1,)


def test_malformed_requests_are_refused_before_the_call():
    fn = capi.lib().kba_track_group_frame_step
    with pytest.raises(ValueError, match="request 0: run_sel has 2 flags for 3 runs"):
        capi._frame_step_records(fn, [_req(run_sel=[1, 1])], 1)
    with pytest.raises(ValueError, match="one entry per measurement"):
        capi._frame_step_records(fn, [_req(u=[1, 2])], 1)
    with pytest.raises(TypeError, match="request 0"):
        capi._frame_step_records(fn, [_req(bogus=1)], 1)
    with pytest.raises(capi.KbaError, match="track 1: no keyframes"):
        capi._frame_step_records(fn, [None, _req(kf_slots=[])], 1)
