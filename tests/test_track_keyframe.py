"""Keyframe selection on the device-resident store -- the flow scheme's quantity (kba_track_frame_flow, kba_track_group_frame_flow)
-- against the Python statement of limo's KeyframeSelector (limo_b200/keyframe_selector.py) and the facade's.

test_statement_equals_facade pins the statement to the facade's KeyframeSelector and schemes without a GPU
(tests/cpp/test_facade_keyframe.cpp, host mode) on the closed-loop drives of tests/keyframe_drive.py.  On the GPU the device must
equal the statement bit for bit at every frame: n_matched, flow_sum and mean_flow_sq as bit patterns, the match indices and the
verdict; and the closed loop must pick the same keyframes with the device's flow as with the host's."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from limo_b200.keyframe_selector import (Frame, KeyframeRejectionSchemeFlow, KeyframeSelectionSchemePose, KeyframeSelector,
                                         KeyframeSparsificationSchemeTime, convert_sec, eraseRejected, frame_flow, newest)
from tests.keyframe_drive import KeyframeDrive, selector

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_keyframe")

DRIVES = [dict(seed=1, window=12, rig=True), dict(seed=2, window=12, rig=False), dict(seed=3, window=20, rig=True, n_frames=80),
          dict(seed=4, window=20, rig=False, n_frames=80)]
IDS = lambda kw: "w%d_%s" % (kw["window"], "rig" if kw["rig"] else "mono")  # noqa: E731


def _build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])


def _bits(x):
    return int(np.float64(x).view(np.uint64))


def replay(dr):
    """the drive's closed loop as a caller replays it: per frame k a dict with the buffer's newest keyframe (its index among the
    selected frames, kf, or None), the frame's request (the measurements whose landmark has a slot, in measurements_ order), the
    statement's quantities and verdicts, the expected match indices and the selection"""
    buffer, order, slots = {}, [], set()
    for k, f in enumerate(dr.frames):
        lm, cam, u, v = dr.arena(k)
        st = dict(k=k, kf=None, thr=dr.thr[k])
        sel = selector(dr.thr[k], dr.critical, dr.time_sec)
        st["verdicts"] = [s.isUsable(f, buffer) for s in sel.rejection_schemes_ + sel.selection_schemes_ + sel.sparsification_schemes_]
        st["sel"] = bool(sel.select([f], buffer))
        assert st["sel"] == dr.selected[k]
        if buffer:
            last = newest(buffer)
            i = order.index(last.timestamp_)
            keep = np.array([int(a) in slots for a in lm], bool)
            st.update(kf=i, lm=lm[keep], cam=cam[keep], u=u[keep], v=v[keep], flow=frame_flow(f, last))
            llm, lcam, _, _ = dr.arena(dr.frames.index(last))
            at = {(int(a), int(b)): j for j, (a, b) in enumerate(zip(llm, lcam))}
            st["match"] = np.array([at.get((int(a), int(b)), -1) for a, b in zip(st["lm"], st["cam"])], np.int32)
            st["lacks_slot"] = int((~keep).sum())
        yield st
        if st["sel"]:
            buffer[f.timestamp_] = f
            order.append(f.timestamp_)
            slots |= set(f.measurements_)
            while len(buffer) > dr.window:
                del buffer[min(buffer)]


def _host_line(st):
    n, s, m = st["flow"] if st["kf"] is not None else (-1, 0.0, 0.0)
    return "F %d %d %016x %016x %d %d %d %d" % (st["k"], n, _bits(s), _bits(m), *[int(x) for x in st["verdicts"]], int(st["sel"]))


# ---- CPU: the statement against the facade --------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", DRIVES, ids=IDS)
def test_statement_equals_facade(kw, tmp_path):
    _build()
    dr = KeyframeDrive(**kw)
    path = tmp_path / "drive.txt"
    dr.write(path)
    r = subprocess.run([EXE, "host", str(path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    facade = r.stdout.strip().split("\n")
    steps = list(replay(dr))
    assert facade == [_host_line(st) for st in steps]
    # the cases the drive is built to reach
    seen = dict(below=0, above=0, nan=0, lacks_slot=0, equal=0, by_pose=0, by_time=0, other_camera=0)
    for st in steps:
        if st["kf"] is None:
            continue
        n, s, m = st["flow"]
        flow_ok, pose_ok, time_ok = st["verdicts"]
        seen["nan"] += n == 0 and not flow_ok
        seen["below"] += n > 0 and not flow_ok
        seen["above"] += flow_ok
        seen["lacks_slot"] += st["lacks_slot"] > 0 and n > 0
        seen["equal"] += _bits(m) == _bits(st["thr"] * st["thr"]) and not flow_ok and time_ok
        seen["by_pose"] += st["sel"] and pose_ok and not time_ok
        seen["by_time"] += st["sel"] and time_ok and not pose_ok
        last = dr.frames[[k for k, x in enumerate(dr.selected) if x][st["kf"]]]
        seen["other_camera"] += sum(1 for a, b in zip(st["lm"], st["cam"])
                                    if int(a) in last.measurements_ and int(b) not in last.measurements_[int(a)])
    if not kw["rig"]:
        seen.pop("other_camera")
    assert all(v > 0 for v in seen.values()), seen
    assert dr.equal is not None


def test_reference_selector_test():
    """the reference's KeyframeSelector.process test (keyframe_bundle_adjustment.cpp:613-647): through the facade, and restated on
    the Python statement"""
    _build()
    r = subprocess.run([EXE, "reference"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    sel = KeyframeSelector()
    scheme0 = KeyframeSparsificationSchemeTime(0.5)
    sel.addScheme(scheme0)
    last = {0: Frame(0, [1, 0, 0, 0, 0, 0, 0], {}), 1: Frame(10000, [1, 0, 0, 0, 0, 0, 0], {})}
    f0, f1 = Frame(10000 + convert_sec(1.0), [1, 0, 0, 0, 0, 0, 0], {}), Frame(10000 + convert_sec(0.25), [1, 0, 0, 0, 0, 0, 0], {})
    assert scheme0.isUsable(f0, last) and not scheme0.isUsable(f1, last)
    assert sel.select([f0, f1], last) == [f0]


def test_time_wrap_and_empty_buffers():
    """the time scheme's unsigned difference wraps for an older frame (usable); on an empty buffer the flow and time schemes take
    the frame and the pose scheme does not; a frame without measurements is not usable by the flow scheme"""
    I = [1.0, 0, 0, 0, 0, 0, 0]
    last = {5: Frame(5_000_000_000, I, {1: {0: (10.0, 10.0)}})}
    older = Frame(4_000_000_000, I, {1: {0: (100.0, 10.0)}})
    time, flow, pose = KeyframeSparsificationSchemeTime(0.4), KeyframeRejectionSchemeFlow(5.0), KeyframeSelectionSchemePose(0.03)
    assert time.isUsable(older, last)  # 4e9 - 5e9 wraps to 2^64 - 1e9
    assert not time.isUsable(Frame(5_400_000_000, I, {}), last) and time.isUsable(Frame(5_400_000_001, I, {}), last)
    assert time.time_difference_nano_sec_ == 400_000_000 and convert_sec(0.3) == int(0.3 * 1e9)
    assert flow.isUsable(older, {}) and time.isUsable(older, {}) and not pose.isUsable(older, {})
    assert not flow.isUsable(Frame(6_000_000_000, I, {}), last)
    assert flow.isUsable(older, last)  # 90 px
    n, s, m = frame_flow(Frame(6_000_000_000, I, {2: {0: (1.0, 1.0)}}), last[5])
    assert n == 0 and s == 0.0 and np.isnan(m)
    # eraseRejected compares counters and skips the entry after an erased one
    cur = {0: "a", 1: "b", 2: "c", 3: "d"}
    eraseRejected(cur, {0: "x"})
    assert cur == {0: "a", 2: "c"}
    cur = {0: "a", 1: "b"}
    eraseRejected(cur, {0: "x"})  # the erased entry is the last: the reference's advance would be undefined, this stops
    assert cur == {0: "a"}
    cur = {0: "a"}
    eraseRejected(cur, {})
    assert cur == {}


def test_flow_struct_sizes_match_header(tmp_path):
    """sizeof() of the flow structs as the C compiler sees them == size of the ctypes mirrors"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu\\n",sizeof(kba_flow_request),'
                    'sizeof(kba_flow_out));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    assert [int(x) for x in subprocess.check_output([str(exe)]).split()] == [C.sizeof(T.KbaFlowRequest), C.sizeof(T.KbaFlowOut)]


def test_flow_null_arguments_need_no_device():
    """a null track, group, request or output is KBA_ERR_BAD_ARG before any device work"""
    _build()
    from limo_b200 import capi
    L = capi.lib()
    q, o = capi.KbaFlowRequest(), capi.KbaFlowOut()
    for fn in (L.kba_track_frame_flow, L.kba_track_group_frame_flow):
        assert fn(None, C.byref(q), C.byref(o)) == 1
        assert "null argument" in L.kba_last_error().decode()


# ---- GPU: the device against the statement -------------------------------------------------------------------------------------
def _track(h, dr):
    from limo_b200 import capi
    total = sum(sum(len(o) for o in f.measurements_.values()) for f in dr.frames)
    most = max(sum(len(o) for o in f.measurements_.values()) for f in dr.frames)
    return capi.Track(h, dr.cam_intr, dr.cam_pose, max_keyframes=dr.window + 2, max_landmarks=dr.n_lm, max_measurements=total,
                      win_keyframes=min(dr.window + 1, 30), win_landmarks=64, win_observations=most)


def _push(t, dr, k, n_kf):
    """frame k, the n_kf-th selected one, into slot n_kf % (W + 2) (the keyframe that held it left the buffer long before)"""
    S = dr.window + 2
    if n_kf >= S:
        t.drop_keyframe(n_kf % S)
    lm, cam, u, v = dr.arena(k)
    t.push_keyframe(n_kf % S, dr.frames[k].pose_, lm, u, v, np.full(len(lm), -1, np.float32), cam=cam)


def _request(dr, st):
    return dict(kf_last=st["kf"] % (dr.window + 2), lm_slot=st["lm"], u=st["u"], v=st["v"], cam=st["cam"], min_median_flow=st["thr"])


def _check(st, res):
    n, s, m = st["flow"]
    assert res["n_matched"] == n and _bits(res["flow_sum"]) == _bits(s) and _bits(res["mean_flow_sq"]) == _bits(m), st["k"]
    assert np.array_equal(res["match"], st["match"]), st["k"]
    assert res["usable"] == (m > st["thr"] * st["thr"]) == st["verdicts"][0], st["k"]


@pytest.mark.gpu
@pytest.mark.parametrize("kw", DRIVES, ids=IDS)
def test_flow_matches_statement(kw):
    from limo_b200 import capi
    dr = KeyframeDrive(**kw)
    h = capi.Handle(0)
    t = _track(h, dr)
    n_kf, checked = 0, 0
    for st in replay(dr):
        if st["kf"] is not None:
            res = t.frame_flow(**_request(dr, st))
            h2d, d2h, _ = t.transfer_bytes()
            n = len(st["lm"])
            assert (h2d, d2h) == (16 * n, 4 * n + 24)
            _check(st, res)
            checked += 1
        if st["sel"]:
            _push(t, dr, st["k"], n_kf)
            n_kf += 1
    assert checked == dr.n_frames - 1
    # n_meas == 0 is a valid request without a match
    res = t.frame_flow(0, np.zeros(0, np.int32), np.zeros(0, np.float32), np.zeros(0, np.float32))
    assert res["n_matched"] == 0 and res["flow_sum"] == 0.0 and np.isnan(res["mean_flow_sq"]) and not res["usable"]
    t.close(); h.close()


@pytest.mark.gpu
def test_group_equals_single_calls():
    """a group of heterogeneous tracks (rigs, windows, sizes) with requests sitting out equals the single calls and the
    statement; a group of one equals the single call; the transfer counts follow the header's formulas"""
    from limo_b200 import capi
    h = capi.Handle(0)
    drives = [KeyframeDrive(31, n_frames=40, window=6, rig=True), KeyframeDrive(32, n_frames=50, window=8, rig=False, n_feat=500),
              KeyframeDrive(33, n_frames=30, window=5, rig=True, n_feat=120)]
    steps = [list(replay(dr)) for dr in drives]
    tracks, singles = [_track(h, dr) for dr in drives], [_track(h, dr) for dr in drives]
    n_kf = [0] * len(drives)
    g = capi.TrackGroup(h, tracks)
    one = capi.TrackGroup(h, [singles[0]])
    for k in range(max(dr.n_frames for dr in drives)):
        reqs = []
        for i, dr in enumerate(drives):
            st = steps[i][k] if k < dr.n_frames else None
            reqs.append(None if st is None or st["kf"] is None or (k + i) % 3 == 2 else _request(dr, st))
        out = g.frame_flow(reqs)
        gb = g.transfer_bytes()
        act = [i for i, r in enumerate(reqs) if r is not None]
        for i in range(len(drives)):
            if i not in act:
                assert out[i] is None
                continue
            single = one.frame_flow([reqs[0]])[0] if i == 0 else singles[i].frame_flow(**reqs[i])
            for key in ("n_matched", "usable"):
                assert out[i][key] == single[key]
            for key in ("flow_sum", "mean_flow_sq"):
                assert _bits(out[i][key]) == _bits(single[key])
            assert np.array_equal(out[i]["match"], single["match"])
            _check(steps[i][k], out[i])
        if not act:
            assert gb == (0, 0)
        else:
            R = gb[0] - 16 * sum(len(reqs[i]["lm_slot"]) for i in act)
            assert (R == 0) if len(act) == 1 else (R > 0 and R % (len(act) - 1) == 0)
            assert gb[1] == sum(4 * len(reqs[i]["lm_slot"]) + 24 for i in act)
        for i, dr in enumerate(drives):
            if k < dr.n_frames and steps[i][k]["sel"]:
                _push(tracks[i], dr, k, n_kf[i]); _push(singles[i], dr, k, n_kf[i])
                n_kf[i] += 1
    assert g.frame_flow([None] * 3) == [None] * 3 and g.transfer_bytes() == (0, 0)
    for x in (g, one, *tracks, *singles):
        x.close()
    h.close()


@pytest.mark.gpu
def test_flow_errors_write_nothing():
    """every invalid request fails with its code before anything is written: the outputs of the single call and of every request
    of a group stay as they were; a valid call afterwards equals the statement"""
    from limo_b200 import capi
    dr = KeyframeDrive(41, n_frames=16, window=4, rig=True, n_feat=80)
    steps = list(replay(dr))
    h = capi.Handle(0)
    t, other = _track(h, dr), _track(h, dr)
    g = capi.TrackGroup(h, [other, t])
    n_kf = 0
    for st in steps[:-1]:
        if st["sel"]:
            _push(t, dr, st["k"], n_kf); _push(other, dr, st["k"], n_kf)
            n_kf += 1
    st = steps[-1]
    good = _request(dr, st)
    lm, cam = list(st["lm"]), list(st["cam"])
    j = next(i for i in range(1, len(lm)) if lm[i] != lm[i - 1] and (i + 1 == len(lm) or lm[i + 1] != lm[i]))  # a run of one entry
    runs2 = next(i for i in range(1, len(lm)) if lm[i] == lm[i - 1])  # the second entry of a two-camera run
    S = dr.window + 2
    unpushed = next(s for s in range(S) if s >= n_kf)
    more = dict(good, lm_slot=np.arange(_track_obs(dr) + 1, dtype=np.int32) % dr.n_lm, u=np.zeros(_track_obs(dr) + 1, np.float32),
                v=np.zeros(_track_obs(dr) + 1, np.float32), cam=None)
    bad = [(dict(good, kf_last=unpushed), 1, "kf_last not pushed"), (dict(good, kf_last=S), 1, "kf_last not pushed"),
           (dict(good, lm_slot=np.array(lm[:-1] + [dr.n_lm], np.int32)), 1, "landmark slot out of range"),
           (dict(good, lm_slot=np.array(lm[:-1] + [-1], np.int32)), 1, "landmark slot out of range"),
           (dict(good, cam=np.array(cam[:-1] + [len(dr.cam_pose)], np.int32)), 1, "camera out of range"),
           (dict(good, lm_slot=np.array(lm + [lm[0]], np.int32), cam=np.array(cam + [cam[0]], np.int32), u=np.append(st["u"], 1.0),
                 v=np.append(st["v"], 1.0)), 1, "reappears after its run"),
           (dict(good, cam=np.array(cam[:runs2] + [cam[runs2 - 1]] + cam[runs2 + 1:], np.int32)), 1, "not ascending"),
           (dict(good, lm_slot=np.array(lm[:j] + [lm[j - 1]] + lm[j + 1:], np.int32),
                 cam=np.array(cam[:j] + [cam[j - 1]] + cam[j + 1:], np.int32)), 1, "not ascending"),
           (more, 4, "more measurements than win_observations")]
    L = capi.lib()

    def call(fn, p, reqs):
        qs = [t._flow_request(**r) for r in reqs]
        for q, o, (match, *_keep), _done in qs:
            match[:] = -7
            o.n_matched, o.usable, o.flow_sum, o.mean_flow_sq = 99, 7, 1.5, 2.5
        if len(qs) == 1:
            rc = fn(p, C.byref(qs[0][0]), C.byref(qs[0][1]))
        else:
            rc = fn(p, (capi.KbaFlowRequest * 2)(*[q[0] for q in qs]), (capi.KbaFlowOut * 2)(*[q[1] for q in qs]))
        return rc, qs

    for r, code, msg in bad:
        rc, qs = call(L.kba_track_frame_flow, t._p, [r])
        assert rc == code, msg
        assert msg in L.kba_last_error().decode()
        rc, qs2 = call(L.kba_track_group_frame_flow, g._p, [good, r])
        assert rc == code and re.search("track 1: .*" + msg, L.kba_last_error().decode()), msg
        for _q, o, (match, *_keep), _done in qs + qs2:  # nothing written
            assert (o.n_matched, o.usable, o.flow_sum, o.mean_flow_sq) == (99, 7, 1.5, 2.5) and (match == -7).all()
    q, o, _keep, _done = t._flow_request(**dict(good, kf_last=-1))
    assert L.kba_track_frame_flow(t._p, C.byref(q), C.byref(o)) == 1  # kf_last < 0 sits out only in a group call
    q, o, _keep, _done = t._flow_request(**good)
    q.lm_slot = C.cast(None, C.POINTER(C.c_int32))
    assert L.kba_track_frame_flow(t._p, C.byref(q), C.byref(o)) == 1 and "null argument" in L.kba_last_error().decode()
    q, o, _keep, _done = t._flow_request(**good)
    q.n_meas = -1
    assert L.kba_track_frame_flow(t._p, C.byref(q), C.byref(o)) == 1 and "negative size" in L.kba_last_error().decode()
    for x in (t, other):
        _check(st, x.frame_flow(**good))
    g.close(); t.close(); other.close(); h.close()


def _track_obs(dr):
    return max(sum(len(o) for o in f.measurements_.values()) for f in dr.frames)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", DRIVES[:2], ids=IDS)
def test_closed_loop_device_flow_picks_same_keyframes(kw):
    """the drive's closed loop again, with the flow scheme's quantity taken from the store: the same keyframes"""
    from limo_b200 import capi
    dr = KeyframeDrive(**kw)
    h = capi.Handle(0)
    t = _track(h, dr)
    S = dr.window + 2
    order, slots, n_kf = [], set(), 0

    def device_flow(new_frame, last_keyframe):
        k = dr.frames.index(new_frame)
        lm, cam, u, v = dr.arena(k)
        keep = np.array([int(a) in slots for a in lm], bool)
        r = t.frame_flow(order.index(last_keyframe.timestamp_) % S, lm[keep], u[keep], v[keep], cam=cam[keep], min_median_flow=dr.thr[k])
        return r["n_matched"], r["flow_sum"], r["mean_flow_sq"]

    buffer, picked = {}, []
    for k, f in enumerate(dr.frames):
        keep = bool(selector(dr.thr[k], dr.critical, dr.time_sec, flow_fn=device_flow).select([f], buffer))
        picked.append(keep)
        if keep:
            _push(t, dr, k, n_kf)
            n_kf += 1
            order.append(f.timestamp_)
            slots |= set(f.measurements_)
            buffer[f.timestamp_] = f
            while len(buffer) > dr.window:
                del buffer[min(buffer)]
    assert picked == dr.selected
    t.close(); h.close()


@pytest.mark.gpu
def test_facade_device_flow_equals_facade(tmp_path):
    """tests/cpp/test_facade_keyframe: the drives mirrored into a track; at every frame kba_track_frame_flow equals the facade's
    flow scheme bit for bit and the selection composed from its verdict equals KeyframeSelector::select"""
    _build()
    for kw in DRIVES:
        path = tmp_path / "drive.txt"
        KeyframeDrive(**kw).write(path)
        r = subprocess.run([EXE, "device", str(path)], capture_output=True, text=True, timeout=1200)
        print(r.stdout)
        assert r.returncode == 0, r.stdout + r.stderr
