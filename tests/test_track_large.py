"""Persistent windows beyond 184 reduced rows: a track created with win_rows > 184 also owns a large-window solver.

A ground-plane window of 19 or more keyframes (10 rows per keyframe + 1 > 184) or a plane-free window of more than 30 keyframes
does not fit the fused path.  Such a track solves it on the large-window path (k_schur_syrk, row-major or split factorisation),
packed on the device, and picks per solve the solver kba_batch_create would pick for the window, with the Schur split and the
factorisation of the solved window.  Every GPU test compares with kba_solve_window on the host-built window or with single
solves, bit for bit wherever both take the same path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from limo_b200.capi_types import Window
from tests.test_track import _scale, _window_lists
from tests.test_track_ground import _GroundDrive, _equal_blocks
from tests.test_track_group import ROOT, _Drive, _equal


def test_track_caps_size_matches_header(tmp_path):
    """sizeof(kba_track_caps) as the C compiler sees it == size of the ctypes mirror"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu\\n",sizeof(kba_track_caps));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    assert int(subprocess.check_output([str(exe)])) == C.sizeof(T.KbaTrackCaps)


def _track(dr, h, win_rows, win_keyframes=None, win_ground=None):
    """dr.make_track with a reduced-system capacity"""
    from limo_b200 import capi
    W, win = dr.W, dr.win
    if win_ground is None:
        win_ground = 64 if dr.ground else 0
    t = capi.Track(h, dr.cam_intr, dr.cam_pose, max_keyframes=W + 1, max_landmarks=win.n_lm, max_measurements=sum(dr.counts()),
                   win_keyframes=win_keyframes or W, win_landmarks=win.n_lm, win_observations=dr.window_obs()[0],
                   win_ground=win_ground, win_rows=win_rows)
    t.set_landmarks(np.arange(win.n_lm, dtype=np.int32), pos=win.lm_pos, weight=win.lm_weight)
    for k in range(W):
        dr._push(t, k)
    return t


def _sub(dr, first, n):
    """the request of keyframes first .. first + n - 1 of a ground drive (explicit scale regulariser), as _GroundDrive.base"""
    last = first + n - 1
    lm_sel, ptr, okf, ou, ov, od = _window_lists(dr.per_kf, first, last)
    fixed = np.zeros(n, dtype=np.uint8); fixed[0] = 1
    dr.cur = (first, last, lm_sel, ptr, okf)
    dr.obs = (ou, ov, od)
    return dict(kf_slots=[k % (dr.W + 1) for k in range(first, last + 1)], kf_fixed=fixed, lm_slots=lm_sel,
                **_scale(dr.poses[first:last + 1], int((od > 0).sum())))


def _host_window(dr, req, gp=None):
    """kba_solve_window's window of the current request at the mirrored state; gp = (gp_lm, gp_kf, gp_weight) or None"""
    first, last, lm_sel, ptr, okf = dr.cur
    ou, ov, od = dr.obs
    sc = {k: req[k] for k in ("scale_kf0", "scale_kf1", "scale_weight", "scale_value")}
    extra = {}
    if gp is not None and len(gp[0]):
        extra = dict(gp_lm=gp[0], gp_kf=gp[1], gp_weight=gp[2], plane_reg_weight=10.0)
    return Window(dr.poses[first:last + 1], req["kf_fixed"], dr.cam_intr, dr.cam_pose, dr.lm[lm_sel], dr.win.lm_weight[lm_sel],
                  ptr, okf, ou, ov, od, kf_plane=dr.planes[first:last + 1], **sc, **extra)


def _candidates(dr, target, n_far=3):
    """device candidates (target that attach, up to n_far that do not) and the host lists they give at the mirrored state"""
    keep, best, wgt = dr.attach()
    near, far = np.nonzero(keep)[0], np.nonzero(~keep)[0]
    cand = np.sort(np.concatenate([near[:target], far[:n_far]])).astype(np.int32)
    k = keep[cand]
    return cand, (cand[k], best[cand][k].astype(np.int32), wgt[cand][k]), int(k.sum())


def _device_request(dr, step, target):
    """step's window of a ground drive with candidates (the reference's scale and plane rules on the device)"""
    base = dr.base(step)
    cand, _, n_att = _candidates(dr, target)
    assert n_att > 0
    return dict(base, gp_lm=cand, plane_reg_weight=-1.0)


def _close(a, b, what):
    """the north-star tolerances: translations to 1e-6 m, the final cost to 1e-8 relative"""
    assert a.c.status == 0 and b.c.status == 0, what
    assert np.max(np.abs(a.kf_pose[:, 4:] - b.kf_pose[:, 4:])) <= 1e-6, what
    assert abs(a.c.final_cost - b.c.final_cost) <= 1e-8 * abs(b.c.final_cost), what


@pytest.mark.gpu
def test_create_time_rules():
    """win_rows = 0 keeps the fused limits; win_rows from 6 * win_keyframes + 1 to 640 is accepted, anything else refused; a
    request beyond win_rows is refused and names it"""
    from limo_b200 import capi
    from tests.test_track import _drive
    win, per_kf = _drive()
    h = capi.Handle(0)
    mk = lambda **kw: capi.Track(h, win.cam_intr, win.cam_pose, 64, 100, 1000, win_landmarks=100, win_observations=1000, **kw)
    with pytest.raises(capi.KbaError, match="error 4"):
        mk(win_keyframes=40)
    mk(win_keyframes=40, win_rows=241).close()
    mk(win_keyframes=20, win_rows=640).close()
    for rows in (240, 1, -1):
        with pytest.raises(capi.KbaError, match="error 1"):
            mk(win_keyframes=40, win_rows=rows)
    with pytest.raises(capi.KbaError, match="error 4"):
        mk(win_keyframes=40, win_rows=641)
    # a win_rows = 0 ground track still refuses 19 keyframes with candidates
    dr = _GroundDrive(seed=311, W=30, n_lm=1500, n_obs=14000, steps=1)
    t0 = _track(dr, h, 0)
    req = _sub(dr, 0, 19)
    with pytest.raises(capi.KbaError, match="error 4.*18 keyframes"):
        t0.solve(**dict(req, gp_lm=np.arange(5, dtype=np.int32), plane_reg_weight=-1.0))
    t0.close()
    # win_rows = 251: 25 keyframes with plane blocks fit, 26 do not
    t1 = _track(dr, h, 251)
    with pytest.raises(capi.KbaError, match="error 4.*261 reduced rows.*win_rows = 251"):
        t1.solve(**dict(_sub(dr, 0, 26), plane_reg_weight=10.0))
    assert t1.solve(**dict(_sub(dr, 0, 25), plane_reg_weight=10.0)).c.status == 0
    t1.close(); h.close()


@pytest.mark.gpu
def test_ground_track_across_the_fused_boundary():
    """a win_rows = 301 ground track solves windows of 12, 18 (fused) and 19, 20, 24, 30 keyframes (large-window path) with
    candidates that attach, and a plane-free 30-keyframe window (fused): each equals kba_solve_window on the host-built window
    bit for bit; refused requests change no store"""
    from limo_b200 import capi
    h = capi.Handle(0)
    dr = _GroundDrive(seed=312, W=30, n_lm=1500, n_obs=14000, steps=1)
    t = _track(dr, h, 301)
    plan = [(12, 6), (18, 20), (19, 12), (20, 30), (24, 4), (30, 25), (30, None), (20, 15)]
    for i, (n, target) in enumerate(plan):
        req = _sub(dr, 30 - n, n)
        what = "%d keyframes, target %s" % (n, target)
        if target is None:
            ra, gp, n_att = t.solve(**req), None, 0
        else:
            cand, gp, n_att = _candidates(dr, target)
            assert n_att > 0, what
            dev = dict(req, gp_lm=cand, plane_reg_weight=-1.0)
            if i == 3:  # refused before anything runs: the solve below still equals the host-built window
                with pytest.raises(capi.KbaError, match="error 1"):
                    t.solve(**dict(dev, gp_lm=cand[::-1].copy()))
                with pytest.raises(capi.KbaError, match="error 4"):
                    t.solve(**dict(dev, gp_lm=np.arange(65, dtype=np.int32)))
            ra = t.solve(**dev)
        rw = h.solve_window(_host_window(dr, req, gp))
        n_lm = len(req["lm_slots"])
        _equal(ra, rw, n_lm, what)
        _equal_blocks(ra, rw, what)
        print("%s: %d attached, %d iterations" % (what, n_att, sum(s.num_iterations for s in ra.solves)))
        dr.record(ra)
    t.close(); h.close()


@pytest.mark.gpu
def test_forty_plane_free_keyframes():
    """a 40-keyframe config-2 track (win_rows = 241) through several pushes and solves equals kba_solve_window bit for bit"""
    from limo_b200 import capi
    h = capi.Handle(0)
    dr = _Drive(seed=313, W=40, n_lm=2500, n_obs=30000, steps=4)
    t = _track(dr, h, 241)
    lm = dr.win.lm_pos.copy()
    for step in range(dr.steps):
        if step:
            dr.advance(t, step)
        req = dr.request(step)
        ra = t.solve(**req)
        first, last, lm_sel, ptr, okf = dr.cur
        _, _, _, ou, ov, od = _window_lists(dr.per_kf, first, last)
        sc = {k: req[k] for k in ("scale_kf0", "scale_kf1", "scale_weight", "scale_value")}
        rw = h.solve_window(Window(dr.poses[first:last + 1], req["kf_fixed"], dr.cam_intr, dr.cam_pose, lm[lm_sel],
                                   dr.win.lm_weight[lm_sel], ptr, okf, ou, ov, od, **sc))
        n_lm = len(lm_sel)
        assert ra.c.status == 0 and rw.c.status == 0
        assert [s.num_iterations for s in ra.solves] == [s.num_iterations for s in rw.solves], step
        assert np.array_equal(ra.kf_pose, rw.kf_pose), step
        assert np.array_equal(ra.lm_pos[:n_lm], rw.lm_pos[:n_lm]), step
        assert np.array_equal(ra.lm_rejected[:n_lm], rw.lm_rejected[:n_lm]), step
        assert ra.c.final_cost == rw.c.final_cost, step
        dr.record(ra)
        lm[lm_sel] = ra.lm_pos[:n_lm]
    t.close(); h.close()


@pytest.mark.gpu
def test_candidates_with_nothing_attached():
    """the documented exception: 20 keyframes with candidates of which none attaches take the large-window path, chosen before
    the attachment; kba_solve_window sees a plane-free window (fused path).  Equal to the north-star tolerances, also to a
    plane-free solve of a twin track, which equals kba_solve_window bit for bit; the planes come back as stored"""
    from limo_b200 import capi
    h = capi.Handle(0)
    dr = _GroundDrive(seed=314, W=30, n_lm=1500, n_obs=14000, steps=1)
    ta, tb = _track(dr, h, 301), _track(dr, h, 301)
    req = _sub(dr, 10, 20)
    keep = dr.attach()[0]
    far = np.nonzero(~keep)[0].astype(np.int32)
    assert len(far) >= 1
    ra = ta.solve(**dict(req, gp_lm=far[:10], plane_reg_weight=-1.0))
    rb = tb.solve(**req)
    rw = h.solve_window(_host_window(dr, req))
    _equal(rb, rw, len(req["lm_slots"]), "plane-free twin")
    _close(ra, rw, "candidates, nothing attached")
    _close(ra, rb, "candidates, nothing attached, against the twin")
    _equal_blocks(ra, rw, "residual blocks")
    assert np.array_equal(ra.kf_plane, dr.planes[10:30])
    ta.close(); tb.close(); h.close()


@pytest.mark.gpu
def test_groups_on_the_large_path(monkeypatch):
    """three 20-keyframe ground tracks and an idle one equal their single solves bit for bit; a group of a fused-sized ground
    track, a 20-keyframe ground track and a mono track takes the large-window path for all three: the 20-keyframe window is
    bit-equal to its single solve, the others agree to the north-star tolerances; a bad request names its track and changes
    no store"""
    from limo_b200 import capi
    monkeypatch.setenv("KBA_P_SPLIT", "6")
    h = capi.Handle(0)
    drives = [_GroundDrive(seed=315 + i, W=20, n_lm=1100, n_obs=10000, steps=3) for i in range(3)]
    idle = _Drive(seed=318, W=8, n_lm=600, n_obs=5000, steps=3)
    ga, tw = [_track(d, h, 301) for d in drives], [_track(d, h, 301) for d in drives]
    gi = idle.make_track(h)
    grp = capi.TrackGroup(h, ga + [gi])
    for step in range(3):
        reqs = []
        for i, d in enumerate(drives):
            if step:
                d.advance(ga[i], step); d.advance(tw[i], step)
            reqs.append(_device_request(d, step, (6, 18, 31)[(step + i) % 3]))
        if step == 1:
            with pytest.raises(capi.KbaError, match="error 1.*track 2"):
                grp.solve(reqs[:2] + [dict(reqs[2], gp_lm=reqs[2]["gp_lm"][::-1].copy()), None])
        res = grp.solve(reqs + [None])
        assert res[3].c.num_solves == 0
        for i, d in enumerate(drives):
            rt = tw[i].solve(**reqs[i])
            what = "step %d track %d" % (step, i)
            _equal(res[i], rt, len(reqs[i]["lm_slots"]), what)
            _equal_blocks(res[i], rt, what)
            d.record(rt)
    grp.close()
    for t in ga + tw + [gi]:
        t.close()
    # mixed: a 12-keyframe ground track (fused alone), a 20-keyframe ground track (large alone), a mono track
    small = _GroundDrive(seed=319, W=12, n_lm=900, n_obs=8000, steps=3)
    big = _GroundDrive(seed=320, W=20, n_lm=1100, n_obs=10000, steps=3)
    mono = _Drive(seed=321, W=8, n_lm=700, n_obs=6000, steps=3)
    gm = [small.make_track(h), _track(big, h, 301), mono.make_track(h)]
    tm = [small.make_track(h), _track(big, h, 301), mono.make_track(h)]
    grp = capi.TrackGroup(h, gm)
    # the fused-sized windows run a different solver in the group than alone: converged further than by default, so that the two
    # end points do not differ by where each path's function tolerance stopped it (2.6e-6 m in one step at the defaults)
    opt = capi.default_options()
    opt.function_tolerance, opt.parameter_tolerance = 1e-12, 1e-10
    for step in range(3):
        if step:
            for d, a, b in ((small, gm[0], tm[0]), (big, gm[1], tm[1]), (mono, gm[2], tm[2])):
                d.advance(a, step); d.advance(b, step)
        reqs = [_device_request(small, step, 10), _device_request(big, step, 20), mono.request(step)]
        res = grp.solve(reqs, opt)
        single = [tm[i].solve(opt=opt, **reqs[i]) for i in range(3)]
        _equal(res[1], single[1], len(reqs[1]["lm_slots"]), "step %d large window" % step)
        _equal_blocks(res[1], single[1], "step %d large window" % step)
        _close(res[0], single[0], "step %d fused-sized ground window" % step)
        _close(res[2], single[2], "step %d mono window" % step)
        small.record(single[0]); big.record(single[1]); mono.record(single[2])
        # the group's members continue from the single solves' states, so that both stay comparable
        for d, t, r in ((small, gm[0], single[0]), (big, gm[1], single[1])):
            first, last, lm_sel = d.cur[0], d.cur[1], d.cur[2]
            t.set_keyframe_poses([k % (d.W + 1) for k in range(first, last + 1)], r.kf_pose, r.kf_plane)
            t.set_landmarks(lm_sel, pos=r.lm_pos[:len(lm_sel)])
        first, last, lm_sel = mono.cur[0], mono.cur[1], mono.cur[2]
        gm[2].set_keyframe_poses([k % (mono.W + 1) for k in range(first, last + 1)], single[2].kf_pose)
        gm[2].set_landmarks(lm_sel, pos=single[2].lm_pos[:len(lm_sel)])
    grp.close()
    for t in gm + tm:
        t.close()
    h.close()


@pytest.mark.gpu
def test_facade_twenty_keyframe_ground_window():
    """limo's default 20-keyframe window with ground points through the facade: every solve() on the device-resident window,
    bit-identical to the rebuild path at every step (tests/cpp/test_facade_large.cpp)"""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])
    out = subprocess.run([os.path.join(ROOT, "tests", "cpp", "test_facade_large")], capture_output=True, text=True)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
