"""adjustPoseOnly against a track's store (kba_track_adjust_pose / kba_track_group_adjust_pose): one kernel per frame.

The reference is kba_solve_window on the equivalent window: one free keyframe at the frame's initial pose, the frame's
measurements as its observations, the store's landmark positions and weights, landmarks_fixed = 1.  The one-CTA kernel sums in
another order than the batch kernels, so costs agree to rounding and every count and decision must be equal."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from limo_b200 import synth, geometry as geo
from limo_b200.capi_types import Window

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_track_frame_size_matches_header(tmp_path):
    """sizeof(kba_track_frame) as the C compiler sees it == size of the ctypes mirror"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu\\n",sizeof(kba_track_frame));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    assert int(subprocess.check_output([str(exe)])) == C.sizeof(T.KbaTrackFrame)


def test_adjust_pose_symbols_are_bound():
    from limo_b200 import capi
    assert "kba_track_adjust_pose" in capi.SYMBOLS and "kba_track_group_adjust_pose" in capi.SYMBOLS


class _Frame:
    """The newest keyframe of a seeded synthetic window as a frame: its measurements in ascending landmark id (one run per
    landmark), landmark positions in store slots = landmark ids.  rig: camera 1 (camera 0's mount) sees every fourth landmark
    once more, inside the landmark's run."""

    def __init__(self, seed, n_lm=1200, n_obs=12000, depth=True, rig=False, speed=False, keep=None):
        win, truth = synth.make_window(2, n_kf=12, n_lm=n_lm, n_obs=n_obs, seed=seed, return_truth=True)
        k = win.n_kf - 1
        lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
        sel = np.nonzero(win.obs_kf == k)[0]
        if keep is not None:
            sel = sel[:keep]
        lm, u, v, d = lm_of_obs[sel].astype(np.int32), win.obs_u[sel], win.obs_v[sel], win.obs_d[sel]
        if not depth:
            d = np.full(len(lm), -1.0, np.float32)
        cam = np.zeros(len(lm), np.int32)
        self.n_cam = 1
        if rig:
            self.n_cam = 2
            rows = []
            for a in range(len(lm)):
                rows.append((lm[a], 0, u[a], v[a], d[a]))
                if a % 4 == 0:
                    rows.append((lm[a], 1, u[a] + 0.25, v[a] - 0.25, -1.0))
            lm = np.array([r[0] for r in rows], np.int32); cam = np.array([r[1] for r in rows], np.int32)
            u = np.array([r[2] for r in rows], np.float32); v = np.array([r[3] for r in rows], np.float32)
            d = np.array([r[4] for r in rows], np.float32)
        self.win, self.lm, self.cam, self.u, self.v, self.d = win, lm, cam, u, v, d
        self.cam_intr, self.cam_pose = np.tile(win.cam_intr, (self.n_cam, 1)), np.tile(win.cam_pose, (self.n_cam, 1))
        self.lm_pos = truth["lm_pos"].copy()
        self.lm_weight = np.ones(win.n_lm)
        self.pose7 = win.kf_pose[k].copy()
        self.speed = None
        if speed:
            Tb, Tb2 = geo.pose_to_iso(truth["kf_pose"][k - 1]), geo.pose_to_iso(truth["kf_pose"][k - 2])
            self.speed = dict(weight=0.7, dt=0.1, v_before=(Tb @ geo.iso_inv(Tb2))[:3, 3] / 0.1,
                              T_origin_before=geo.iso_to_pose(geo.iso_inv(Tb)))

    def runs(self):
        starts = np.concatenate([[0], np.nonzero(self.lm[1:] != self.lm[:-1])[0] + 1, [len(self.lm)]]).astype(np.int32)
        return self.lm[starts[:-1]], starts

    def window(self):
        """the equivalent landmarks_fixed window of kba_solve_window"""
        slots, ptr = self.runs()
        sp = {}
        if self.speed:
            sp = dict(speed_kf=0, speed_weight=self.speed["weight"], speed_dt=self.speed["dt"], speed_v_before=self.speed["v_before"],
                      speed_T_origin_before=self.speed["T_origin_before"])
        return Window(kf_pose=self.pose7[None], kf_fixed=[0], cam_intr=self.cam_intr, cam_pose=self.cam_pose,
                      lm_pos=self.lm_pos[slots], lm_weight=self.lm_weight[slots], lm_obs_ptr=ptr,
                      obs_kf=np.zeros(len(self.lm), np.int32), obs_u=self.u, obs_v=self.v, obs_d=self.d,
                      obs_cam=self.cam if self.n_cam > 1 else None, landmarks_fixed=True, **sp)

    def track(self, h):
        from limo_b200 import capi
        n = self.win.n_lm
        t = capi.Track(h, self.cam_intr, self.cam_pose, max_keyframes=3, max_landmarks=n, max_measurements=1, win_keyframes=3,
                       win_landmarks=n, win_observations=max(len(self.lm), 1))
        t.set_landmarks(np.arange(n, dtype=np.int32), pos=self.lm_pos, weight=self.lm_weight)
        return t

    def args(self):
        return dict(pose7=self.pose7, lm_slot=self.lm, u=self.u, v=self.v, d=self.d, cam=self.cam if self.n_cam > 1 else None,
                    speed=self.speed)


def _opt(rounds=-1, **kw):
    from limo_b200 import capi
    o = capi.default_options()
    o.num_trim_rounds = rounds
    o.min_landmarks_for_trimming = 30  # adjustPoseOnly's threshold (cpp:865)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _equal_to_general(a, b, n_runs, label=""):
    """a: track path, b: kba_solve_window on the equivalent window"""
    assert a.c.status == 0 and b.c.status == 0, label
    assert a.c.num_solves == b.c.num_solves, (label, a.c.num_solves, b.c.num_solves)
    for i, (x, y) in enumerate(zip(a.solves, b.solves)):
        key = (label, i)
        assert x.termination == y.termination, key
        assert x.num_iterations == y.num_iterations, (key, x.num_iterations, y.num_iterations)
        assert x.num_successful_steps == y.num_successful_steps, key
        assert x.num_landmarks == y.num_landmarks and x.num_residual_blocks == y.num_residual_blocks, key
        assert x.initial_cost == pytest.approx(y.initial_cost, rel=1e-10), key
        assert x.final_cost == pytest.approx(y.final_cost, rel=1e-10), key
    assert np.array_equal(a.lm_rejected[:n_runs], b.lm_rejected[:n_runs]), label
    assert np.linalg.norm(a.kf_pose[0, 4:] - b.kf_pose[0, 4:]) <= 1e-9, label
    assert np.abs(a.kf_pose[0, :4] - b.kf_pose[0, :4]).max() <= 1e-9, label


def _check_case(h, fr, opt, label):
    t = fr.track(h)
    try:
        a = t.adjust_pose(opt=opt, **fr.args())
    finally:
        t.close()
    win = fr.window()
    b = h.solve_window(win, opt)
    _equal_to_general(a, b, win.n_lm, label)
    return a, b


@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [True, False])
@pytest.mark.parametrize("rounds", [1, 2])
def test_mono_equals_general_path(handle, depth, rounds):
    a, _ = _check_case(handle, _Frame(11 + rounds, depth=depth), _opt(rounds), "mono depth=%s rounds=%d" % (depth, rounds))
    assert a.c.num_solves >= rounds + 1 and a.lm_rejected.sum() > 0


@pytest.mark.gpu
def test_speed_prior_equals_general_path(handle):
    a, _ = _check_case(handle, _Frame(21, speed=True), _opt(1), "speed prior")
    assert a.solves[0].num_residual_blocks > 1


@pytest.mark.gpu
def test_rig_equals_general_path(handle):
    fr = _Frame(31, rig=True)
    assert (np.diff(fr.runs()[1]) == 2).any()  # some landmark seen by both cameras in the frame
    _check_case(handle, fr, _opt(1), "rig")


@pytest.mark.gpu
def test_few_landmarks_no_trimming(handle):
    fr = _Frame(41, keep=25)
    a, _ = _check_case(handle, fr, _opt(-1), "25 landmarks")
    assert a.c.num_solves == 1 and a.lm_rejected[:25].sum() == 0


@pytest.mark.gpu
def test_shrubbery_weights(handle):
    fr = _Frame(51)
    fr.lm_weight[::3] = 0.2  # set through kba_track_set_landmarks by fr.track()
    _check_case(handle, fr, _opt(1), "weights")


@pytest.mark.gpu
def test_landmark_behind_camera_fails_like_general_path(handle):
    fr = _Frame(61)
    T = geo.pose_to_iso(fr.cam_pose[0]) @ geo.pose_to_iso(fr.pose7)
    fr.lm_pos[fr.lm[5]] = geo.iso_inv(T)[:3, 3]  # at the camera centre: |z_cam| < 0.01
    a, _ = _check_case(handle, fr, _opt(1), "behind camera")
    assert a.solves[0].termination == 2 and a.solves[0].initial_cost == -1.0


@pytest.mark.gpu
def test_solver_time_limit(handle):
    _check_case(handle, _Frame(71, speed=True), _opt(1, solver_time_sec=1e-9), "solver_time_sec")


@pytest.mark.gpu
@pytest.mark.parametrize("with_prior", [False, True])
def test_matches_oracle(handle, oracle, with_prior):
    from tests.test_gpu_parity import _compare_solves
    fr = _Frame(81, speed=with_prior)
    opt = _opt(-1, solver_time_sec=20.0)
    t = fr.track(handle)
    try:
        a = t.adjust_pose(opt=opt, **fr.args())
    finally:
        t.close()
    win = fr.window()
    a.lm_pos[:win.n_lm] = win.lm_pos  # constant landmarks: the track path does not return them
    _compare_solves(a, oracle.solve_window(win, opt), win, "oracle prior=%s" % with_prior)


def _same(a, b):
    assert a.c.status == b.c.status and a.c.num_solves == b.c.num_solves
    assert np.array_equal(a.kf_pose, b.kf_pose)
    assert np.array_equal(a.lm_rejected, b.lm_rejected)
    assert bytes(a.c.solves) == bytes(b.c.solves)
    assert a.c.initial_cost == b.c.initial_cost and a.c.final_cost == b.c.final_cost
    assert a.c.num_iteration_records == b.c.num_iteration_records
    for x, y in zip(a.iterations, b.iterations):
        assert bytes(x) == bytes(y)


@pytest.mark.gpu
def test_group_is_bit_identical_to_single_frames(handle):
    from limo_b200 import capi
    frames = [_Frame(91, n_lm=600, n_obs=6000), _Frame(92, rig=True), None, _Frame(93, n_lm=2000, n_obs=20000, speed=True)]
    tracks = []
    for fr in frames:
        tracks.append((fr or frames[0]).track(handle))
    g = capi.TrackGroup(handle, tracks)
    try:
        opt = _opt(-1)
        res = g.adjust_pose([None if fr is None else fr.args() for fr in frames], opt)
        assert res[2].c.status == 0 and res[2].c.num_solves == 0
        for fr, t, r in zip(frames, tracks, res):
            if fr is not None:
                _same(r, t.adjust_pose(opt=opt, **fr.args()))
    finally:
        g.close()
        for t in tracks:
            t.close()


@pytest.mark.gpu
def test_store_untouched_by_adjust_pose(handle):
    from tests.test_track_group import _Drive
    drv = _Drive(7, W=8, n_lm=1500, n_obs=18000, steps=4)
    a, b = drv.make_track(handle), drv.make_track(handle)
    try:
        for step in range(1, 4):
            for t in (a, b):
                drv.advance(t, step)
            k = drv.W - 1 + step
            lm, u, v, d, cam = drv.measurements(k)
            for _ in range(2):
                a.adjust_pose(drv.win.kf_pose[k], lm, u, v, d, opt=_opt(-1))
            req = drv.request(step)
            ra = a.solve(req["kf_slots"], req["kf_fixed"], req["lm_slots"],
                         **{k2: v2 for k2, v2 in req.items() if k2 not in ("kf_slots", "kf_fixed", "lm_slots")})
            rb = b.solve(req["kf_slots"], req["kf_fixed"], req["lm_slots"],
                         **{k2: v2 for k2, v2 in req.items() if k2 not in ("kf_slots", "kf_fixed", "lm_slots")})
            drv.record(rb)
            assert np.array_equal(ra.kf_pose, rb.kf_pose) and np.array_equal(ra.lm_pos, rb.lm_pos)
            assert bytes(ra.c.solves) == bytes(rb.c.solves)
    finally:
        a.close(); b.close()


@pytest.mark.gpu
def test_validation_errors_launch_nothing(handle):
    from limo_b200 import capi
    fr = _Frame(101, n_lm=400, n_obs=4000)
    t = fr.track(handle)
    t2 = _Frame(102, n_lm=400, n_obs=4000).track(handle)
    g = capi.TrackGroup(handle, [t2, t])
    try:
        ref = t.adjust_pose(opt=_opt(1), **fr.args())
        n = len(fr.lm)
        bad = []
        slot = fr.lm.copy(); slot[3] = 10 ** 6
        bad.append((dict(lm_slot=slot), 1))                       # slot out of range
        cam = np.zeros(n, np.int32); cam[2] = 1
        bad.append((dict(cam=cam), 1))                             # camera out of range (mono track)
        slot = fr.lm.copy(); slot[-1] = slot[0]
        bad.append((dict(lm_slot=slot), 1))                        # slot reappears after its run
        bad.append((dict(speed=dict(weight=1.0, dt=0.0, v_before=(0, 0, 0), T_origin_before=(1, 0, 0, 0, 0, 0, 0))), 1))
        bad.append((dict(lm_slot=np.sort(np.tile(fr.lm, 2)), u=np.tile(fr.u, 2), v=np.tile(fr.v, 2), d=np.tile(fr.d, 2)), 4))
        for change, code in bad:
            args = fr.args(); args.update(change)
            before = handle.counters().launches_total
            with pytest.raises(capi.KbaError, match="error %d" % code):
                t.adjust_pose(opt=_opt(1), **args)
            with pytest.raises(capi.KbaError, match="error %d.*track 1" % code):
                g.adjust_pose([None, args], _opt(1))
            assert handle.counters().launches_total == before
        with pytest.raises(capi.KbaError, match="error 1"):
            t.adjust_pose(opt=_opt(1, precision=1), **fr.args())
        _same(t.adjust_pose(opt=_opt(1), **fr.args()), ref)  # the store is as it was
    finally:
        g.close(); t.close(); t2.close()


@pytest.mark.gpu
def test_facade_adjust_pose_on_the_store():
    """tests/cpp/test_facade_motion.cpp: the facade's adjustPoseOnly() on the device-resident store against a rebuild-path twin
    (poses to 1e-9 m, equal iteration counts, a smaller upload), and one solve() with the persistent window switched off and on
    again keeping every later solve() bit-identical to the twin"""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])
    out = subprocess.run([os.path.join(ROOT, "tests", "cpp", "test_facade_motion")], capture_output=True, text=True)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
