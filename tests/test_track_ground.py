"""Ground points attached on the device (kba_track_solve with candidate ground landmarks) against host-built lists.

A caller with ground-plane landmarks may send only which selected landmarks are ground points; the track attaches each to its
nearest keyframe exactly as addGroundPlaneResiduals does (reference bundle_adjuster_keyframes.cpp:517-562), from the poses,
planes and positions in its store.  Every GPU test replays a seeded ground drive into two tracks: one attaches on the device, its
twin gets host lists computed from the twin's store as mirrored on the host.  Both must agree bit for bit at every step."""
import numpy as np
import pytest

from limo_b200 import synth
from tests.test_track import _scale, _window_lists
from tests.test_track_group import PLANE, _Drive, _equal

DBL_MAX = np.finfo(np.float64).max


def _attach(poses, planes, pos):
    """the facade's host computation of the attachment (mini_eigen.hpp: convert() of the 7-vector with Eigen's un-normalised
    toRotationMatrix, R * p + t, sqrt of the squared norm), one elementwise operation at a time in its order.
    Returns (kept, keyframe, weight) per candidate."""
    qw, qx, qy, qz = (poses[:, i] for i in range(4))
    tx, ty, tz = 2.0 * qx, 2.0 * qy, 2.0 * qz
    twx, twy, twz = tx * qw, ty * qw, tz * qw
    txx, txy, txz, tyy, tyz, tzz = tx * qx, ty * qx, tz * qx, ty * qy, tz * qy, tz * qz
    Rq = [[1.0 - (tyy + tzz), txy - twz, txz + twy],
          [txy + twz, 1.0 - (txx + tzz), tyz - twx],
          [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]
    eye = np.eye(3)
    R = [[((0.0 + eye[i, 0] * Rq[0][j]) + eye[i, 1] * Rq[1][j]) + eye[i, 2] * Rq[2][j] for j in range(3)] for i in range(3)]
    t = [0.0 + ((eye[i, 0] * poses[:, 4] + eye[i, 1] * poses[:, 5]) + eye[i, 2] * poses[:, 6]) for i in range(3)]
    px, py, pz = (pos[:, i][:, None] for i in range(3))     # candidates x keyframes
    x, y, z = (((R[i][0] * px + R[i][1] * py) + R[i][2] * pz) + t[i] for i in range(3))
    dist = np.sqrt((x * x + y * y) + z * z)
    md, best = np.full(len(pos), DBL_MAX), np.zeros(len(pos), dtype=np.int32)
    for k in range(len(poses)):              # window order, first strict minimum
        if planes[k, 3] < -10.0:
            continue
        upd = dist[:, k] < md
        md, best = np.where(upd, dist[:, k], md), np.where(upd, k, best)
    return md < 25.0, best, 10.0 * (1.0 - md / 25.0)


class _GroundDrive(_Drive):
    """a config-3 drive (ground plane 0.31 m below the vehicle) without lidar depth, so that the number of attached ground points
    alone decides the scale rule; the host mirrors the twin's store: poses, planes and landmark positions"""

    def __init__(self, seed, W, n_lm, n_obs, steps):
        self.W, self.rig, self.ground, self.steps = W, False, True, steps
        self.n_kf = W + steps
        self.win = win = synth.make_window(3, seed=seed, n_kf=self.n_kf, n_lm=n_lm, n_obs=n_obs, depth_frac=0.0)
        lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
        self.per_kf = []
        for k in range(self.n_kf):
            sel = np.nonzero(win.obs_kf == k)[0]
            self.per_kf.append((lm_of_obs[sel].astype(np.int32), win.obs_u[sel], win.obs_v[sel], win.obs_d[sel]))
        self.poses, self.planes, self.lm = win.kf_pose.copy(), np.tile(PLANE, (self.n_kf, 1)), win.lm_pos.copy()
        self.cam_intr, self.cam_pose = win.cam_intr, win.cam_pose

    def make_track(self, h, win_ground=64, win_keyframes=None):
        from limo_b200 import capi
        W, win = self.W, self.win
        t = capi.Track(h, self.cam_intr, self.cam_pose, max_keyframes=W + 1, max_landmarks=win.n_lm,
                       max_measurements=sum(self.counts()), win_keyframes=win_keyframes or W, win_landmarks=win.n_lm,
                       win_observations=self.window_obs()[0], win_ground=win_ground)
        t.set_landmarks(np.arange(win.n_lm, dtype=np.int32), pos=win.lm_pos, weight=win.lm_weight)
        for k in range(W):
            self._push(t, k)
        return t

    def base(self, step, scale_rule=True):
        """the plane-free request of a step: active keyframes, selected landmarks, scale regulariser"""
        W = self.W
        first, last = step, step + W - 1
        lm_sel, ptr, okf, ou, ov, od = _window_lists(self.per_kf, first, last)
        fixed = np.zeros(W, dtype=np.uint8); fixed[0] = 1
        req = dict(kf_slots=[k % (W + 1) for k in range(first, last + 1)], kf_fixed=fixed, lm_slots=lm_sel,
                   **_scale(self.poses[first:last + 1], int((od > 0).sum())))
        if scale_rule:
            req["scale_weight"] = -1.0
        self.cur = (first, last, lm_sel, ptr, okf)
        self.obs = (ou, ov, od)
        return req

    def attach(self):
        """host attachment of every selected landmark at the mirrored state of the current window"""
        first, last, lm_sel = self.cur[0], self.cur[1], self.cur[2]
        return _attach(self.poses[first:last + 1], self.planes[first:last + 1], self.lm[lm_sel])

    def record(self, res):
        first, last, lm_sel = self.cur[0], self.cur[1], self.cur[2]
        self.poses[first:last + 1] = res.kf_pose
        self.planes[first:last + 1] = res.kf_plane
        self.lm[lm_sel] = res.lm_pos[:len(lm_sel)]


def _requests(dr, step, target, n_far=3):
    """device request (candidates) and host request (lists) of one step: `target` landmarks that attach and n_far that do not"""
    base = dr.base(step)
    keep, best, wgt = dr.attach()
    near, far = np.nonzero(keep)[0], np.nonzero(~keep)[0]
    assert len(near) >= target and len(far) >= n_far
    cand = np.sort(np.concatenate([near[:target], far[:n_far]])).astype(np.int32)
    k = keep[cand]
    dev = dict(base, gp_lm=cand, plane_reg_weight=-1.0)
    host = dict(base, plane_reg_weight=-1.0)
    if k.any():
        host.update(gp_lm=cand[k], gp_kf=best[cand][k].astype(np.int32), gp_weight=wgt[cand][k])
    return dev, host, int(k.sum())


def _equal_blocks(a, b, what):
    assert [s.num_residual_blocks for s in a.solves] == [s.num_residual_blocks for s in b.solves], what
    assert [s.num_landmarks for s in a.solves] == [s.num_landmarks for s in b.solves], what


@pytest.mark.gpu
def test_device_attachment_equals_host_lists():
    """attached counts of 0, 1-10, 11-29 and >= 30 (every branch of the scale rule), candidates beyond 25 m of every keyframe, a
    keyframe whose plane distance is below -10: poses, planes, landmarks, rejections, iterations, residual blocks and the final
    cost bit-equal at every step; a window with nothing attached gives the stored planes back and equals a plane-free solve; every
    bad request is refused before it changes a store; the candidates travel in fewer bytes than the lists"""
    from limo_b200 import capi
    h = capi.Handle(0)
    dr = _GroundDrive(seed=301, W=12, n_lm=900, n_obs=8000, steps=8)
    ta, tb = dr.make_track(h), dr.make_track(h)
    targets = [5, 20, 40, 0, 8, 15, 35, 2]
    counts, up_a, up_b = [], 0, 0
    for step in range(dr.steps):
        if step:
            dr.advance(ta, step); dr.advance(tb, step)
        if step == 4:  # the window's fourth keyframe leaves the attachment: plane distance below -10, in both stores
            first = step
            slot = [(first + 3) % (dr.W + 1)]
            dr.planes[first + 3, 3] = -11.0
            for t in (ta, tb):
                t.set_keyframe_poses(slot, dr.poses[first + 3:first + 4], dr.planes[first + 3:first + 4])
        dev, host, n_att = _requests(dr, step, targets[step])
        counts.append(n_att)
        n_lm = len(dev["lm_slots"])
        if step == 2:
            cand = dev["gp_lm"]
            bad = [dict(dev, gp_lm=cand[::-1].copy()), dict(dev, gp_lm=np.concatenate([cand[:1], cand])),
                   dict(dev, gp_lm=np.concatenate([cand, [n_lm]]).astype(np.int32)),
                   dict(dev, gp_kf=np.zeros(len(cand), np.int32)), dict(dev, gp_weight=np.ones(len(cand)))]
            for b in bad:
                with pytest.raises(capi.KbaError, match="error 1"):
                    ta.solve(**b)
            with pytest.raises(capi.KbaError, match="error 4"):
                ta.solve(**dict(dev, gp_lm=np.arange(65, dtype=np.int32)))
        ra = ta.solve(**dev)
        up_a += ta.transfer_bytes()[0]
        rb = tb.solve(**host)
        up_b += tb.transfer_bytes()[0]
        what = "step %d (%d attached)" % (step, n_att)
        _equal(ra, rb, n_lm, what)
        _equal_blocks(ra, rb, what)
        if n_att == 0:  # nothing attached: the planes come back as stored
            first, last = dr.cur[0], dr.cur[1]
            assert np.array_equal(ra.kf_plane, dr.planes[first:last + 1]), what
        dr.record(rb)
    assert 0 in counts and any(1 <= c <= 10 for c in counts) and any(11 <= c <= 29 for c in counts) and any(c >= 30 for c in counts)
    assert up_a < up_b, (up_a, up_b)
    print("attached per step %s; upload %d B with candidates, %d B with host lists" % (counts, up_a, up_b))
    ta.close(); tb.close(); h.close()


@pytest.mark.gpu
def test_thirty_keyframes_on_a_ground_track():
    """a ground-capacity track takes 30-keyframe windows: without candidates such a window equals kba_solve_window bit for bit;
    19 keyframes with candidates are refused (more than 184 reduced rows with plane blocks) and change nothing"""
    from limo_b200 import capi
    from limo_b200.capi_types import Window
    h = capi.Handle(0)
    dr = _GroundDrive(seed=302, W=30, n_lm=1500, n_obs=14000, steps=2)
    ta = dr.make_track(h, win_ground=64)
    for step in range(dr.steps):
        if step:
            dr.advance(ta, step)
        req = dr.base(step, scale_rule=False)
        if step == 1:
            cand = np.arange(5, dtype=np.int32)
            bad = dict(req, kf_slots=req["kf_slots"][:19], kf_fixed=req["kf_fixed"][:19], gp_lm=cand, plane_reg_weight=-1.0)
            with pytest.raises(capi.KbaError, match="error 4.*18 keyframes"):
                ta.solve(**bad)
            with pytest.raises(capi.KbaError, match="error 4.*18 keyframes"):
                ta.solve(**dict(req, plane_reg_weight=10.0))
        ra = ta.solve(**req)
        first, last, lm_sel, ptr, okf = dr.cur
        ou, ov, od = dr.obs
        sc = {k: req[k] for k in ("scale_kf0", "scale_kf1", "scale_weight", "scale_value")}
        win = Window(dr.poses[first:last + 1], req["kf_fixed"], dr.cam_intr, dr.cam_pose, dr.lm[lm_sel], dr.win.lm_weight[lm_sel],
                     ptr, okf, ou, ov, od, **sc)
        rw = h.solve_window(win)
        what = "step %d" % step
        assert ra.c.status == 0 and rw.c.status == 0, what
        assert [s.num_iterations for s in ra.solves] == [s.num_iterations for s in rw.solves], what
        assert np.array_equal(ra.kf_pose, rw.kf_pose), what
        n_lm = len(lm_sel)
        assert np.array_equal(ra.lm_pos[:n_lm], rw.lm_pos[:n_lm]), what
        assert np.array_equal(ra.lm_rejected[:n_lm], rw.lm_rejected[:n_lm]), what
        assert ra.c.final_cost == rw.c.final_cost, what
        assert np.array_equal(ra.kf_plane, dr.planes[first:last + 1]), what
        dr.record(ra)
    ta.close(); h.close()


@pytest.mark.gpu
def test_mixed_group(monkeypatch):
    """one group of a device-attached track, a host-list track and a plane-free mono track equals the single solves; a bad
    candidate list names its track and changes nothing"""
    from limo_b200 import capi
    monkeypatch.setenv("KBA_P_SPLIT", "6")
    h = capi.Handle(0)
    dr = _GroundDrive(seed=303, W=10, n_lm=800, n_obs=7000, steps=6)
    mono = _Drive(seed=304, W=8, n_lm=700, n_obs=6000, steps=6)
    ga, gb, gc = dr.make_track(h), dr.make_track(h), mono.make_track(h)
    tw, tc = dr.make_track(h), mono.make_track(h)
    grp = capi.TrackGroup(h, [ga, gb, gc])
    for step in range(dr.steps):
        if step:
            for t in (ga, gb, tw):
                dr.advance(t, step)
            mono.advance(gc, step); mono.advance(tc, step)
        dev, host, n_att = _requests(dr, step, (4, 25, 33)[step % 3])
        rm = mono.request(step)
        if step == 1:
            with pytest.raises(capi.KbaError, match="error 1.*track 0"):
                grp.solve([dict(dev, gp_lm=dev["gp_lm"][::-1].copy()), host, rm])
        res = grp.solve([dev, host, rm])
        rt, rc = tw.solve(**host), tc.solve(**rm)
        n_lm = len(dev["lm_slots"])
        for r, what in ((res[0], "device"), (res[1], "host lists")):
            what = "step %d %s (%d attached)" % (step, what, n_att)
            _equal(r, rt, n_lm, what)
            _equal_blocks(r, rt, what)
        _equal(res[2], rc, len(rm["lm_slots"]), "step %d mono" % step)
        dr.record(rt); mono.record(rc)
    grp.close()
    for t in (ga, gb, gc, tw, tc):
        t.close()
    h.close()
