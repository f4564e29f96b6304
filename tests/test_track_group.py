"""Track groups (kba_track_group_*): one window of each of several persistent tracks solved as one batch.

Every GPU test replays seeded synthetic drives into two tracks per sequence: the group member and a twin that kba_track_solve
solves alone.  A step is one push per track (the keyframe that left the window is dropped before its slot is reused) and one
solve of the sliding window.  The group's results and the stores they leave behind must be those of the single solves."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from limo_b200 import synth
from tests.test_track import _scale, _window_lists

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANE = np.array([0.0, 0.0, 1.0, 0.31])


def test_track_request_size_matches_header(tmp_path):
    """sizeof(kba_track_request) as the C compiler sees it == size of the ctypes mirror"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu\\n",sizeof(kba_track_request));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    assert int(subprocess.check_output([str(exe)])) == C.sizeof(T.KbaTrackRequest)


class _Drive:
    """One synthetic sequence: keyframe k lives in slot k % (W + 1); step s solves keyframes s .. s + W - 1.  `poses` mirrors
    the twin's store on the host (scale-regulariser values are computed from it, as a caller would)."""

    def __init__(self, seed, W, n_lm, n_obs, config=2, rig=False, ground=False, steps=15):
        self.W, self.rig, self.ground, self.steps = W, rig, ground, steps
        self.n_kf = W + steps
        self.win = win = synth.make_window(config, seed=seed, n_kf=self.n_kf, n_lm=n_lm, n_obs=n_obs)
        lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
        self.per_kf = []
        for k in range(self.n_kf):
            sel = np.nonzero(win.obs_kf == k)[0]          # landmark-major order = ascending landmark id inside a keyframe
            self.per_kf.append((lm_of_obs[sel].astype(np.int32), win.obs_u[sel], win.obs_v[sel], win.obs_d[sel]))
        self.poses = win.kf_pose.copy()
        n_cam = 2 if rig else 1
        self.cam_intr, self.cam_pose = np.tile(win.cam_intr, (n_cam, 1)), np.tile(win.cam_pose, (n_cam, 1))
        if ground:
            self.gp = {int(j): (int(k), float(w)) for j, k, w in zip(win.gp_lm, win.gp_kf, win.gp_weight)}
            assert self.gp

    def measurements(self, k):
        lm, u, v, d = self.per_kf[k]
        cam = np.zeros(len(lm), dtype=np.int32)
        if self.rig:  # camera 1, on camera 0's mount, sees every fourth landmark of the keyframe once more
            e = np.arange(0, len(lm), 4)
            lm, u, v = np.concatenate([lm, lm[e]]), np.concatenate([u, u[e] + 0.25]), np.concatenate([v, v[e] - 0.25])
            d, cam = np.concatenate([d, np.full(len(e), -1.0, np.float32)]), np.concatenate([cam, np.ones(len(e), np.int32)])
        return lm, u, v, d, cam

    def counts(self):
        return [len(self.measurements(k)[0]) for k in range(self.n_kf)]

    def window_obs(self):
        """observations of the fullest window the drive solves, and the step that solves it"""
        c = self.counts()
        sums = [sum(c[s:s + self.W]) for s in range(self.steps)]
        return max(sums), int(np.argmax(sums))

    def make_track(self, h, max_measurements=None, win_keyframes=None, win_observations=None):
        from limo_b200 import capi
        W, win = self.W, self.win
        t = capi.Track(h, self.cam_intr, self.cam_pose, max_keyframes=W + 1, max_landmarks=win.n_lm,
                       max_measurements=max_measurements or sum(self.counts()), win_keyframes=win_keyframes or W,
                       win_landmarks=win.n_lm, win_observations=win_observations or self.window_obs()[0],
                       win_ground=len(self.gp) if self.ground else 0)
        t.set_landmarks(np.arange(win.n_lm, dtype=np.int32), pos=win.lm_pos, weight=win.lm_weight)
        for k in range(W):
            self._push(t, k)
        return t

    def _push(self, t, k):
        lm, u, v, d, cam = self.measurements(k)
        t.push_keyframe(k % (self.W + 1), self.win.kf_pose[k], lm, u, v, d, cam=cam, plane4=PLANE if self.ground else None)

    def advance(self, t, step):
        """step >= 1: keyframe W - 1 + step enters the window; the one that left a step ago frees its slot"""
        k = self.W - 1 + step
        if k >= self.W + 1:
            t.drop_keyframe(k % (self.W + 1))
        self._push(t, k)

    def request(self, step):
        W = self.W
        first, last = step, step + W - 1
        lm_sel, ptr, okf, _, _, od = _window_lists(self.per_kf, first, last)
        fixed = np.zeros(W, dtype=np.uint8); fixed[0] = 1
        req = dict(kf_slots=[k % (W + 1) for k in range(first, last + 1)], kf_fixed=fixed, lm_slots=lm_sel,
                   **_scale(self.poses[first:last + 1], int((od > 0).sum())))
        if self.ground:
            # addGroundPlaneResiduals at problem-build time: a ground point is attached to its nearest window keyframe if that
            # is closer than 25 m, with weight 10 (1 - distance / 25)
            from limo_b200 import geometry as geo
            gi = np.array([i for i, j in enumerate(lm_sel) if int(j) in self.gp], dtype=np.int64)
            T = np.stack([geo.pose_to_iso(p) for p in self.poses[first:last + 1]])
            pk = np.einsum("kij,nj->nki", T[:, :3, :3], self.win.lm_pos[lm_sel[gi]]) + T[None, :, :3, 3]
            dist = np.linalg.norm(pk, axis=2)
            best = np.argmin(dist, axis=1)
            md = dist[np.arange(len(gi)), best]
            keep = md < 25.0
            req.update(gp_lm=gi[keep].astype(np.int32), gp_kf=best[keep].astype(np.int32), gp_weight=10.0 * (1.0 - md[keep] / 25.0),
                       plane_reg_weight=10.0)
        self.cur = (first, last, lm_sel, ptr, okf)
        return req

    def record(self, res):
        first, last = self.cur[0], self.cur[1]
        self.poses[first:last + 1] = res.kf_pose

    def nudge_landmarks(self, tracks, step):
        """what a caller changes between solves: weights and positions of some landmarks, identically in every track"""
        lm_sel = self.cur[2]
        pick = lm_sel[step % 5::7][:40].astype(np.int32)
        pos = self.win.lm_pos[pick] + 0.01 * (step % 3 - 1)
        for t in tracks:
            t.set_landmarks(pick, pos=pos, weight=np.full(len(pick), 0.8))


def _equal(a, b, n_lm, what):
    assert a.c.status == 0 and b.c.status == 0, what
    assert [s.num_iterations for s in a.solves] == [s.num_iterations for s in b.solves], what
    assert np.array_equal(a.kf_pose, b.kf_pose), what
    assert np.array_equal(a.kf_plane, b.kf_plane), what
    assert np.array_equal(a.lm_pos[:n_lm], b.lm_pos[:n_lm]), what
    assert np.array_equal(a.lm_rejected[:n_lm], b.lm_rejected[:n_lm]), what
    assert a.c.final_cost == b.c.final_cost, what


@pytest.mark.gpu
def test_group_of_one_equals_track_solve():
    """a one-window group batch takes the same landmark split as the track's own batch: bit-identical with the default split"""
    from limo_b200 import capi
    h = capi.Handle(0)
    dr = _Drive(seed=71, W=10, n_lm=900, n_obs=9000)
    ta, tb = dr.make_track(h), dr.make_track(h)
    grp = capi.TrackGroup(h, [ta])
    for step in range(15):
        if step:
            dr.advance(ta, step); dr.advance(tb, step)
        req = dr.request(step)
        rg = grp.solve([req])[0]
        rt = tb.solve(**req)
        _equal(rg, rt, len(req["lm_slots"]), "step %d" % step)
        dr.record(rt)
    grp.close(); ta.close(); tb.close(); h.close()


def _mono_drives():
    """five mono sequences of different seeds, window lengths and capacities (all under 176 free reduced rows)"""
    return [_Drive(seed=81, W=5, n_lm=500, n_obs=4000), _Drive(seed=82, W=7, n_lm=700, n_obs=6000),
            _Drive(seed=83, W=9, n_lm=800, n_obs=7000), _Drive(seed=84, W=11, n_lm=1000, n_obs=9000),
            _Drive(seed=85, W=12, n_lm=1100, n_obs=10000)]


@pytest.mark.gpu
def test_homogeneous_group_equals_single_solves(monkeypatch):
    """with the landmark split pinned, a group of mono windows is bit-identical to solving them one by one -- through landmark
    updates between steps, dropped keyframes, an arena that compacts mid-drive and an automatic scale-regulariser weight"""
    from limo_b200 import capi
    monkeypatch.setenv("KBA_P_SPLIT", "6")
    h = capi.Handle(0)
    drives = _mono_drives()
    # drive 2's arena holds little more than the keyframes alive at a push: pushing the whole drive needs compactions
    c2 = drives[2].counts()
    small = max(sum(c2[k:k + drives[2].W + 1]) for k in range(drives[2].n_kf - drives[2].W)) + 50
    assert sum(c2) > small
    ga = [d.make_track(h, max_measurements=small if i == 2 else None) for i, d in enumerate(drives)]
    tw = [d.make_track(h, max_measurements=small if i == 2 else None) for i, d in enumerate(drives)]
    grp = capi.TrackGroup(h, ga)
    for step in range(15):
        reqs = []
        for i, d in enumerate(drives):
            if step:
                d.advance(ga[i], step); d.advance(tw[i], step)
            reqs.append(d.request(step))
        reqs[4]["scale_weight"] = -1.0   # the reference's rule, evaluated on the device per window
        res = grp.solve(reqs)
        for i, d in enumerate(drives):
            rt = tw[i].solve(**reqs[i])
            _equal(res[i], rt, len(reqs[i]["lm_slots"]), "step %d track %d" % (step, i))
            d.record(rt)
            if step % 4 == 2:
                d.nudge_landmarks([ga[i], tw[i]], step)
    # every push of drive 2 succeeded although its keyframes' measurements add up to more than its arena: it compacted,
    # and the group kept gathering from the arena the track points at now
    assert sum(c2[:drives[2].W + 14]) > small
    grp.close()
    for t in ga + tw:
        t.close()
    h.close()


@pytest.mark.gpu
def test_mixed_group_matches_single_solves(monkeypatch):
    """a rig and two mono tracks in one group.  The rig turns the fused linearisation off for every window, so the mono windows
    round differently than alone: compared at north_star tolerance, two-view landmarks excluded.  (A ground-plane window of
    these drives needs 30-40 iterations in its final solve, and that rounding moves its last iteration by a few: it is
    compared bit for bit in a group without a rig instead, test_skipped_tracks_keep_their_store.)"""
    from limo_b200 import capi
    monkeypatch.setenv("KBA_P_SPLIT", "6")
    h = capi.Handle(0)
    drives = [_Drive(seed=91, W=8, n_lm=800, n_obs=7000, rig=True, steps=8),
              _Drive(seed=93, W=6, n_lm=600, n_obs=5000, steps=8), _Drive(seed=94, W=10, n_lm=1000, n_obs=9000, steps=8)]
    ga = [d.make_track(h) for d in drives]
    tw = [d.make_track(h) for d in drives]
    grp = capi.TrackGroup(h, ga)
    for step in range(8):
        reqs = []
        for i, d in enumerate(drives):
            if step:
                d.advance(ga[i], step); d.advance(tw[i], step)
            reqs.append(d.request(step))
        res = grp.solve(reqs)
        for i, d in enumerate(drives):
            rt = tw[i].solve(**reqs[i])
            rg, what = res[i], "step %d track %d" % (step, i)
            n_lm = len(reqs[i]["lm_slots"])
            assert rg.c.status == 0 and rt.c.status == 0, what
            assert [s.num_iterations for s in rg.solves] == [s.num_iterations for s in rt.solves], what
            assert np.array_equal(rg.lm_rejected[:n_lm], rt.lm_rejected[:n_lm]), what
            assert np.abs(rg.kf_pose[:, 4:] - rt.kf_pose[:, 4:]).max() <= 1e-6, what
            assert abs(rg.c.final_cost - rt.c.final_cost) <= 1e-8 * abs(rt.c.final_cost), what
            _, _, _, ptr, okf = d.cur
            multi = np.array([len(np.unique(okf[ptr[j]:ptr[j + 1]])) >= 3 for j in range(n_lm)], dtype=bool)
            assert multi.sum() > 0.1 * n_lm, what
            assert np.abs(rg.lm_pos[:n_lm][multi] - rt.lm_pos[:n_lm][multi]).max() <= 1e-6, what
            d.record(rt)
            # the stores drift apart by the same rounding: restart the group member's from the twin's, so that every step
            # compares one solve
            ga[i].set_keyframe_poses(reqs[i]["kf_slots"], rt.kf_pose, rt.kf_plane)
            ga[i].set_landmarks(reqs[i]["lm_slots"], pos=rt.lm_pos[:n_lm])
    grp.close()
    for t in ga + tw:
        t.close()
    h.close()


@pytest.mark.gpu
def test_skipped_tracks_keep_their_store(monkeypatch):
    """a track that sits a step out is not solved and its store is left alone: its next solve still equals the twin's,
    which skipped the same steps.  A step in which every track sits out changes nothing.  Track 3 solves with ground-plane
    lists and the plane chain (plane_reg_weight 10) on a track created with ground capacity."""
    from limo_b200 import capi
    monkeypatch.setenv("KBA_P_SPLIT", "6")
    h = capi.Handle(0)
    drives = _mono_drives()[:3] + [_Drive(seed=92, W=8, n_lm=800, n_obs=7000, config=3, ground=True)]
    ga = [d.make_track(h) for d in drives]
    tw = [d.make_track(h) for d in drives]
    grp = capi.TrackGroup(h, ga)
    skipped = 0
    for step in range(15):
        reqs = []
        for i, d in enumerate(drives):
            if step:
                d.advance(ga[i], step); d.advance(tw[i], step)
            reqs.append(None if (step + i) % 3 == 0 or step == 7 else d.request(step))
        assert reqs[3] is None or len(reqs[3]["gp_lm"]) > 0
        res = grp.solve(reqs)
        for i, d in enumerate(drives):
            if reqs[i] is None:
                assert res[i].c.status == 0 and res[i].c.num_solves == 0 and res[i].c.num_iteration_records == 0
                skipped += 1
                continue
            rt = tw[i].solve(**reqs[i])
            _equal(res[i], rt, len(reqs[i]["lm_slots"]), "step %d track %d" % (step, i))
            d.record(rt)
    assert skipped >= 15
    grp.close()
    for t in ga + tw:
        t.close()
    h.close()


@pytest.mark.gpu
def test_group_errors_change_nothing(monkeypatch):
    from limo_b200 import capi
    monkeypatch.setenv("KBA_P_SPLIT", "6")
    h, h2 = capi.Handle(0), capi.Handle(0)
    drives = _mono_drives()[:3]
    W2 = drives[2].W
    # track 2 takes one keyframe more than its window, and exactly the observations of its fullest window: its W + 1 live
    # keyframes hold more than that at the step that solves the fullest window (at step 1 if that is step 0), as they
    # contain that window and one more keyframe
    c2, (full, full_step) = drives[2].counts(), drives[2].window_obs()
    over_step = max(full_step, 1)
    ga = [d.make_track(h, win_keyframes=W2 + 1 if i == 2 else None) for i, d in enumerate(drives)]
    tw = [d.make_track(h, win_keyframes=W2 + 1 if i == 2 else None) for i, d in enumerate(drives)]
    other = drives[0].make_track(h2)
    with pytest.raises(capi.KbaError, match="error 1"):
        capi.TrackGroup(h, [])
    with pytest.raises(capi.KbaError, match="error 1"):
        capi.TrackGroup(h, [ga[0], ga[1], ga[0]])
    with pytest.raises(capi.KbaError, match="error 1.*another handle"):
        capi.TrackGroup(h, [ga[0], other])
    grp = capi.TrackGroup(h, ga)
    checked = set()
    for step in range(15):
        reqs = []
        for i, d in enumerate(drives):
            if step:
                d.advance(ga[i], step); d.advance(tw[i], step)
            reqs.append(d.request(step))
        if step == 1:
            bad = [dict(r) for r in reqs]
            bad[1].update(kf_slots=reqs[1]["kf_slots"][:2], kf_fixed=reqs[1]["kf_fixed"][:2])
            with pytest.raises(capi.KbaError, match="error 3.*track 1"):
                grp.solve(bad)
            checked.add("kf")
        if step == 2:
            bad = [dict(r) for r in reqs]
            bad[0].update(plane_reg_weight=10.0)
            with pytest.raises(capi.KbaError, match="error 4.*track 0.*ground-plane capacity"):
                grp.solve(bad)
            checked.add("ground")
        if step == over_step:
            first = step - 1   # live keyframes: step - 1 .. step + W2 - 1
            assert sum(c2[first:first + W2 + 1]) > full
            bad = [dict(r) for r in reqs]
            fixed = np.zeros(W2 + 1, dtype=np.uint8); fixed[0] = 1
            bad[2].update(kf_slots=[k % (W2 + 1) for k in range(first, first + W2 + 1)], kf_fixed=fixed)
            with pytest.raises(capi.KbaError, match="error 4.*track 2.*win_observations"):
                grp.solve(bad)
            checked.add("obs")
        res = grp.solve(reqs)
        for i, d in enumerate(drives):
            rt = tw[i].solve(**reqs[i])
            _equal(res[i], rt, len(reqs[i]["lm_slots"]), "step %d track %d" % (step, i))
            d.record(rt)
    assert checked == {"kf", "ground", "obs"}
    grp.close()
    for t in ga + tw + [other]:
        t.close()
    h.close(); h2.close()


@pytest.mark.gpu
def test_group_upload_is_a_fraction_of_a_batch_upload():
    """the test_track.py criterion for the group: a solve sends under 10 % of what kba_batch_upload of the same windows sends"""
    from limo_b200 import capi
    from limo_b200.capi_types import Window
    h = capi.Handle(0)
    drives = _mono_drives()[2:]
    ga = [d.make_track(h) for d in drives]
    grp = capi.TrackGroup(h, ga)
    for step in range(3):
        reqs = []
        for i, d in enumerate(drives):
            if step:
                d.advance(ga[i], step)
            reqs.append(d.request(step))
        res = grp.solve(reqs)
        for d, r in zip(drives, res):
            d.record(r)
    h2d, d2h = grp.transfer_bytes()
    wins = []
    for d, r in zip(drives, reqs):
        first, last, lm_sel, ptr, okf = d.cur
        _, _, _, ou, ov, od = _window_lists(d.per_kf, first, last)
        wins.append(Window(d.poses[first:last + 1], r["kf_fixed"], d.cam_intr, d.cam_pose, d.win.lm_pos[lm_sel],
                           d.win.lm_weight[lm_sel], ptr, okf, ou, ov, od))
    batch = h.batch(wins)
    batch_h2d = batch.transfer_bytes()[0]
    assert 0 < h2d < 0.1 * batch_h2d, (h2d, batch_h2d)
    assert d2h > 0
    batch.close(); grp.close()
    for t in ga:
        t.close()
    h.close()
