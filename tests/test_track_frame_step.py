"""limo's frame step as one store call -- kba_track_frame_step and its group forms -- against the chain of store calls it replaces:
adjust_pose on the selected runs, frame_flow over all rows, the Python statement of limo's KeyframeSelector with the adjusted pose,
push_keyframe with the adjusted pose and create_landmarks.  Two copies of each store (Track.clone) go through the closed-loop drives
of tests/keyframe_drive.py; after every frame the outputs and the snapshots of the two stores must be equal byte for byte."""
import ctypes as C

import numpy as np
import pytest

from limo_b200.capi_types import parse_snapshot
from limo_b200.keyframe_selector import calcQuaternionDiff, convert_sec
from tests.keyframe_drive import KeyframeDrive
from tests.test_track_rank import _same_result


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


class Loop:
    """a caller's bookkeeping of one track over a KeyframeDrive: the active keyframes (slot, stamp), LandmarkId -> slot with slots
    recycled after drops, the created landmarks; it builds each frame's request and runs the chain of single calls"""

    def __init__(self, dr, seed, lm_cap):
        self.dr, self.rng = dr, np.random.default_rng(seed)
        self.window = dr.window // 2       # the keyframes a caller keeps: the oldest is dropped beyond it, so slots recycle
        self.S = self.window + 2
        self.active = []                   # (slot, stamp), oldest first
        self.slot_of, self.created, self.free, self.used = {}, set(), [], set()
        self.next_slot, self.lm_cap = 0, lm_cap
        self.seen = dict(flow_reject=0, nan=0, by_pose=0, by_time=0, no_adjust=0, speed=0, by_depth=0, by_tri=0, not_created=0,
                         reused=0)
        self.pushed_rows = 0

    def _slot(self, lid):
        if lid not in self.slot_of:
            s = self.free.pop(0) if self.free else self.next_slot
            if s == self.next_slot:
                self.next_slot += 1
            self.seen["reused"] += s in self.used
            self.slot_of[lid] = s
        return self.slot_of[lid]

    def request(self, k):
        dr, rng = self.dr, self.rng
        lid, cam, u, v = dr.arena(k)
        d = np.where(rng.random(len(lid)) < 0.4, rng.uniform(4.0, 40.0, len(lid)), -1.0).astype(np.float32)
        lm = np.array([self._slot(int(a)) for a in lid], np.int32)
        starts = np.r_[True, lid[1:] != lid[:-1]] if len(lid) else np.zeros(0, bool)
        run_ids = lid[starts]
        run_sel = np.array([int(a) in self.created and rng.random() < 0.9 for a in run_ids], bool)
        new = [self.slot_of[int(a)] for a in run_ids if int(a) not in self.created]
        f = dr.frames[k]
        free_kf = sorted(set(range(self.S)) - {s for s, _ in self.active})
        r = dict(kf_slots=[s for s, _ in self.active], lm_slot=lm, cam=cam, u=u, v=v, d=d, run_sel=run_sel, kf_new=free_kf[0],
                 new_slots=new, pose7=f.pose_, plane4=[0.0, 0.0, 1.0, 0.01 * k], adjust=k % 6 != 5, min_median_flow=dr.thr[k],
                 critical_quaternion_diff=dr.critical, time_difference_ns=convert_sec(dr.time_sec), stamp=f.timestamp_,
                 stamp_last=self.active[-1][1] if self.active else 0)
        if k % 4 == 1:
            r["speed"] = dict(weight=0.5, dt=0.1, v_before=rng.normal(0, 1, 3), T_origin_before=f.pose_)
        return r, run_ids

    def chain(self, t, r, ref_snap, opt):
        """the single calls a caller runs today, with the selector's verdicts on the host; sets a pose threshold the frame passes
        on some frames where only the pose scheme could select it"""
        lm, cam, u, v, d = (np.asarray(r[k]) for k in ("lm_slot", "cam", "u", "v", "d"))
        starts = np.r_[True, lm[1:] != lm[:-1]] if len(lm) else np.zeros(0, bool)
        rows = np.asarray(r["run_sel"], bool)[np.cumsum(starts) - 1] if len(lm) else np.zeros(0, bool)
        res, pose = None, np.asarray(r["pose7"], np.float64)
        if r["adjust"] and rows.any():
            res = t.adjust_pose(r["pose7"], lm[rows], u[rows], v[rows], d[rows], cam=cam[rows], speed=r.get("speed"), opt=opt)
            pose = res.kf_pose[0].copy()
        fl = t.frame_flow(r["kf_slots"][-1], lm, u, v, cam=cam, min_median_flow=r["min_median_flow"])
        sn = parse_snapshot(ref_snap)
        last = sn["pose"][list(sn["slot"]).index(r["kf_slots"][-1])]
        angle = calcQuaternionDiff(list(pose), list(last))
        flow_ok = len(lm) > 0 and fl["usable"]
        time_ok = (r["stamp"] - r["stamp_last"]) % 2**64 > r["time_difference_ns"]
        if flow_ok and not time_ok and angle > 0 and self.rng.random() < 0.5:
            r["critical_quaternion_diff"] = angle * 0.5
        pose_ok = angle > r["critical_quaternion_diff"]
        sel = flow_ok and (pose_ok or time_ok)
        out = dict(fl, angle=angle, usable_flow=flow_ok, usable_pose=pose_ok, usable_time=time_ok, selected=sel, result=res, pos=None, flags=None)
        if sel:
            t.push_keyframe(r["kf_new"], pose, lm, u, v, d, cam=cam, plane4=r["plane4"])
            out["pos"], out["flags"] = t.create_landmarks(list(r["kf_slots"]) + [r["kf_new"]], len(r["kf_slots"]), r["new_slots"])
        return out

    def advance(self, tracks, r, run_ids, out, k):
        """the bookkeeping after a frame: coverage, the new keyframe, the window's oldest keyframe dropped, freed slots recycled"""
        s = self.seen
        s["flow_reject"] += not out["usable_flow"]
        s["nan"] += out["n_matched"] == 0 and len(r["lm_slot"]) > 0
        s["by_pose"] += out["selected"] and out["usable_pose"] and not out["usable_time"]
        s["by_time"] += out["selected"] and out["usable_time"] and not out["usable_pose"]
        s["no_adjust"] += not r["adjust"]
        s["speed"] += "speed" in r and out["result"] is not None and out["result"].c.num_solves > 0
        if not out["selected"]:
            return
        fl = out["flags"]
        s["by_depth"] += int(((fl & 3) == 3).sum())
        s["by_tri"] += int(((fl & 3) == 1).sum())
        s["not_created"] += int(((fl & 1) == 0).sum())
        self.pushed_rows += len(r["lm_slot"])
        by_slot = {self.slot_of[int(a)]: int(a) for a in run_ids}
        self.created |= {by_slot[sl] for sl, f in zip(r["new_slots"], fl) if f & 1}
        self.used |= set(int(x) for x in r["lm_slot"])
        self.active.append((r["kf_new"], r["stamp"]))
        if len(self.active) > self.window:
            self.drop(tracks, [self.active[0][0]])

    def drop(self, tracks, slots):
        for t in tracks:
            for sl in slots:
                t.drop_keyframe(sl)
        self.active = [a for a in self.active if a[0] not in slots]
        freed = set(int(x) for x in tracks[0].reclaim_landmarks(0, self.next_slot))
        for lid in [a for a, sl in self.slot_of.items() if sl in freed]:
            del self.slot_of[lid]
            self.created.discard(lid)
        self.free = sorted(set(self.free) | freed)

    def first(self, tracks):
        """frame 0 pushed as the first keyframe on every copy, its landmarks created by depth where it has one"""
        r, run_ids = self.request(0)
        r.update(d=np.where(np.arange(len(r["d"])) % 3 == 0, -1.0, 10.0).astype(np.float32))
        for t in tracks:
            t.push_keyframe(r["kf_new"], r["pose7"], r["lm_slot"], r["u"], r["v"], r["d"], cam=r["cam"])
            pos, fl = t.create_landmarks([r["kf_new"]], 0, r["new_slots"])
        by_slot = {self.slot_of[int(a)]: int(a) for a in run_ids}
        self.created |= {by_slot[sl] for sl, f in zip(r["new_slots"], fl) if f & 1}
        self.used |= set(int(x) for x in r["lm_slot"])
        self.active.append((r["kf_new"], r["stamp"]))


def _track(h, dr, m_cap):
    from limo_b200 import capi
    rows = max(len(dr.arena(k)[0]) for k in range(dr.n_frames))
    w = dr.window // 2
    return capi.Track(h, dr.cam_intr, dr.cam_pose, max_keyframes=w + 2, max_landmarks=dr.n_lm + 1, max_measurements=m_cap,
                      win_keyframes=w + 1, win_landmarks=max(rows, dr.n_lm + 1), win_observations=(w + 1) * rows), rows


def _options():
    from limo_b200 import capi
    opt = capi.default_options()
    opt.solver_time_sec = 0.0  # no time limit: both copies run the same iterations
    return opt


def _same_step(one, ref, where):
    for key in ("n_matched", "usable_flow", "usable_pose", "usable_time", "selected"):
        assert one[key] == ref[key], (where, key)
    for key in ("flow_sum", "mean_flow_sq", "angle"):
        assert _bits(one[key]) == _bits(ref[key]), (where, key)
    assert np.array_equal(one["match"], ref["match"]), where
    if ref["result"] is None:
        assert one["result"].c.num_solves == 0 and one["result"].c.status == 0, where
    else:
        _same_result(one["result"], ref["result"])
        assert (one["result"].c.num_iteration_records, [i.cost for i in one["result"].iterations]) == \
            (ref["result"].c.num_iteration_records, [i.cost for i in ref["result"].iterations]), where
    if ref["selected"]:
        assert np.array_equal(_bits(one["pos"]), _bits(ref["pos"])) and np.array_equal(one["flags"], ref["flags"]), where
    else:
        assert one["pos"] is None and one["flags"] is None, where


DRIVES = [dict(seed=1, window=12, rig=False), dict(seed=2, window=12, rig=True), dict(seed=3, window=20, rig=False, n_frames=80),
          dict(seed=4, window=20, rig=True, n_frames=80)]


@pytest.mark.gpu
@pytest.mark.parametrize("kw", DRIVES, ids=lambda kw: "w%d_%s" % (kw["window"], "rig" if kw["rig"] else "mono"))
def test_frame_step_equals_the_chain(kw):
    from limo_b200 import capi
    dr = KeyframeDrive(**kw)
    h = capi.Handle(0)
    probe, rows = _track(h, dr, 1)
    probe.close()
    m_cap = (dr.window // 2 + 1) * rows + rows // 2  # small: the arena compacts inside steps
    a, _ = _track(h, dr, m_cap)
    b = a.clone()
    loop = Loop(dr, kw["seed"], dr.n_lm + 1)
    loop.first([a, b])
    opt = _options()
    for k in range(1, dr.n_frames):
        r, run_ids = loop.request(k)
        snap = a.snapshot()
        ref = loop.chain(a, r, snap, opt)
        one = b.frame_step(opt=opt, **r)
        _same_step(one, ref, k)
        assert bytes(a.snapshot()) == bytes(b.snapshot()), k
        if not one["selected"]:
            assert bytes(b.snapshot()) == bytes(snap), k  # a frame that is not selected leaves the store untouched
        loop.advance([a, b], r, run_ids, one, k)
    assert loop.pushed_rows > m_cap, (loop.pushed_rows, m_cap)  # some step compacted the arena
    assert all(v > 0 for v in loop.seen.values()), loop.seen
    a.close(); b.close(); h.close()


@pytest.mark.gpu
def test_group_frame_step_equals_single_calls():
    """8 tracks, one sitting out per frame, per-track options: every output and snapshot equals the single call's on a clone;
    the calls include frames where no track is selected; the transfers follow the header's formulas"""
    from limo_b200 import capi
    h = capi.Handle(0)
    drs = [KeyframeDrive(60 + i, n_frames=40, window=6 + (i % 3), rig=bool(i % 2), n_feat=120 + 20 * i) for i in range(8)]
    gt, st, loops = [], [], []
    for i, dr in enumerate(drs):
        t, rows = _track(h, dr, 1)
        t.close()
        t, _ = _track(h, dr, (dr.window // 2 + 1) * rows + rows // 2)
        gt.append(t)
        st.append(t.clone())
        loops.append(Loop(dr, 90 + i, dr.n_lm + 1))
        loops[i].first([gt[i], st[i]])
    g = capi.TrackGroup(h, gt)
    opts = [_options() for _ in drs]
    for i, o in enumerate(opts):
        o.reprojection_thres = 1.2 + 0.1 * i
    none_selected = mixed = 0
    terms = []
    for k in range(1, 40):
        reqs, ids = [], []
        for i, lp in enumerate(loops):
            r, run_ids = lp.request(k)
            reqs.append(None if i == k % 8 else r)
            ids.append(run_ids)
        outs = g.frame_step(reqs, opt=opts)
        assert outs[k % 8] is None
        terms.append(_transfer_terms(reqs, outs, *g.transfer_bytes()))
        picked = [o["selected"] for o in outs if o is not None]
        none_selected += not any(picked)
        mixed += any(picked) and not all(picked)
        for i, r in enumerate(reqs):
            if r is None:
                continue
            one = st[i].frame_step(opt=opts[i], **r)
            _same_step(outs[i], one, (k, i))
            assert bytes(gt[i].snapshot()) == bytes(st[i].snapshot()), (k, i)
            loops[i].advance([gt[i], st[i]], r, ids[i], one, k)
    assert none_selected > 0 and mixed > 0, (none_selected, mixed)
    _check_transfers(terms)
    g.close()
    for t in gt + st:
        t.close()
    h.close()


def _transfer_terms(reqs, outs, up, down):
    """(W, A, S, the constant part of h2d, of d2h) of a group call: what the header's formulas leave after the per-request terms"""
    live = [(r, o) for r, o in zip(reqs, outs) if r is not None]
    adj = [r for r, _ in live if r["adjust"] and np.any(r["run_sel"])]
    sel = [r for r, o in live if o["selected"]]
    var_up = sum(20 * len(r["lm_slot"]) + 4 * (len(r["kf_slots"]) + 1 + len(r["new_slots"])) + len(r["run_sel"]) for r, _ in live)
    var_down = sum(4 * len(r["lm_slot"]) + 80 for r, _ in live) + sum(int(np.sum(r["run_sel"])) for r in adj)
    var_down += 25 * sum(len(r["new_slots"]) for r in sel)
    return len(live), len(adj), len(sel), up - var_up, down - var_down


def _check_transfers(terms):
    """h2d without a selection is R_1 W + R_a A and d2h is (R_f + 160 R_i) A (iteration capacity 256 > 160 records) for one set of
    record sizes, multiples of 8, over every call"""
    rows = [(w, a, c) for w, a, s, c, _ in terms if s == 0]
    M = np.array([[w, a] for w, a, _ in rows], float)
    R, *_ = np.linalg.lstsq(M, np.array([c for *_, c in rows], float), rcond=None)
    R = np.round(R).astype(np.int64)
    assert np.array_equal(M.astype(np.int64) @ R, [c for *_, c in rows]) and np.all(R % 8 == 0) and np.all(R > 0), R
    per = {d // a for _, a, _, _, d in terms if a}
    assert len(per) == 1 and all(d == 0 for _, a, _, _, d in terms if not a), per
    for w, a, s, c, _ in terms:  # a selection adds its records to the upload
        assert s == 0 or c > R[0] * w + R[1] * a


@pytest.mark.gpu
def test_refused_requests_write_nothing():
    from limo_b200 import capi
    dr = KeyframeDrive(5, n_frames=12, window=6, rig=False)
    h = capi.Handle(0)
    t, rows = _track(h, dr, 1)
    t.close()
    t, _ = _track(h, dr, (dr.window // 2 + 1) * rows + rows // 2)
    u = t.clone()
    g = capi.TrackGroup(h, [t, u])
    loop = Loop(dr, 5, dr.n_lm + 1)
    loop.first([t, u])
    r, _ids = loop.request(1)
    snap = bytes(t.snapshot())
    bad = [dict(r, kf_new=r["kf_slots"][0]),                              # a push slot in use
           dict(r, lm_slot=np.where(np.arange(len(r["lm_slot"])) == 0, 10**6, r["lm_slot"])),  # a slot out of range
           dict(r, new_slots=list(r["new_slots"][:1]) * 2)]                # a new slot listed twice
    for q in bad:
        with pytest.raises(capi.KbaError):
            t.frame_step(**q)
        with pytest.raises(capi.KbaError, match="track 1"):
            g.frame_step([r, q])
        assert bytes(t.snapshot()) == snap and bytes(u.snapshot()) == snap
    small, _ = _track(h, dr, rows // 2)  # an arena too small for the frame, were it selected
    small_r = dict(r, kf_slots=[0])
    small.push_keyframe(0, r["pose7"], [], [], [], [])
    before = bytes(small.snapshot())
    with pytest.raises(capi.KbaError, match="arena full"):
        small.frame_step(**dict(small_r, kf_new=1))
    assert bytes(small.snapshot()) == before
    # a refused group call writes no output: the records' outputs keep their initial values
    fn = capi.lib().kba_track_group_frame_step
    req, out, ress, _keep, _res = capi._frame_step_records(fn, [r, bad[0]], 4)
    rc = fn(g._p, req.ctypes.data_as(C.POINTER(capi.KbaFrameStepRequest)), C.byref(_options()),
            out.ctypes.data_as(C.POINTER(capi.KbaFrameStepOut)), ress)
    assert rc != 0
    assert out["n_matched"].tolist() == [0, 0] and out["angle"].tolist() == [0.0, 0.0]
    assert _keep[5][0] == 0 and ress[0].num_iteration_records == 0
    small.close(); g.close(); t.close(); u.close(); h.close()


@pytest.mark.gpu
def test_whole_loop_with_keyframe_solves():
    """40 frames of frame_step with keyframe_solve on the selected ones, against the chain of single calls with the same solves:
    the snapshots stay equal"""
    from limo_b200 import capi
    dr = KeyframeDrive(7, n_frames=40, window=12, rig=True)
    h = capi.Handle(0)
    t, rows = _track(h, dr, 1)
    t.close()
    a, _ = _track(h, dr, (dr.window // 2 + 1) * rows + rows // 2)
    b = a.clone()
    loop = Loop(dr, 7, dr.n_lm + 1)
    loop.first([a, b])
    opt = _options()
    solves = 0
    for k in range(1, 40):
        r, run_ids = loop.request(k)
        ref = loop.chain(a, r, a.snapshot(), opt)
        one = b.frame_step(opt=opt, **r)
        _same_step(one, ref, k)
        loop.advance([a, b], r, run_ids, one, k)
        if one["selected"] and len(loop.active) >= 3:
            kf = [s for s, _ in loop.active]
            lms = sorted(loop.slot_of[i] for i in loop.created)
            kw = dict(kf_slots=kf, lm_slots=lms, max_window=dr.window, draws=np.arange(len(lms) + 1), voxel_size=(0.5, 0.5, 0.3),
                      scale_weight=-1.0, scale_value=1.5)
            sa, sb = a.keyframe_solve(opt=opt, **kw), b.keyframe_solve(opt=opt, **kw)
            _same_result(sa["result"], sb["result"])
            gone = [s for s, f in zip(kf, sb["kf_active"]) if not f]
            if gone:
                loop.drop([a, b], gone)
            solves += sa["result"].c.num_solves > 0
        assert bytes(a.snapshot()) == bytes(b.snapshot()), k
    assert solves > 0
    a.close(); b.close(); h.close()
