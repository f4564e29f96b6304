"""Store writes of a track group (kba_track_group_push_keyframes / _drop_keyframes / _set_landmarks / _set_keyframe_poses): a group
written with the group calls holds, bit for bit, what a twin group written with the single calls holds, which the solves and the
store reads (frame flow, selection, creation) compare after every step.  A compacting arena equals one that never compacts; a
failing request changes no store; a write makes the rankings of exactly the tracks it changed stale."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_track_group import PLANE, _Drive

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = 6          # keyframes per window
STEPS = 30     # pushes per track


def test_write_struct_sizes_match_header(tmp_path):
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu %zu\\n",sizeof(kba_push_request),'
                    'sizeof(kba_landmark_write),sizeof(kba_pose_write));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(t) for t in (T.KbaPushRequest, T.KbaLandmarkWrite, T.KbaPoseWrite)]


def test_write_symbols_exported():
    from limo_b200 import capi
    L = capi.lib()
    for n in ("kba_track_group_push_keyframes", "kba_track_group_drop_keyframes", "kba_track_group_set_landmarks",
              "kba_track_group_set_keyframe_poses"):
        assert n in capi.SYMBOLS and hasattr(L, n), n


def test_group_store_bench_dry_run():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "group_store_bench.py"), "--dry-run"], capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr
    assert '"dry_run": true' in out.stdout


# ---- the drive: four kinds of track, each keyframe k in slot k % (W + 1); slot W + 1 holds an empty keyframe for one step -------
class _Kind:
    def __init__(self, seed, rig=False, ground=False, mono_cam=False, tight=False):
        self.d = _Drive(seed=seed, W=W, n_lm=500, n_obs=(W + STEPS) * 160, config=3 if ground else 2, rig=rig, ground=ground,
                        steps=STEPS)
        self.mono_cam, self.tight = mono_cam, tight
        c = self.d.counts()
        # a tight arena holds little more than the live keyframes and the pushed one: it compacts on most pushes
        self.m_cap = max(sum(c[s:s + W + 1]) for s in range(len(c) - W)) + 8 if tight else 4 * sum(c)

    def push_args(self, k, empty=False):
        lm, u, v, d, cam = self.d.measurements(k)
        o = np.lexsort((cam, lm))[:0 if empty else len(lm)]  # the store's contract: one run per landmark, cameras ascending
        lm, u, v, d, cam = lm[o], u[o], v[o], d[o], cam[o]
        return dict(slot=W + 1 if empty else k % (W + 1), pose7=self.d.win.kf_pose[k], lm_slot=lm, u=u, v=v, d=d,
                    cam=None if self.mono_cam else cam, plane4=PLANE if self.d.ground else None)

    def make(self, h, m_cap=None):
        from limo_b200 import capi
        d = self.d
        t = capi.Track(h, d.cam_intr, d.cam_pose, max_keyframes=W + 2, max_landmarks=d.win.n_lm, max_measurements=m_cap or self.m_cap,
                       win_keyframes=W, win_landmarks=d.win.n_lm, win_observations=d.window_obs()[0],
                       win_ground=len(d.gp) if d.ground else 0)
        t.set_landmarks(np.arange(d.win.n_lm, dtype=np.int32), pos=d.win.lm_pos, weight=d.win.lm_weight)
        for k in range(W):
            t.push_keyframe(**self.push_args(k))
        return t


def _kinds():
    # mono (cameras NULL), two-camera rig, ground plane with plane4, mono with an arena that compacts
    return [_Kind(71), _Kind(72, rig=True), _Kind(73, ground=True), _Kind(74, mono_cam=True, tight=True)]


def _same(a, b, what):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _same(a[k], b[k], "%s.%s" % (what, k))
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, "%s[%d]" % (what, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), what
    else:
        assert a == b or (a != a and b != b), (what, a, b)


def _same_result(a, b, what):
    assert a.c.status == 0 and b.c.status == 0, what
    assert [s.num_iterations for s in a.solves] == [s.num_iterations for s in b.solves], what
    for f in ("kf_pose", "kf_plane", "lm_pos", "lm_rejected"):
        _same(getattr(a, f), getattr(b, f), "%s %s" % (what, f))
    assert (a.c.initial_cost, a.c.final_cost) == (b.c.initial_cost, b.c.final_cost), what


def _reads(grp, kinds, si):
    """the store reads that cover every arena field: frame flow (lm, cam, u, v), selection (lm), creation (lm, cam, u, v, d)"""
    flow, sel, cre = [], [], []
    for kd, s in zip(kinds, si):
        first, newest = s, s + W - 1
        slots = [k % (W + 1) for k in range(first, newest + 1)]
        lm, u, v, _, cam = kd.d.measurements(newest + 1)
        o = np.lexsort((cam, lm))  # a frame's measurements in runs by landmark, cameras ascending
        flow.append(dict(kf_last=newest % (W + 1), lm_slot=lm[o], u=u[o], v=v[o], cam=cam[o]))
        sel.append(dict(kf_slots=slots, lm_slots=np.unique(np.concatenate([kd.d.per_kf[k][0] for k in range(first, newest + 1)]))))
        cre.append(dict(kf_slots=slots, kf_new=W - 1, lm_slots=np.unique(kd.d.per_kf[newest][0])[:80]))
    return grp.frame_flow(flow), grp.select_landmarks(sel), grp.create_landmarks(cre)


def _solve(grp, kinds, si):
    from limo_b200 import capi
    opt = capi.default_options()
    opt.solver_time_sec = 20.0
    return grp.solve([kd.d.request(s) for kd, s in zip(kinds, si)], opt=opt)


@pytest.mark.gpu
def test_group_pushes_equal_single_pushes():
    """30 steps of drop + push with sit-outs and an empty keyframe: group A written with the group calls, B with the single calls,
    and a never-compacting twin of the compacting track; solves and store reads bit-identical after every step"""
    from limo_b200 import capi
    h = capi.Handle(0)
    kinds = _kinds()
    ta = [kd.make(h) for kd in kinds]
    tb = [kd.make(h) for kd in kinds]
    twin = kinds[3].make(h, m_cap=4 * sum(kinds[3].d.counts()))
    ga, gb = capi.TrackGroup(h, ta + [kinds[3].make(h, m_cap=4 * sum(kinds[3].d.counts()))]), capi.TrackGroup(h, tb + [twin])
    kinds5 = kinds + [kinds[3]]
    si = [0] * 5             # each track's step: its newest keyframe is W - 1 + si
    counts3 = kinds[3].d.counts()
    used3, compactions = sum(counts3[:W]), 0  # the compacting track's arena, as its host mirror keeps it
    for step in range(STEPS):
        sits = [(step + i) % 4 == 3 for i in range(4)]
        sits.append(sits[3])  # the twin follows the compacting track
        drops, pushes = [None] * 5, [None] * 5
        for i in range(5):
            if sits[i]:
                continue
            k = W + si[i]
            if k >= W + 1:
                drops[i] = k % (W + 1)
            pushes[i] = kinds5[i].push_args(k)
            si[i] += 1
        if pushes[3] is not None:
            k = W - 1 + si[3]
            if used3 + counts3[k] > kinds[3].m_cap:
                compactions += 1
                used3 = sum(counts3[k - W:k])
            used3 += counts3[k]
        if step == 8:  # the empty keyframe of step 7 leaves
            ga.drop_keyframes([W + 1] + [None] * 4)
            tb[0].drop_keyframe(W + 1)
        ga.drop_keyframes(drops)
        ga.push_keyframes(pushes)
        for i, t in enumerate(tb + [twin]):
            if drops[i] is not None:
                t.drop_keyframe(drops[i])
            if pushes[i] is not None:
                t.push_keyframe(**pushes[i])
        if step == 7:  # a keyframe without measurements in the spare slot of track 0
            req = kinds[0].push_args(0, empty=True)
            ga.push_keyframes([req] + [None] * 4)
            tb[0].push_keyframe(**req)
        ra, rb = _solve(ga, kinds5, si), _solve(gb, kinds5, si)
        for i in range(5):
            _same_result(ra[i], rb[i], "step %d track %d" % (step, i))
        _same_result(ra[3], ra[4], "step %d: compacting track against its twin" % step)
        for kd, s, r in zip(kinds, si, ra):
            kd.d.request(s)
            kd.d.record(r)
        reads = _reads(ga, kinds5, si)
        _same(reads, _reads(gb, kinds5, si), "step %d reads" % step)
        for q in range(3):
            _same(reads[q][3], reads[q][4], "step %d: compacting track's reads against its twin" % step)
    assert compactions > 10
    for g in (ga, gb):
        g.close()
    for t in ta + tb + [twin] + ga.tracks[4:]:
        t.close()
    h.close()


def _write_tracks(h, n_tracks, big):
    """tracks with more landmark slots than one window (max(win_landmarks, 64) rows is a write's staging per track)"""
    from limo_b200 import capi
    d = _Drive(seed=81, W=W, n_lm=120, n_obs=(W + 2) * 60, steps=2)
    out = []
    for _ in range(n_tracks):
        t = capi.Track(h, d.cam_intr, d.cam_pose, max_keyframes=W + 1, max_landmarks=big, max_measurements=sum(d.counts()),
                       win_keyframes=W, win_landmarks=d.win.n_lm, win_observations=d.window_obs()[0])
        pos, wt = np.zeros((big, 3)), np.ones(big)  # every slot written: the free ones are read back
        pos[:d.win.n_lm], wt[:d.win.n_lm] = d.win.lm_pos, d.win.lm_weight
        t.set_landmarks(np.arange(big, dtype=np.int32), pos=pos, weight=wt)
        for k in range(W):
            lm, u, v, dd, cam = d.measurements(k)
            t.push_keyframe(k, d.win.kf_pose[k], lm, u, v, dd, cam=cam)
        out.append(t)
    return d, out


@pytest.mark.gpu
def test_set_landmarks_and_poses_equal_single_calls():
    """NULL pos / weight / planes, n = 0, and lists longer than the staging of a track: group and single writes bit-identical, read
    back through the free slots' stored values (reclaim with evict) and through a solve with every keyframe fixed"""
    from limo_b200 import capi
    h = capi.Handle(0)
    big = 1000
    d, ta = _write_tracks(h, 3, big)
    _, tb = _write_tracks(h, 3, big)
    ga = capi.TrackGroup(h, ta)
    rng = np.random.default_rng(5)
    n_lm = d.win.n_lm
    for rnd in range(3):
        reqs = []
        for i in range(3):
            n = [0, 700, 40][(i + rnd) % 3]  # 700 > the 120-row staging of a track
            slot = rng.permutation(np.arange(n_lm, big))[:n].astype(np.int32)
            pos = rng.normal(size=(n, 3)) if (i + rnd) % 2 == 0 else None
            wt = None if (i + rnd) % 3 == 1 else rng.uniform(0.5, 1.0, n)  # i + rnd = 1: neither pos nor weight
            reqs.append(None if n == 0 and rnd == 0 else dict(lm_slot=slot, pos=pos, weight=wt))
        ga.set_landmarks(reqs)
        for t, r in zip(tb, reqs):
            if r is not None:
                t.set_landmarks(r["lm_slot"], pos=r["pos"], weight=r["weight"])
        for a, b in zip(ta, tb):
            _same(a.reclaim_landmarks(n_lm, big, evict=True), b.reclaim_landmarks(n_lm, big, evict=True), "landmarks round %d" % rnd)
    # poses: more keyframes than the store has slots come in as duplicates, so stay within them; planes NULL on one track
    for rnd in range(2):
        reqs = []
        for i in range(3):
            slots = rng.permutation(W)[:[W, 0, 3][(i + rnd) % 3]].astype(np.int32)
            poses = d.win.kf_pose[slots] + np.r_[0.0, 0, 0, 0, 1e-3, 0, 0] * (rnd + 1)
            reqs.append(dict(kf_slots=slots, pose7s=poses, plane4s=None if i == 1 else np.tile(PLANE, (len(slots), 1))))
        ga.set_keyframe_poses(reqs)
        for t, r in zip(tb, reqs):
            t.set_keyframe_poses(r["kf_slots"], r["pose7s"], r["plane4s"])
    opt = capi.default_options()
    req = d.request(0)
    req["kf_fixed"] = np.ones(W, np.uint8)
    for a, b in zip(ta, tb):
        _same_result(a.solve(opt=opt, **req), b.solve(opt=opt, **req), "poses")
    assert ga.set_landmarks([None, dict(lm_slot=[]), None]) is None and ga.transfer_bytes() == (0, 0)
    ga.close()
    for t in ta + tb:
        t.close()
    h.close()


@pytest.mark.gpu
def test_failing_write_changes_nothing():
    """a slot in use, a slot or camera out of range, an arena full even after compaction: the single call's code, the track named,
    and every store as an untouched twin's"""
    from limo_b200 import capi
    h = capi.Handle(0)
    kinds = _kinds()
    ta = [kd.make(h) for kd in kinds]
    tb = [kd.make(h) for kd in kinds]
    ga = capi.TrackGroup(h, ta)
    good = [kd.push_args(W) for kd in kinds]  # slot W: free
    bad_cam = dict(good[1], cam=np.full(len(good[1]["lm_slot"]), 2, np.int32))
    lm3 = kinds[3].d.measurements(W)[0]
    n_full = kinds[3].m_cap + 1
    full = dict(good[3], lm_slot=np.resize(lm3, n_full), u=np.zeros(n_full, np.float32), v=np.zeros(n_full, np.float32),
                d=np.zeros(n_full, np.float32))
    cases = [(2, dict(good[2], slot=0), 1, "slot in use"), (1, dict(good[1], slot=W + 2), 1, "out of range"),
             (1, bad_cam, 1, "camera out of range"), (3, full, 4, "arena full")]
    for i, bad, code, msg in cases:
        reqs = list(good)
        reqs[i] = bad
        with pytest.raises(capi.KbaError, match="error %d: kba_track_group_push_keyframes: track %d: .*%s" % (code, i, msg)):
            ga.push_keyframes(reqs)
        with pytest.raises(capi.KbaError, match="error %d: .*%s" % (code, msg)):
            tb[i].push_keyframe(**bad)
    with pytest.raises(capi.KbaError, match="track 2: keyframe slot out of range"):
        ga.drop_keyframes([None, 1, W + 2, None])
    with pytest.raises(capi.KbaError, match="track 1: landmark slot out of range"):
        ga.set_landmarks([dict(lm_slot=[1], weight=[0.5]), dict(lm_slot=[10 ** 6], weight=[0.5]), None, None])
    with pytest.raises(capi.KbaError, match="track 3: keyframe slot out of range"):
        ga.set_keyframe_poses([dict(kf_slots=[0], pose7s=[kinds[0].d.win.kf_pose[0]]), None, None,
                               dict(kf_slots=[-1], pose7s=[kinds[0].d.win.kf_pose[0]])])
    gb = capi.TrackGroup(h, tb)
    ra, rb = _solve(ga, kinds, [0] * 4), _solve(gb, kinds, [0] * 4)
    for i in range(4):
        _same_result(ra[i], rb[i], "track %d after the failed calls" % i)
    ga.close()
    gb.close()
    for t in ta + tb:
        t.close()
    h.close()


@pytest.mark.gpu
def test_writes_make_exactly_the_changed_rankings_stale():
    from limo_b200 import capi
    h = capi.Handle(0)
    kinds = _kinds()[:3]
    ts = [kd.make(h) for kd in kinds]
    g = capi.TrackGroup(h, ts)
    slots = list(range(W))
    fixed = np.r_[1, np.zeros(W - 1)].astype(np.uint8)
    writes = [lambda i: g.set_landmarks([dict(lm_slot=[3], weight=[0.7]) if j == i else None for j in range(3)]),
              lambda i: g.set_keyframe_poses([dict(kf_slots=[1], pose7s=[kinds[j].d.win.kf_pose[1]]) if j == i else None for j in range(3)]),
              lambda i: g.drop_keyframes([W if j == i else None for j in range(3)]),
              lambda i: g.push_keyframes([dict(kinds[j].push_args(W), slot=W) if j == i else None for j in range(3)])]
    for wi, write in enumerate(writes):
        changed = wi % 3
        ranks = [dict(kf_slots=slots, lm_slots=np.unique(kd.d.per_kf[W - 1][0]), draws=lambda n: np.arange(n)) for kd in kinds]
        g.rank_landmarks(ranks)
        write(changed)
        for i, t in enumerate(ts):
            if i == changed:
                with pytest.raises(capi.KbaError, match="stale"):
                    t.solve_ranked(slots, fixed)
            else:
                assert t.solve_ranked(slots, fixed).c.status == 0
    g.close()
    for t in ts:
        t.close()
    h.close()


@pytest.mark.gpu
def test_group_push_upload_is_its_rows_plus_a_record_per_track():
    from limo_b200 import capi
    h = capi.Handle(0)
    kinds = [_Kind(91 + i) for i in range(4)]
    ts = [kd.make(h) for kd in kinds]
    g = capi.TrackGroup(h, ts)
    reqs = [dict(kd.push_args(W), slot=W) for kd in kinds]
    reqs[1]["lm_slot"], reqs[1]["u"], reqs[1]["v"], reqs[1]["d"] = (reqs[1][k][:0] for k in ("lm_slot", "u", "v", "d"))
    g.push_keyframes(reqs)
    rows = 20 * sum(len(r["lm_slot"]) for r in reqs)
    h2d, d2h = g.transfer_bytes()
    assert rows <= h2d <= rows + 256 * len(reqs) and d2h == 0, (h2d, rows)
    _, _, push = ts[0].transfer_bytes()
    g.drop_keyframes([W, None, None, None])
    assert g.transfer_bytes() == (0, 0) and ts[0].transfer_bytes()[2] == push
    g.close()
    for t in ts:
        t.close()
    h.close()
