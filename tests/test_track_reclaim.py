"""Free landmark slots of the device-resident store (kba_track_reclaim_landmarks / kba_track_group_reclaim_landmarks).

Without a GPU: the C structs against their ctypes mirrors, and the statement of the call (free = in the range and named by no
arena entry of a live keyframe, tests/reclaim_drive.free_slots) driving a caller's slot bookkeeping (SlotBook) over a long drive.
On the GPU:
  - twin tracks: A has far fewer landmark slots than the drive has landmarks, reclaims whenever a push needs more, hands freed
    slots out LIFO and restores re-measured landmarks from what the reclaim evicted; B has slot = landmark id.  At every step
    every store call -- create_landmarks, deactivate_keyframes, depth_costs, select_landmarks, solve, adjust_pose, frame_flow --
    gives A and B the same outputs bit for bit, and after every drop and push A's and B's free slots equal the statement, the
    evicted values what was last written to those slots;
  - a group equals the single calls (with a request sitting out), and the transfer counts follow the header;
  - every invalid request fails before anything is written."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.reclaim_drive import ReclaimDrive, SlotBook, free_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all"])


def _live_cap(dr, ring):
    """the most distinct landmarks of `ring` consecutive keyframes, plus one keyframe's: what A needs at least"""
    most = max(len(set().union(*[set(dr.meas[kk]) for kk in range(max(0, k - ring + 1), k + 1)])) for k in range(dr.n_push))
    return most + max(len(m) for m in dr.meas)


# ---- CPU --------------------------------------------------------------------------------------------------------------------------
def test_reclaim_struct_sizes_match_header(tmp_path):
    """sizeof() of the reclaim structs as the C compiler sees them == size of the ctypes mirrors"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu\\n",sizeof(kba_reclaim_request),'
                    'sizeof(kba_reclaim_out));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(T.KbaReclaimRequest), C.sizeof(T.KbaReclaimOut)]


def test_reclaim_null_arguments_need_no_device():
    """a null track, group, request or output is KBA_ERR_BAD_ARG before any device work"""
    _build()
    from limo_b200 import capi
    L = capi.lib()
    q, o = capi.KbaReclaimRequest(), capi.KbaReclaimOut()
    for fn in (L.kba_track_reclaim_landmarks, L.kba_track_group_reclaim_landmarks):
        assert fn(None, C.byref(q), C.byref(o)) == 1
        assert "null argument" in L.kba_last_error().decode()


def _walk(dr, book, reclaim, on_step=None):
    """the ring slot policy of the twin tracks over drive dr: keyframe k in slot k % ring, the keyframe ring pushes older dropped.
    book assigns the landmark slots; on_step(k, slots of k's arena, evicted landmarks that got a slot again) after each push."""
    for k in range(dr.n_push):
        ids = sorted(dr.meas[k])
        slots, back = book.assign(ids, lambda lo, hi: reclaim(k, lo, hi))
        if on_step:
            on_step(k, slots, back)


def test_statement_drives_the_slot_bookkeeping():
    """the statement as the reclaim of a caller with ~1.3x the live landmarks in slots: every landmark of a live keyframe keeps
    one slot of its own, no slot is free while a live keyframe names it, the caller reclaims five times or more, landmarks are
    re-measured after their eviction, and slot order is not id order"""
    dr = ReclaimDrive(5)
    ring = dr.window + 2
    book = SlotBook(int(1.3 * _live_cap(dr, ring)))
    assert book.cap < dr.n_lm // 3
    arenas = {}                                   # keyframe -> its landmark ids (arena order, one entry per landmark)

    def reclaim(k, lo, hi):
        live = [np.array([book.slot[i] for i in arenas[kk]]) for kk in range(max(0, k - ring + 1), k)]
        s = free_slots(live, lo, hi)
        return s, np.zeros((len(s), 3)), np.ones(len(s))

    unordered = 0

    def step(k, slots, back):
        nonlocal unordered
        arenas[k] = sorted(dr.meas[k])
        unordered += bool(np.any(np.diff(slots) < 0))
        live = set().union(*[set(arenas[kk]) for kk in range(max(0, k - ring + 1), k + 1)])
        taken = [book.slot[i] for i in live]
        assert len(set(taken)) == len(taken) and max(taken) < book.cap
    _walk(dr, book, reclaim, step)
    assert book.reclaims >= 5 and len(book.restored & dr.revisited) > 0 and unordered > 0


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
def _tracks(h, dr, caps):
    from limo_b200 import capi
    n_meas = sum(len(o) for m in dr.meas for o in m.values())
    return [capi.Track(h, dr.cam_intr, dr.cam_pose, max_keyframes=dr.window + 2, max_landmarks=c, max_measurements=n_meas,
                       win_keyframes=dr.window, win_landmarks=4096, win_observations=1 << 15) for c in caps]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _same(a, b, what):
    assert np.array_equal(_bits(np.asarray(a)), _bits(np.asarray(b))), what


def _opt():
    from limo_b200 import capi
    o = capi.default_options()
    o.solver_time_sec = 1e3  # no time-outs: the two solves run to the same end
    return o


def _check_free(t, hi, live, written, what):
    """t's free slots of [0, hi) equal the statement over its live arenas, the evicted values what was last written there"""
    slots, pos, weight = t.reclaim_landmarks(0, hi, evict=True)
    assert np.array_equal(slots, free_slots(live, 0, hi)), what
    for s, p, w in zip(slots, pos, weight):
        if s in written:
            _same(p, written[s][0], what)
            _same(w, written[s][1], what)
    h2d, d2h, _ = t.transfer_bytes()
    assert (h2d, d2h) == (4 * len(live), 4 + 36 * hi), what


@pytest.mark.gpu
def test_twin_tracks_equal_in_every_call():
    from limo_b200 import capi
    dr = ReclaimDrive(5)
    W, ring = dr.window, dr.window + 2
    h = capi.Handle(0)
    book = SlotBook(int(1.3 * _live_cap(dr, ring)))
    A, B = _tracks(h, dr, [book.cap, dr.n_lm])
    opt = _opt()
    written = {}                                   # A's slot -> (pos, weight) last written to it
    written_b = {}
    created, pos_of = set(), {}
    arena_a, arena_b = {}, {}                      # keyframe slot -> landmark slots of its entries
    device_reclaims = [0]

    def reclaim(k, lo, hi):
        device_reclaims[0] += 1
        return A.reclaim_landmarks(lo, hi, evict=True)

    unordered = 0
    for k in range(dr.n_push):
        ks = k % ring
        if k >= ring:
            for t in (A, B):
                t.drop_keyframe(ks)
            arena_a.pop(ks), arena_b.pop(ks)
            _check_free(A, len(book.owner), list(arena_a.values()), written, "drop %d" % k)
            _check_free(B, dr.n_lm, list(arena_b.values()), written_b, "drop %d" % k)
        ids = sorted(dr.meas[k])
        slots, back = book.assign(ids, lambda lo, hi: reclaim(k, lo, hi))
        unordered += bool(np.any(np.diff(slots) < 0))
        sa = dict(zip(ids, slots))
        lm, cam, u, v, d = dr.arena(k)
        lma = np.array([sa[i] for i in lm], np.int32)
        A.push_keyframe(ks, dr.kf_pose[k], lma, u, v, d, cam=cam)
        B.push_keyframe(ks, dr.kf_pose[k], lm, u, v, d, cam=cam)
        arena_a[ks], arena_b[ks] = lma, lm
        for lid, s, p, w in back:              # re-measured after its eviction: restored from what the reclaim returned
            A.set_landmarks([s], pos=p.reshape(1, 3), weight=[w])
            written[s] = (p.copy(), np.float64(w))
        _check_free(A, len(book.owner), list(arena_a.values()), written, "push %d" % k)
        _check_free(B, dr.n_lm, list(arena_b.values()), written_b, "push %d" % k)

        active = list(range(max(0, k - W + 1), k + 1))
        kfs = [a % ring for a in active]
        slot_a = lambda ids_: np.array([book.slot[i] for i in ids_], np.int32)  # noqa: E731
        new = [i for i in ids if i not in created]
        pa, fa = A.create_landmarks(kfs, len(active) - 1, slot_a(new))
        pb, fb = B.create_landmarks(kfs, len(active) - 1, new)
        _same(pa, pb, "create %d" % k); _same(fa, fb, "create %d" % k)
        for j, i in enumerate(new):
            if fa[j] & 1:
                created.add(i); pos_of[i] = pb[j].copy()
                written[book.slot[i]] = (pa[j].copy(), np.float64(1.0)); written_b[i] = (pb[j].copy(), np.float64(1.0))
        if k < 2:
            continue
        act = sorted(set().union(*[set(dr.meas[a]) for a in active]) & created)
        out_a = A.deactivate_keyframes(kfs, slot_a(act), 3, 4, W)
        out_b = B.deactivate_keyframes(kfs, act, 3, 4, W)
        for x, y in zip(out_a, out_b):
            _same(x, y, "deactivate %d" % k)
        elig = [i for i in act if i % 3 != 1]
        for x, y in zip(A.depth_costs(kfs, slot_a(elig)), B.depth_costs(kfs, elig)):
            _same(x, y, "depth costs %d" % k)
        sel_a, sel_b = A.select_landmarks(kfs, slot_a(act)), B.select_landmarks(kfs, act)
        for key in sel_b:
            _same(sel_a[key], sel_b[key], "select %s %d" % (key, k))
        chosen = [i for c, i in enumerate(act) if sel_b["cheiral"][c] and sel_b["bin"][c] >= 0 and np.all(np.isfinite(pos_of[i]))]
        chosen = chosen[:4096]
        if not chosen:
            continue
        fixed = [1 if j < 2 else 0 for j in range(len(kfs))]
        ra = A.solve(kfs, fixed, slot_a(chosen), opt=opt)
        rb = B.solve(kfs, fixed, chosen, opt=opt)
        assert ra.c.status == rb.c.status == 0, k
        for x, y in ((ra.kf_pose, rb.kf_pose), (ra.kf_plane, rb.kf_plane), (ra.lm_pos[:len(chosen)], rb.lm_pos[:len(chosen)])):
            _same(x, y, "solve %d" % k)
        for j, i in enumerate(chosen):
            pos_of[i] = rb.lm_pos[j].copy()
            written[book.slot[i]] = (ra.lm_pos[j].copy(), written[book.slot[i]][1])
            written_b[i] = (rb.lm_pos[j].copy(), written_b[i][1])
        if k + 1 < dr.n_push:
            nxt = dr.meas[k + 1]
            sel = set(chosen)
            rows = [(i, c, uu, vv, dd) for i in sorted(nxt) if i in sel for c, uu, vv, dd in nxt[i]]
            if rows:
                li, ci, ui, vi, di = (np.array(x) for x in zip(*rows))
                fa_ = A.adjust_pose(dr.kf_pose[k + 1], slot_a(li), ui, vi, di, cam=ci, opt=opt)
                fb_ = B.adjust_pose(dr.kf_pose[k + 1], li, ui, vi, di, cam=ci, opt=opt)
                assert fa_.c.status == fb_.c.status and fa_.c.num_solves == fb_.c.num_solves, k
                _same(fa_.kf_pose, fb_.kf_pose, "adjust_pose %d" % k)
            rows = [(i, c, uu, vv) for i in sorted(nxt) if i in book.slot for c, uu, vv, _ in nxt[i]]
            if not rows:
                continue
            li, ci, ui, vi = (np.array(x) for x in zip(*rows))
            wa = A.frame_flow(ks, slot_a(li), ui, vi, cam=ci)
            wb = B.frame_flow(ks, li, ui, vi, cam=ci)
            for key in wb:
                _same(wa[key], wb[key], "frame_flow %s %d" % (key, k))
    assert device_reclaims[0] == book.reclaims >= 5, book.reclaims
    assert len(book.restored & dr.revisited) > 0 and unordered > 0
    for t in (A, B):
        t.close()
    h.close()


@pytest.mark.gpu
def test_group_equals_single_calls():
    """a group of three tracks (one sitting out at each call) equals the single calls on the same stores -- the call does not
    write the store -- with and without the eviction outputs; the transfer counts follow the header; a group of one too"""
    from limo_b200 import capi
    h = capi.Handle(0)
    drives = [ReclaimDrive(11, n_push=30, window=6), ReclaimDrive(12, n_push=24, window=8, rig=False, new_per_push=30),
              ReclaimDrive(13, n_push=20, window=5, new_per_push=20)]
    tracks = [_tracks(h, dr, [dr.n_lm])[0] for dr in drives]
    g, one = capi.TrackGroup(h, tracks), capi.TrackGroup(h, tracks[:1])
    for k in range(max(dr.n_push for dr in drives)):
        reqs = []
        for i, (t, dr) in enumerate(zip(tracks, drives)):
            ring = dr.window + 2
            if k < dr.n_push:
                if k >= ring:
                    t.drop_keyframe(k % ring)
                lm, cam, u, v, d = dr.arena(k)
                t.push_keyframe(k % ring, dr.kf_pose[k], lm, u, v, d, cam=cam)
                t.set_landmarks(np.unique(lm), pos=np.random.default_rng(k).normal(size=(len(np.unique(lm)), 3)),
                                weight=np.full(len(np.unique(lm)), 0.5 + i))
            sit = (k + i) % 3 == 2
            lo = (7 * k) % 50
            reqs.append(None if sit else dict(lo=lo, hi=min(dr.n_lm, lo + 40 * (k + 1)), evict=bool((k + i) % 2)))
        res = g.reclaim_landmarks(reqs)
        h2d, d2h = g.transfer_bytes()
        act = [i for i, r in enumerate(reqs) if r is not None]
        for i in range(3):
            if i not in act:
                assert res[i] is None
                continue
            single = tracks[i].reclaim_landmarks(**reqs[i])
            for x, y in zip(res[i] if reqs[i]["evict"] else [res[i]], single if reqs[i]["evict"] else [single]):
                _same(x, y, "group %d track %d" % (k, i))
        if act:
            n = {i: reqs[i]["hi"] - reqs[i]["lo"] for i in act}
            assert d2h == sum(4 + 4 * n[i] + (32 * n[i] if reqs[i]["evict"] else 0) for i in act)
            live = {i: min(k + 1, drives[i].window + 2, drives[i].n_push) for i in act}
            R = h2d - 4 * sum(live.values())
            assert (R == 0) if len(act) == 1 else (R > 0 and R % (len(act) - 1) == 0)
        if reqs[0] is not None:
            _same(one.reclaim_landmarks(reqs[:1])[0][0] if reqs[0]["evict"] else one.reclaim_landmarks(reqs[:1])[0],
                  res[0][0] if reqs[0]["evict"] else res[0], "group of one %d" % k)
    assert g.reclaim_landmarks([None] * 3) == [None] * 3 and g.transfer_bytes() == (0, 0)
    for x in (g, one, *tracks):
        x.close()
    h.close()


@pytest.mark.gpu
def test_reclaim_errors_write_nothing():
    """a range outside [0, max_landmarks], hi < lo and a null free_slot are KBA_ERR_BAD_ARG before anything is written: the
    sentinel outputs stay; a group names the failing track; an empty range is n_free = 0 alone and sits a group's track out"""
    from limo_b200 import capi
    L = capi.lib()
    dr = ReclaimDrive(21, n_push=6, window=4)
    h = capi.Handle(0)
    tracks = [_tracks(h, dr, [dr.n_lm])[0] for _ in range(2)]
    for t in tracks:
        for k in range(dr.n_push):
            lm, cam, u, v, d = dr.arena(k)
            t.push_keyframe(k, dr.kf_pose[k], lm, u, v, d, cam=cam)
    g = capi.TrackGroup(h, tracks)
    n = dr.n_lm
    slot = np.full(n + 8, -7, np.int32)
    ip = slot.ctypes.data_as(capi.c_int32_p)
    bad = [(-1, 5, ip), (0, n + 1, ip), (9, 3, ip), (0, 10, C.cast(None, capi.c_int32_p))]
    for lo, hi, p in bad:
        q, o = capi.KbaReclaimRequest(lo, hi), capi.KbaReclaimOut(n_free=-3, free_slot=p)
        assert L.kba_track_reclaim_landmarks(tracks[0]._p, C.byref(q), C.byref(o)) == 1
        assert o.n_free == -3 and np.all(slot == -7)
        qs = (capi.KbaReclaimRequest * 2)(capi.KbaReclaimRequest(0, 10), q)
        os_ = (capi.KbaReclaimOut * 2)(capi.KbaReclaimOut(n_free=-3, free_slot=ip), capi.KbaReclaimOut(n_free=-3, free_slot=p))
        assert L.kba_track_group_reclaim_landmarks(g._p, qs, os_) == 1
        assert "track 1" in L.kba_last_error().decode()
        assert os_[0].n_free == -3 and os_[1].n_free == -3 and np.all(slot == -7)
    assert len(tracks[0].reclaim_landmarks(5, 5)) == 0 and tracks[0].transfer_bytes()[:2] == (0, 0)
    res = g.reclaim_landmarks([dict(lo=3, hi=3), dict(lo=0, hi=n)])
    assert len(res[0]) == 0 and np.array_equal(res[1], tracks[1].reclaim_landmarks(0, n))
    # every landmark of the drive is measured by a live keyframe; slots beyond them are free
    assert len(tracks[0].reclaim_landmarks(0, n)) == n - len(set().union(*[set(m) for m in dr.meas]))
    for x in (g, *tracks):
        x.close()
    h.close()
