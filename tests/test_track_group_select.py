"""Landmark selection for every track of a group in one launch sequence (kba_track_group_select_landmarks).

Each request of a group call must give exactly what kba_track_select_landmarks gives for the same request on its own track --
the integers equal, the flows bit for bit, NaN in the same places -- and both must equal the restatement of the facade's host
code in tests/test_track_select.py.  The groups mix rigs, landmark counts, keyframe lists and selection parameters, sit tracks
out, fail on one bad request, and select again after a group solve has moved the stores."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.test_track_select import F32, PARAMS, Scene, _candidates, _check, host_select

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _transfer(reqs, record):
    """the header's transfer formula over the requests that do not sit out, with `record` bytes per argument record: (h2d, d2h)"""
    act = [r for r in reqs if r is not None]
    if not act:
        return 0, 0
    h2d = sum(4 * (len(r["kf_slots"]) + len(r["lm_slots"])) for r in act) + record * (len(act) - 1)
    d2h = sum(18 * len(r["lm_slots"]) for r in act) + 16 * len(act)
    return h2d, d2h


def _record_bytes(grp, reqs):
    """the size of one window's argument record, from the upload of a call with every request active (the header leaves it
    to the library build); the other calls of a test must then follow the formula with it"""
    grp.select_landmarks(reqs)
    h2d, _ = grp.transfer_bytes()
    extra = h2d - _transfer(reqs, 0)[0]
    assert len(reqs) > 1 and extra > 0 and extra % (len(reqs) - 1) == 0, extra
    return extra // (len(reqs) - 1)


def _equal(a, b, what):
    for key in ("cheiral", "bin", "near_order", "seen"):
        assert np.array_equal(a[key], b[key]), (what, key)
    assert np.array_equal(a["flow"].view(np.int64), b["flow"].view(np.int64)), (what, "flow bit patterns")


SENTINEL = dict(cheiral=0xAB, bin=-77, near_order=-7, flow=1234.5, seen=-3)


def _raw_select(grp, reqs, n_out):
    """kba_track_group_select_landmarks through ctypes, every output array pre-filled with a sentinel (n_out[i] entries; n_near
    -9); a request may set n_kf apart from its list.  Returns the return code and the arrays."""
    from limo_b200 import capi
    from limo_b200.capi_types import KbaSelectOut, KbaSelectParams, KbaSelectRequest, c_double_p, c_int32_p
    n = len(reqs)
    creq, cout = (KbaSelectRequest * n)(), (KbaSelectOut * n)()
    keep, outs = [], []
    for i, r in enumerate(reqs):
        m = n_out[i]
        o = dict(cheiral=np.full(m, SENTINEL["cheiral"], np.uint8), bin=np.full(m, SENTINEL["bin"], np.int8),
                 near_order=np.full(m, SENTINEL["near_order"], np.int32), flow=np.full(m, SENTINEL["flow"]),
                 seen=np.full(m, SENTINEL["seen"], np.int32), n_near=np.full(1, -9, np.int32))
        c = cout[i]
        c.cheiral, c.bin = o["cheiral"].ctypes.data_as(C.POINTER(C.c_uint8)), o["bin"].ctypes.data_as(C.POINTER(C.c_int8))
        c.near_order, c.n_near = o["near_order"].ctypes.data_as(c_int32_p), o["n_near"].ctypes.data_as(c_int32_p)
        c.flow, c.seen = o["flow"].ctypes.data_as(c_double_p), o["seen"].ctypes.data_as(c_int32_p)
        outs.append(o)
        if r is None:
            continue
        kf = np.ascontiguousarray(r["kf_slots"], np.int32)
        lm = np.ascontiguousarray(r["lm_slots"], np.int32)
        prm = dict(capi.SELECT_DEFAULTS, **{k: v for k, v in r.items() if k not in ("kf_slots", "lm_slots", "n_kf")})
        p = KbaSelectParams((C.c_double * 3)(*prm["voxel_size"]), prm["roi_far"], prm["roi_middle"])
        q = creq[i]
        q.n_kf, q.n_cand = r.get("n_kf", len(kf)), len(lm)
        q.kf_slot, q.lm_slot, q.params = kf.ctypes.data_as(c_int32_p), lm.ctypes.data_as(c_int32_p), C.pointer(p)
        keep.append((kf, lm, p))
    rc = capi.lib().kba_track_group_select_landmarks(grp._p, creq, cout)
    return rc, outs


def _untouched(o, what):
    for key, v in SENTINEL.items():
        assert (o[key] == v).all(), (what, key)


# three tracks of different scenes: two-camera and mono rigs, 600 and 4000 landmarks, different keyframe lists and parameters
MIXED = [dict(seed=11, n_kf=8, n_lm=600, rig=True, kf=list(range(1, 8)), params=PARAMS[0]),
         dict(seed=12, n_kf=10, n_lm=600, rig=False, kf=[0, 2, 3, 5, 6, 7, 9], params=PARAMS[1]),
         dict(seed=13, n_kf=8, n_lm=4000, rig=True, kf=list(range(0, 6)), params=dict(voxel_size=(1.0, 1.0, 0.5), roi_far=50.0,
                                                                                      roi_middle=25.0))]


def _mixed(h):
    scenes, tracks, reqs = [], [], []
    for m in MIXED:
        sc = Scene(m["seed"], n_kf=m["n_kf"], n_lm=m["n_lm"], rig=m["rig"])
        scenes.append(sc)
        tracks.append(sc.make_track(h))
        reqs.append(dict(kf_slots=m["kf"], lm_slots=sc.slot[_candidates(sc, m["kf"])], **m["params"]))
    return scenes, tracks, reqs


@pytest.mark.gpu
def test_mixed_group_equals_single_calls_and_host():
    from limo_b200 import capi
    h = capi.Handle(0)
    scenes, tracks, reqs = _mixed(h)
    grp = capi.TrackGroup(h, tracks)
    out = grp.select_landmarks(reqs)
    record = _record_bytes(grp, reqs)
    assert grp.transfer_bytes() == _transfer(reqs, record)
    grp.select_landmarks(reqs[:2] + [None])
    assert grp.transfer_bytes() == _transfer(reqs[:2] + [None], record)
    behind = 0
    for i, (sc, t, r, m) in enumerate(zip(scenes, tracks, reqs, MIXED)):
        single = t.select_landmarks(**r)
        _equal(out[i], single, "track %d against its single call" % i)
        ref = host_select(sc, m["kf"], _candidates(sc, m["kf"]), r["voxel_size"], r["roi_far"], r["roi_middle"])
        _check(out[i], ref)
        assert len(ref["near_order"]) > 0 and (ref["bin"] == 1).any() and (ref["bin"] == 2).any()
        behind += int((ref["cheiral"] == 0).sum())
    assert behind > 0
    # the single calls in between leave the scratch as the group expects it: the same group call again, the same results
    again = grp.select_landmarks(reqs)
    for i in range(len(tracks)):
        _equal(again[i], out[i], "track %d, second group call" % i)
    grp.close()
    for t in tracks:
        t.close()
    h.close()


@pytest.mark.gpu
def test_group_of_one_equals_single_call():
    from limo_b200 import capi
    h = capi.Handle(0)
    sc = Scene(21, n_lm=600, rig=True)
    t = sc.make_track(h)
    grp = capi.TrackGroup(h, [t])
    kf = list(range(1, sc.n_kf))
    for p in PARAMS:
        r = dict(kf_slots=kf, lm_slots=sc.slot[_candidates(sc, kf)], **p)
        g = grp.select_landmarks([r])[0]
        s = t.select_landmarks(**r)
        _equal(g, s, str(p))
        assert grp.transfer_bytes() == t.transfer_bytes()[:2] == _transfer([r], 0)
    grp.close(); t.close(); h.close()


@pytest.mark.gpu
def test_sitting_out():
    """sit-out entries among active ones: their arrays keep the sentinels and n_near is 0; the active ones are exact; a later
    single call on a track that sat out is unaffected; a call in which everyone sits out moves nothing"""
    from limo_b200 import capi
    h = capi.Handle(0)
    scenes, tracks, reqs = _mixed(h)
    grp = capi.TrackGroup(h, tracks)
    n_out = [len(r["lm_slots"]) for r in reqs]
    record = _record_bytes(grp, reqs)
    for sit in ([1], [0, 2], [0, 1, 2]):
        rs = [None if i in sit else r for i, r in enumerate(reqs)]
        rc, outs = _raw_select(grp, rs, n_out)
        assert rc == 0, capi.lib().kba_last_error().decode()
        assert grp.transfer_bytes() == _transfer(rs, record)
        for i, (sc, m) in enumerate(zip(scenes, MIXED)):
            if i in sit:
                _untouched(outs[i], "track %d sat out" % i)
                assert outs[i]["n_near"][0] == 0
            else:
                cand = _candidates(sc, m["kf"])
                ref = host_select(sc, m["kf"], cand, reqs[i]["voxel_size"], reqs[i]["roi_far"], reqs[i]["roi_middle"])
                o = dict(outs[i], near_order=outs[i]["near_order"][:outs[i]["n_near"][0]])
                _check(o, ref)
        py = grp.select_landmarks(rs)
        assert [x is None for x in py] == [i in sit for i in range(3)]
    for i, (sc, t, m) in enumerate(zip(scenes, tracks, MIXED)):
        ref = host_select(sc, m["kf"], _candidates(sc, m["kf"]), reqs[i]["voxel_size"], reqs[i]["roi_far"], reqs[i]["roi_middle"])
        _check(t.select_landmarks(**reqs[i]), ref)
    grp.close()
    for t in tracks:
        t.close()
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pos", [0, 1, 2])
def test_bad_request_names_its_track(pos):
    """one bad request in position pos: the call fails with that request's code and names track pos, and no output of any track
    is written"""
    from limo_b200 import capi
    h = capi.Handle(0)
    scenes, tracks, reqs = _mixed(h)
    grp = capi.TrackGroup(h, tracks)
    sc = scenes[pos]
    lm = reqs[pos]["lm_slots"]
    bad = [(dict(kf_slots=[1, 1, 2]), "keyframe slot listed twice", 1),
           (dict(lm_slots=np.r_[lm[:5], lm[:1]]), "landmark slot listed twice", 1),
           (dict(kf_slots=[1, 2, sc.n_kf]), "not pushed", 1),                        # a slot of the track that was never pushed
           (dict(voxel_size=(0.5, 0.0, 0.3)), "voxel", 1),
           (dict(lm_slots=np.arange(len(sc.lm_pos) + 1, dtype=np.int32)), "more keyframes or candidates", 4),
           (dict(n_kf=-1), "no keyframes", 1)]                                       # n_kf < 0 is bad, not a sit-out
    for change, msg, code in bad:  # codes: KBA_ERR_BAD_ARG = 1, KBA_ERR_CAPACITY = 4
        rs = list(reqs)
        rs[pos] = dict(reqs[pos], **change)
        n_out = [len(r["lm_slots"]) for r in rs]
        rc, outs = _raw_select(grp, rs, n_out)
        err = capi.lib().kba_last_error().decode()
        assert rc == code, (msg, rc, err)
        assert ("track %d: " % pos) in err and msg in err, err
        for i in range(3):
            _untouched(outs[i], "%s: track %d" % (msg, i))
            assert outs[i]["n_near"][0] == -9
        if "n_kf" not in change:
            with pytest.raises(capi.KbaError, match="track %d: .*%s" % (pos, msg)):
                grp.select_landmarks(rs)
    # the group is usable after the failures
    out = grp.select_landmarks(reqs)
    for i, (s, m) in enumerate(zip(scenes, MIXED)):
        _check(out[i], host_select(s, m["kf"], _candidates(s, m["kf"]), reqs[i]["voxel_size"], reqs[i]["roi_far"],
                                   reqs[i]["roi_middle"]))
    grp.close()
    for t in tracks:
        t.close()
    h.close()


@pytest.mark.gpu
def test_binding_rejects_requests_the_library_would_read_otherwise():
    """a dict request with no keyframes is an error, as for Track.select_landmarks (n_kf = 0 would make the track sit out), and
    a voxel_size that is not 3 long cannot shift the parameters of the other requests"""
    from limo_b200 import capi
    h = capi.Handle(0)
    scenes, tracks, reqs = _mixed(h)
    grp = capi.TrackGroup(h, tracks)
    with pytest.raises(capi.KbaError, match="no keyframes"):
        tracks[1].select_landmarks(**dict(reqs[1], kf_slots=[]))
    with pytest.raises(capi.KbaError, match="track 1: no keyframes"):
        grp.select_landmarks([reqs[0], dict(reqs[1], kf_slots=[]), reqs[2]])
    with pytest.raises(ValueError, match="request 2: voxel_size"):
        grp.select_landmarks([reqs[0], reqs[1], dict(reqs[2], voxel_size=(0.5, 0.5))])
    out = grp.select_landmarks(reqs)
    for i, (sc, m) in enumerate(zip(scenes, MIXED)):
        _check(out[i], host_select(sc, m["kf"], _candidates(sc, m["kf"]), reqs[i]["voxel_size"], reqs[i]["roi_far"],
                                   reqs[i]["roi_middle"]))
    grp.close()
    for t in tracks:
        t.close()
    h.close()


class _DriveScene:
    """host_select's view of a synthetic mono drive of tests/test_track_group.py after step 0 (keyframe k in slot k, landmark
    id = slot), with the poses and positions of its track's store"""

    def __init__(self, dr):
        self.kf_pose = [np.array(p) for p in dr.win.kf_pose[:dr.W]]
        self.cam_pose = [np.array(p) for p in dr.cam_pose]
        self.lm_pos = [list(map(float, p)) for p in dr.win.lm_pos]
        self.meas = []
        for k in range(dr.W):
            lm, u, v, _, cam = dr.measurements(k)
            d = {}
            for j, c, uu, vv in zip(lm, cam, u, v):
                d.setdefault(int(j), []).append((int(c), F32(uu), F32(vv)))
            self.meas.append(d)


@pytest.mark.gpu
def test_selection_reads_the_store_after_a_group_solve():
    """group selection, a group solve that moves poses and landmarks, group selection again: the second equals host_select on
    the solved state"""
    from limo_b200 import capi
    from tests.test_track_group import _Drive
    h = capi.Handle(0)
    drives = [_Drive(seed=91, W=6, n_lm=500, n_obs=4000), _Drive(seed=92, W=8, n_lm=700, n_obs=6000)]
    tracks = [dr.make_track(h) for dr in drives]
    scenes = [_DriveScene(dr) for dr in drives]
    grp = capi.TrackGroup(h, tracks)
    prm = [dict(voxel_size=(0.5, 0.5, 0.3), roi_far=40.0, roi_middle=15.0), dict(voxel_size=(2.0, 2.0, 1.0), roi_far=30.0, roi_middle=8.0)]
    kfs = [list(range(dr.W)) for dr in drives]
    cands = [_candidates(sc, kf) for sc, kf in zip(scenes, kfs)]
    sel = [dict(kf_slots=kf, lm_slots=np.array(c, np.int32), **p) for kf, c, p in zip(kfs, cands, prm)]
    before = grp.select_landmarks(sel)
    for sc, kf, c, p, o in zip(scenes, kfs, cands, prm, before):
        _check(o, host_select(sc, kf, c, p["voxel_size"], p["roi_far"], p["roi_middle"]))
    reqs = [dr.request(0) for dr in drives]
    res = grp.solve(reqs)
    for sc, dr, r, q in zip(scenes, drives, res, reqs):
        assert r.c.status == 0
        lm = np.asarray(q["lm_slots"])
        assert not np.array_equal(r.kf_pose, dr.win.kf_pose[:dr.W]) and not np.array_equal(r.lm_pos[:len(lm)], dr.win.lm_pos[lm])
        sc.kf_pose = [np.array(p) for p in r.kf_pose]
        for j, pos in zip(lm, r.lm_pos[:len(lm)]):
            sc.lm_pos[int(j)] = list(map(float, pos))
    after = grp.select_landmarks(sel)
    changed = 0
    for sc, kf, c, p, o, b in zip(scenes, kfs, cands, prm, after, before):
        _check(o, host_select(sc, kf, c, p["voxel_size"], p["roi_far"], p["roi_middle"]))
        changed += int((o["bin"] != b["bin"]).sum() + (o["cheiral"] != b["cheiral"]).sum())
    print("selection quantities changed by the solve: %d" % changed)
    grp.close()
    for t in tracks:
        t.close()
    h.close()


def test_select_request_struct_sizes_match_header(tmp_path):
    """sizeof(kba_select_request) and sizeof(kba_select_out) as the C compiler sees them == sizes of the ctypes mirrors"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu\\n",'
                    'sizeof(kba_select_request),sizeof(kba_select_out));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(T.KbaSelectRequest), C.sizeof(T.KbaSelectOut)]

