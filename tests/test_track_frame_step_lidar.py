"""limo's mono-lidar frame step as one store call -- kba_track_frame_step_lidar and its group forms -- against the chain it
replaces: kba_lidar_depth_batch with one view per measured camera, then kba_track_frame_step on those depths.  Two copies of
each store go through the closed-loop drives of tests/keyframe_drive.py with a lidar cloud per frame; after every frame the
outputs, the depths and the snapshots of the two stores must be equal byte for byte.  The struct layout, the exports and the
binding's request builder are checked without a GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from limo_b200 import capi, synth
from limo_b200 import geometry as g
from limo_b200.capi_types import KbaFrameLidar, KbaLidarOptions
from tests.keyframe_drive import KeyframeDrive
from tests.test_track_frame_step import DRIVES, Loop, _options, _same_step, _track

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KBA_ERR_BAD_ARG, KBA_ERR_CAPACITY = 1, 4


# ---- without a GPU ------------------------------------------------------------------------------------------------------
def test_struct_layout_matches_header(tmp_path):
    fields = [f for f, _ in KbaFrameLidar._fields_]
    prog = tmp_path / "lay.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "kba_b200.h"\nint main(){printf("%zu", sizeof(kba_frame_lidar));' +
                    "".join('printf(" %%zu", offsetof(kba_frame_lidar, %s));' % f for f in fields) + 'return 0;}\n')
    exe = tmp_path / "lay"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(KbaFrameLidar)] + [getattr(KbaFrameLidar, f).offset for f in fields]


def test_the_three_symbols_are_exported():
    L = C.CDLL(capi.LIB_PATH)
    for name in ("kba_track_frame_step_lidar", "kba_track_group_frame_step_lidar", "kba_track_group_frame_step_lidar_opts"):
        assert hasattr(L, name) and name in capi.SYMBOLS, name


class _Stub:
    """capi.lib(): every C function records its name and the lidar form's arguments decoded during the call, and succeeds"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            if "frame_step" in name:  # (handle, req, [lid,] opt, out, res)
                lid = args[2] if "lidar" in name else None
                self.calls.append((name, self._decode(args[1], lid, args[-3], len(args[-1]))))
            return 0
        fn.__name__ = name
        return fn

    @staticmethod
    def _decode(req, lid, opt, n):
        out = []
        for i in range(n):
            q = req[i]
            if q.n_kf == 0:
                out.append(None)
                continue
            m = q.n_meas
            rec = dict(u=C.string_at(q.u, 4 * m), d_null=not q.d)
            if lid is not None:
                l = lid[i]
                n_cam = 2 if q.cam else 1
                rec.update(points=C.string_at(l.points, 4 * l.n_points * l.stride), shape=(l.n_points, l.stride),
                           T=C.string_at(l.T_cam_lidar, 56 * n_cam), opts=[(l.opt[c].image_width, l.opt[c].rect_width) for c in range(n_cam)],
                           depth_out=bool(l.depth_out))
            out.append(rec)
        return out, opt


@pytest.fixture
def stub(monkeypatch):
    s = _Stub()
    monkeypatch.setattr(capi, "_lib", s)
    return s


def _fake_track(n_cam):
    t = capi.Track.__new__(capi.Track)
    t._p, t.n_cam = C.c_void_p(0x10), n_cam
    return t


def _fake_group(tracks):
    gr = capi.TrackGroup.__new__(capi.TrackGroup)
    gr._p, gr.tracks = C.c_void_p(0x20), tracks
    return gr


def _lopt(width, rect):
    o = KbaLidarOptions()
    o.image_width, o.rect_width = width, rect
    return o


def _small(rng, rig, **kw):
    r = dict(kf_slots=[0, 1], lm_slot=[3, 3, 5, 9], u=rng.random(4), v=rng.random(4), run_sel=[1, 0, 1], kf_new=2, new_slots=[9],
             pose7=[1.0, 0, 0, 0, 0, 0, 0], stamp=7_000, stamp_last=5_000, critical_quaternion_diff=0.03, time_difference_ns=400,
             cloud=rng.random((20, 4)).astype(np.float32), T_cam_lidar=rng.random((2 if rig else 1, 7)), depths=True)
    if rig:
        r["cam"] = [0, 1, 0, 1]
    r.update(kw)
    return r


def test_binding_passes_arrays_by_content(stub):
    rng = np.random.default_rng(3)
    one = _small(rng, False, lidar_opt=_lopt(640, 6.0))
    res = _fake_track(1).frame_step(**one)
    (name, (recs, _opt)), = stub.calls
    assert name == "kba_track_frame_step_lidar"
    rec, = recs
    assert rec["points"] == one["cloud"].tobytes() and rec["shape"] == (20, 4) and rec["d_null"] and rec["depth_out"]
    assert rec["T"] == np.asarray(one["T_cam_lidar"], np.float64).tobytes() and rec["opts"] == [(640, 6.0)]
    assert rec["u"] == np.asarray(one["u"], np.float32).tobytes() and res["depth"].shape == (4,)
    tr = [_fake_track(2), _fake_track(1), _fake_track(2)]
    reqs = [_small(rng, True, lidar_opt=[_lopt(1280, 6.0), _lopt(640, 10.0)]), None,
            _small(rng, True, lidar_opt=_lopt(320, 3.0), depths=False, cloud=np.zeros((0, 3), np.float32))]
    for opt, fn in ((None, "kba_track_group_frame_step_lidar"), ([None, None, None], "kba_track_group_frame_step_lidar_opts")):
        stub.calls.clear()
        outs = _fake_group(tr).frame_step(reqs, opt=opt)
        (name, (recs, _opt)), = stub.calls
        assert name == fn and recs[1] is None and outs[1] is None
        assert recs[0]["opts"] == [(1280, 6.0), (640, 10.0)] and recs[2]["opts"] == [(320, 3.0)] * 2
        assert recs[0]["points"] == reqs[0]["cloud"].tobytes() and recs[2]["shape"] == (0, 3) and recs[2]["points"] == b""
        assert recs[0]["depth_out"] and not recs[2]["depth_out"] and outs[2]["depth"] is None and outs[0]["depth"].shape == (4,)
    # without clouds the binding keeps the frame step's own symbols
    stub.calls.clear()
    plain = {k: v for k, v in _small(rng, False).items() if k not in ("cloud", "T_cam_lidar", "depths")}
    out = _fake_track(1).frame_step(**dict(plain, d=[1, 2, 3, 4]))
    assert [c[0] for c in stub.calls] == ["kba_track_frame_step"] and out["depth"] is None


def test_malformed_requests_fail_before_the_call(stub):
    rng = np.random.default_rng(4)
    t, gr = _fake_track(2), _fake_group([_fake_track(2), _fake_track(2)])
    bad = [(ValueError, "T_cam_lidar has 1 poses for 2 cameras", dict(T_cam_lidar=np.zeros(7))),
           (ValueError, "one 7-vector per camera", dict(T_cam_lidar=np.zeros(10))),
           (ValueError, "a cloud needs T_cam_lidar", dict(T_cam_lidar=None)),
           (ValueError, "3 lidar option sets for 2 cameras", dict(lidar_opt=[None] * 3)),
           (ValueError, "stride >= 3", dict(cloud=np.zeros((5, 2), np.float32))),
           (ValueError, "stride >= 3", dict(cloud=np.zeros(12, np.float32))),
           (ValueError, "d \\(the depths\\) or a lidar cloud", dict(d=[1, 2, 3, 4]))]
    for err, msg, kw in bad:
        with pytest.raises(err, match=msg):
            t.frame_step(**_small(rng, True, **kw))
        with pytest.raises(err, match="request 1: .*" + msg):
            gr.frame_step([_small(rng, True), _small(rng, True, **kw)])
    plain = {k: v for k, v in _small(rng, True).items() if k not in ("cloud", "T_cam_lidar", "depths")}
    with pytest.raises(ValueError, match="request 1: no cloud in a lidar call"):
        gr.frame_step([_small(rng, True), dict(plain, d=[1, 2, 3, 4])])
    with pytest.raises(ValueError, match="d \\(the depths\\) or a lidar cloud"):
        t.frame_step(**plain)
    assert stub.calls == []


# ---- on the device -----------------------------------------------------------------------------------------------------
def _wall(depth, tilt):
    """a plane in front of camera 0 (camera <- lidar is the identity for it): about a third of a drive's features land on it"""
    xs, ys = np.meshgrid(np.linspace(-8, 8, 500), np.linspace(-2.5, 2.5, 160))
    return np.stack([xs.ravel(), ys.ravel(), (depth + tilt * xs).ravel(), np.zeros(xs.size)], axis=1).astype(np.float32)


def _frame_cloud(seed, k, empty=False):
    """frame k's cloud: a small seeded scan and a wall, or no point at all"""
    if empty:
        return np.zeros((0, 4), np.float32)
    scan, *_ = synth.make_lidar_scene(seed=1000 * seed + k, n_azimuth=400, n_features=1)
    return np.ascontiguousarray(np.concatenate([scan, _wall(9.0 + k % 5, 0.1 * (k % 3))]))


def _rig_lidar(n_cam):
    """camera c <- lidar for every camera of a drive, and per-camera extraction options that differ"""
    T = [np.array([1.0, 0, 0, 0, 0, 0, 0]), g.iso_to_pose(g.iso(g.angle_axis(0.1, [0.0, 1.0, 0.0]), [0.3, 0.0, 0.0]))][:n_cam]
    o0, o1 = capi.lidar_default_options(), capi.lidar_default_options()
    o0.image_width, o0.image_height = 1280, 384
    o1.image_width, o1.image_height, o1.rect_width, o1.rect_height, o1.hist_bin_width = 1280, 384, 10.0, 12.0, 0.5
    return np.array(T), [o0, o1][:n_cam]


def _batch_depths(h, r, cloud, T, opts, intr):
    """the chain's depths: kba_lidar_depth_batch with one view per camera that measures something"""
    cam, u, v = np.asarray(r["cam"]), np.asarray(r["u"], np.float32), np.asarray(r["v"], np.float32)
    d = np.full(len(cam), -1.0, np.float32)
    views, vo, rows = [], [], []
    for c in range(len(T)):
        m = np.flatnonzero(cam == c)
        if len(m):
            views.append((0, T[c], intr[c], np.stack([u[m], v[m]], axis=1)))
            vo.append(opts[c])
            rows.append(m)
    if views:
        depths, _ = h.lidar_depth_batch([cloud], views, vo)
        for m, x in zip(rows, depths):
            d[m] = x
    return d


def _lidar_request(r, cloud, T, opts, depths=True):
    q = {k: x for k, x in r.items() if k != "d"}
    q.update(cloud=cloud, T_cam_lidar=T, lidar_opt=opts, depths=depths)
    return q


def _f32(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _selected_rows(r):
    lm = np.asarray(r["lm_slot"])
    if not len(lm):
        return np.zeros(0, bool)
    return np.asarray(r["run_sel"], bool)[np.cumsum(np.r_[True, lm[1:] != lm[:-1]]) - 1]


def _up_extra(r, cloud, n_cam):
    """what the lidar form uploads beyond the frame step's formula, but the view records (R_v each): 8 (V + 1) bytes of
    prefixes, the run flags' padding to 4 bytes, the cloud; and V"""
    cam = np.asarray(r["cam"])
    V = sum(int(np.any(cam == c)) for c in range(n_cam))
    return 8 * (V + 1) + (-len(r["run_sel"])) % 4 + (cloud.nbytes if len(cam) else 0), V


@pytest.mark.gpu
@pytest.mark.parametrize("kw", DRIVES, ids=lambda kw: "w%d_%s" % (kw["window"], "rig" if kw["rig"] else "mono"))
def test_lidar_frame_step_equals_the_chain(kw):
    dr = KeyframeDrive(**kw)
    h = capi.Handle(0)
    probe, rows = _track(h, dr, 1)
    probe.close()
    a, _ = _track(h, dr, (dr.window // 2 + 1) * rows + rows // 2)
    b = a.clone()
    loop = Loop(dr, kw["seed"], dr.n_lm + 1)
    loop.first([a, b])
    opt = _options()
    T, lo = _rig_lidar(len(dr.cam_intr))
    seen = dict(with_depth=0, without_depth=0, selected=0, rejected=0, adjusted_depth=0, created_by_lidar=0)
    per_view = set()
    for k in range(1, dr.n_frames):
        r, run_ids = loop.request(k)
        cloud = _frame_cloud(kw["seed"], k, empty=k % 9 == 4)
        d = _batch_depths(h, r, cloud, T, lo, dr.cam_intr)
        ref = a.frame_step(opt=opt, **dict(r, d=d))
        up0, down0, _ = a.transfer_bytes()
        one = b.frame_step(opt=opt, **_lidar_request(r, cloud, T, lo))
        up1, down1, _ = b.transfer_bytes()
        _same_step(one, ref, k)
        assert np.array_equal(_f32(one["depth"]), _f32(d)), k
        assert bytes(a.snapshot()) == bytes(b.snapshot()), k
        extra, V = _up_extra(r, cloud, len(T))
        assert down1 - down0 == 4 * len(d), k
        if V:
            per_view.add((up1 - up0 - extra) / V)
        else:
            assert up1 - up0 == extra, k
        seen["with_depth" if (d > 0).any() else "without_depth"] += 1
        seen["selected" if one["selected"] else "rejected"] += 1
        sel = _selected_rows(r)
        seen["adjusted_depth"] += one["result"].c.num_solves > 0 and bool((d[sel] > 0).any())
        if one["selected"]:
            lm = np.asarray(r["lm_slot"])
            for sl, f in zip(r["new_slots"], one["flags"]):
                seen["created_by_lidar"] += (f & 3) == 3 and bool((d[lm == sl] > 0).any())
        loop.advance([a, b], r, run_ids, one, k)
    assert all(x > 0 for x in seen.values()), seen
    R_v, = per_view  # one size of a view's parameter record for every call
    assert R_v > 0 and R_v % 8 == 0, R_v
    a.close(); b.close(); h.close()


def _without_cam(r, run_ids, c):
    """r without camera c's measurements: the runs, flags and new landmarks that remain"""
    lm, cam = np.asarray(r["lm_slot"]), np.asarray(r["cam"])
    keep = cam != c
    run_of = np.cumsum(np.r_[True, lm[1:] != lm[:-1]]) - 1
    runs = np.unique(run_of[keep])
    q = dict(r, lm_slot=lm[keep], cam=cam[keep], u=np.asarray(r["u"])[keep], v=np.asarray(r["v"])[keep], d=np.asarray(r["d"])[keep],
             run_sel=np.asarray(r["run_sel"], bool)[runs])
    left = set(lm[keep].tolist())
    q["new_slots"] = [s for s in r["new_slots"] if s in left]
    return q, np.asarray(run_ids)[runs]


@pytest.mark.gpu
def test_group_lidar_frame_step_equals_single_calls():
    """8 tracks, one sitting out per frame, per-camera options that differ, empty clouds, rig frames in which one camera
    measures nothing, frames with and without depths downloaded, the _opts form on every other frame: every output, depth
    and snapshot equals the single lidar call's on a clone"""
    h = capi.Handle(0)
    drs = [KeyframeDrive(70 + i, n_frames=30, window=6 + (i % 3), rig=bool(i % 2), n_feat=120 + 20 * i) for i in range(8)]
    gt, st, loops, lidar = [], [], [], []
    for i, dr in enumerate(drs):
        t, rows = _track(h, dr, 1)
        t.close()
        t, _ = _track(h, dr, (dr.window // 2 + 1) * rows + rows // 2)
        gt.append(t)
        st.append(t.clone())
        loops.append(Loop(dr, 110 + i, dr.n_lm + 1))
        loops[i].first([gt[i], st[i]])
        lidar.append(_rig_lidar(len(dr.cam_intr)))
    grp = capi.TrackGroup(h, gt)
    opts = [_options() for _ in drs]
    for i, o in enumerate(opts):
        o.reprojection_thres = 1.2 + 0.1 * i
    seen = dict(empty=0, one_camera=0, opts_form=0, single_form=0, depths_none=0, with_depth=0)
    for k in range(1, 30):
        reqs, ids = [], []
        for i, lp in enumerate(loops):
            r, run_ids = lp.request(k)
            if i == 1 and k % 4 == 0:  # a rig frame whose camera 1 measures nothing
                r, run_ids = _without_cam(r, run_ids, 1)
                seen["one_camera"] += 1
            empty = i == 2 and k % 2 == 0
            seen["empty"] += empty
            T, lo = lidar[i]
            reqs.append(None if i == k % 8 else _lidar_request(r, _frame_cloud(80 + i, k, empty), T, lo, depths=i % 3 != 0))
            ids.append(run_ids)
        per_track = k % 2 == 1
        seen["opts_form" if per_track else "single_form"] += 1
        outs = grp.frame_step(reqs, opt=opts if per_track else opts[0])
        assert outs[k % 8] is None
        for i, q in enumerate(reqs):
            if q is None:
                continue
            one = st[i].frame_step(opt=opts[i] if per_track else opts[0], **q)
            _same_step(outs[i], one, (k, i))
            if q["depths"]:
                assert np.array_equal(_f32(outs[i]["depth"]), _f32(one["depth"])), (k, i)
                seen["with_depth"] += bool((one["depth"] > 0).any())
                if i == 2 and k % 2 == 0:
                    assert (one["depth"] == -1).all()
            else:
                assert outs[i]["depth"] is None and one["depth"] is None
                seen["depths_none"] += 1
            assert bytes(gt[i].snapshot()) == bytes(st[i].snapshot()), (k, i)
            loops[i].advance([gt[i], st[i]], q, ids[i], one, k)
    assert all(x > 0 for x in seen.values()), seen
    grp.close()
    for t in gt + st:
        t.close()
    h.close()


def _huge_image():
    o = capi.lidar_default_options()
    o.image_width = o.image_height = 1 << 20  # (2^16)^2 cells: more than 32-bit indexing
    return o


@pytest.mark.gpu
def test_refusals_write_nothing():
    dr = KeyframeDrive(5, n_frames=12, window=6, rig=True)
    h = capi.Handle(0)
    t, rows = _track(h, dr, 1)
    t.close()
    t, _ = _track(h, dr, (dr.window // 2 + 1) * rows + rows // 2)
    u = t.clone()
    loop = Loop(dr, 5, dr.n_lm + 1)
    loop.first([t, u])
    ref = t.clone()  # takes only the good call
    grp = capi.TrackGroup(h, [t, u])
    T, lo = _rig_lidar(2)
    r, _ids = loop.request(1)
    good = _lidar_request(r, _frame_cloud(5, 1), T, lo)
    snap = bytes(t.snapshot())
    opt = _options()

    def field(name, value):
        return lambda lid, i: lid[name].__setitem__(i, value)

    cases = [(KBA_ERR_BAD_ARG, "T_cam_lidar", field("T_cam_lidar", 0), good),
             (KBA_ERR_BAD_ARG, "lidar options", field("opt", 0), good),
             (KBA_ERR_BAD_ARG, "null points", field("points", 0), good),
             (KBA_ERR_BAD_ARG, "negative n_points", field("n_points", -1), good),
             (KBA_ERR_BAD_ARG, "stride < 3", field("stride", 2), good),
             (KBA_ERR_BAD_ARG, "kf_new in use", None, dict(good, kf_new=r["kf_slots"][0])),
             (KBA_ERR_CAPACITY, "32-bit", None, dict(good, lidar_opt=[_huge_image(), lo[1]])),
             (KBA_ERR_BAD_ARG, "null argument", "no lid", good)]
    L = capi.lib()
    for code, msg, spoil, q in cases:
        for group in (False, True):
            fn = L.kba_track_group_frame_step_lidar if group else L.kba_track_frame_step_lidar
            req, out, ress, keep, _res, lid = capi._frame_step_records(fn, [good, q] if group else [q], 4, True)
            keep[8][0][:] = 7.5  # the depth buffer
            if callable(spoil):
                spoil(lid, len(lid) - 1)
            lp = None if spoil == "no lid" else lid.ctypes.data_as(C.POINTER(KbaFrameLidar))
            rc = fn(grp._p if group else t._p, req.ctypes.data_as(C.POINTER(capi.KbaFrameStepRequest)), lp, C.byref(opt),
                    out.ctypes.data_as(C.POINTER(capi.KbaFrameStepOut)), ress)
            err = L.kba_last_error().decode()
            assert rc == code and msg in err, (msg, group, rc, err)
            if group and spoil != "no lid":
                assert "track 1" in err, err
            assert (keep[8][0] == 7.5).all() and not out["n_matched"].any() and not out["angle"].any() and not keep[5].any()
            assert all(ress[i].num_iteration_records == 0 for i in range(len(out)))
            assert bytes(t.snapshot()) == snap and bytes(u.snapshot()) == snap
    a, b = t.frame_step(opt=opt, **good), ref.frame_step(opt=opt, **good)
    _same_step(a, b, "after the refusals")
    assert np.array_equal(_f32(a["depth"]), _f32(b["depth"])) and bytes(t.snapshot()) == bytes(ref.snapshot())
    grp.close(); t.close(); u.close(); ref.close(); h.close()
