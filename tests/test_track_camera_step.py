"""limo's camera callback as one store call -- kba_track_camera_step and its group forms -- against the chain it replaces:
kba_track_frame_step (or its lidar form), the caller's post-push landmark list built on the host from the creation's flags and
the candidates' tags, then kba_track_keyframe_solve when the block is due.  Two copies of each store go through the closed-loop
drives of tests/keyframe_drive.py with limo's solve rule; after every frame the outputs, both results and the snapshots of the
two stores must be equal byte for byte.  The struct layout, the exports and the binding's request builder are checked without a
GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from limo_b200 import capi
from limo_b200.capi_types import KbaCameraStepOut, KbaCameraStepRequest
from tests.keyframe_drive import KeyframeDrive
from tests.test_track_frame_step import Loop, _options, _same_step
from tests.test_track_rank import _same_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KBA_ERR_BAD_ARG = 1
OUTLIER, SHRUB, GROUND = 1, 2, 4
CLASSES = {1: OUTLIER, 2: SHRUB, 3: GROUND, 5: SHRUB | GROUND}


# ---- without a GPU ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("struct,name", [(KbaCameraStepRequest, "kba_camera_step_request"), (KbaCameraStepOut, "kba_camera_step_out")])
def test_struct_layout_matches_header(tmp_path, struct, name):
    fields = [f for f, _ in struct._fields_ if f != "reserved_"]
    prog = tmp_path / "lay.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "kba_b200.h"\nint main(){printf("%%zu", sizeof(%s));' % name +
                    "".join('printf(" %%zu", offsetof(%s, %s));' % (name, f) for f in fields) + 'return 0;}\n')
    exe = tmp_path / "lay"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(struct)] + [getattr(struct, f).offset for f in fields]


def test_the_three_symbols_are_exported():
    L = C.CDLL(capi.LIB_PATH)
    for name in ("kba_track_camera_step", "kba_track_group_camera_step", "kba_track_group_camera_step_opts"):
        assert hasattr(L, name) and name in capi.SYMBOLS, name


class _Stub:
    """capi.lib(): every C function records its name and the camera step's arguments decoded during the call, and succeeds"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            if "camera_step" in name:  # (handle, req, lid, opt_adjust, opt_solve, out, res_adjust, res_solve)
                self.calls.append((name, self._decode(args[1], args[2], len(args[-1])), args[3], args[4]))
            return 0
        fn.__name__ = name
        return fn

    @staticmethod
    def _decode(req, lid, n):
        out = []
        for i in range(n):
            q = req[i]
            if q.step.n_kf == 0:
                out.append(None)
                continue
            L = q.n_cand
            out.append(dict(solve=q.solve, n_kf=q.step.n_kf, kf_new=q.step.kf_new, cand=list(q.lm_slot[:L]), tags=list(q.lm_new[:L]),
                            ground=list(q.lm_ground[:L]) if q.lm_ground else None, d_null=not q.step.d, lidar=bool(lid),
                            n_points=lid[i].n_points if lid else None, outliers=list(q.outlier_slot[:q.n_outlier])))
        return out


@pytest.fixture
def stub(monkeypatch):
    s = _Stub()
    monkeypatch.setattr(capi, "_lib", s)
    return s


def _fake(n_cam, n):
    ts = []
    for i in range(n):
        t = capi.Track.__new__(capi.Track)
        t._p, t.n_cam, t._n_sel = C.c_void_p(0x10 + i), n_cam, None
        ts.append(t)
    gr = capi.TrackGroup.__new__(capi.TrackGroup)
    gr._p, gr.tracks = C.c_void_p(0x100), ts
    return ts, gr


def _small(rng, **kw):
    r = dict(kf_slots=[0, 1], lm_slot=[3, 3, 5, 9], u=rng.random(4), v=rng.random(4), d=rng.random(4), run_sel=[1, 0, 1], kf_new=2,
             new_slots=[9], pose7=[1.0, 0, 0, 0, 0, 0, 0], stamp=7_000, stamp_last=5_000, critical_quaternion_diff=0.03,
             time_difference_ns=400, solve="if_selected", cand_slots=[1, 3, 5, 9], cand_tags=[-2, -2, -1, 0],
             cand_ground=[0, 1, 0, 0], outliers=[1], draws=np.arange(5))
    r.update(kw)
    return r


def test_binding_builds_the_request(stub):
    rng = np.random.default_rng(0)
    (t,), _ = _fake(1, 1)
    t.camera_step(**_small(rng))
    (name, recs, _oa, _os), = stub.calls
    assert name == "kba_track_camera_step"
    assert recs == [dict(solve=2, n_kf=2, kf_new=2, cand=[1, 3, 5, 9], tags=[-2, -2, -1, 0], ground=[0, 1, 0, 0], d_null=False,
                         lidar=False, n_points=None, outliers=[1])]


def test_group_binding_builds_each_request(stub):
    rng = np.random.default_rng(1)
    ts, gr = _fake(1, 3)
    o1, o2 = capi.KbaOptions(), capi.KbaOptions()
    o1.final_solver_iterations, o2.final_solver_iterations = 3, 7
    gr.camera_step([_small(rng, solve="always"), None, _small(rng, solve="never", cand_tags=[-2, -1, -1, 0])],
                   opt_adjust=[o1, o2, None], opt_solve=[o2, o1, None])
    (name, recs, oa, os_), = stub.calls
    assert name == "kba_track_group_camera_step_opts"
    assert recs[1] is None and [r["solve"] for r in (recs[0], recs[2])] == [1, 0]
    assert recs[0]["tags"] == [-2, -2, -1, 0] and recs[2]["tags"] == []  # a request that never solves sends no candidates
    assert [oa[i].final_solver_iterations for i in range(2)] == [3, 7] and [os_[i].final_solver_iterations for i in range(2)] == [7, 3]
    cloud = rng.random((20, 4)).astype(np.float32)
    lid = dict(cloud=cloud, T_cam_lidar=np.tile([1.0, 0, 0, 0, 0, 0, 0], (1, 1)))
    r = _small(rng)
    del r["d"]
    gr.camera_step([dict(r, **lid), None, dict(r, **lid)])
    name, recs, _oa, _os = stub.calls[-1]
    assert name == "kba_track_group_camera_step" and recs[0]["lidar"] and recs[0]["d_null"] and recs[2]["n_points"] == 20


def test_malformed_requests_fail_before_the_call(stub):
    rng = np.random.default_rng(2)
    (t,), gr = _fake(1, 1)
    with pytest.raises(ValueError):
        t.camera_step(**_small(rng, solve="sometimes"))
    with pytest.raises(ValueError):
        t.camera_step(**_small(rng, cand_tags=[-2, -2]))
    r = _small(rng)
    with pytest.raises(ValueError):
        gr.camera_step([dict(r, cloud=rng.random((5, 4)).astype(np.float32), T_cam_lidar=[1.0, 0, 0, 0, 0, 0, 0])])
    assert stub.calls == []


# ---- on the device -----------------------------------------------------------------------------------------------------
def _track(h, dr, m_cap, ground=False, win_rows=0):
    rows = max(len(dr.arena(k)[0]) for k in range(dr.n_frames))
    w = dr.window // 2
    t = capi.Track(h, dr.cam_intr, dr.cam_pose, max_keyframes=w + 2, max_landmarks=dr.n_lm + 1, max_measurements=m_cap,
                   win_keyframes=w + 1, win_landmarks=max(rows, dr.n_lm + 1), win_observations=(w + 1) * rows,
                   win_ground=dr.n_lm + 1 if ground else 0, win_rows=win_rows)
    return t, rows


class CamLoop(Loop):
    """Loop's frame bookkeeping plus the solve block's: the active landmark set, the outlier set, the ground flags"""

    def __init__(self, dr, seed, lm_cap, ground):
        super().__init__(dr, seed, lm_cap)
        self.act, self.outl, self.gflag, self.ground = set(), set(), {}, ground
        self.cover = dict(solved_unselected=0, ifsel_solved=0, ifsel_skipped=0, reactivated=0, not_created=0, solved=0)

    def camera_request(self, k, r, run_ids):
        """the solve keywords of frame k: limo's rule (more than two keyframes, enough time since the last solve) as a policy"""
        n = len(self.active)
        due_time = k % 3 != 0
        solve = "never" if not due_time else ("always" if n >= 3 else ("if_selected" if n == 2 else "never"))
        measured = {int(s) for s in r["lm_slot"]}
        created = {self.slot_of[int(a)] for a in run_ids if int(a) in self.created}
        new = list(r["new_slots"])
        cands = sorted(self.act | (measured & created) | set(new))
        tags = [new.index(s) if s in new else (-2 if s in self.act else -1) for s in cands]
        rng = self.rng
        trk = [(int(s), int(rng.choice([0, 1, 2, 3, 5], p=[0.5, 0.05, 0.15, 0.2, 0.1])), int(rng.random() < 0.02))
               for s in sorted(measured) if rng.random() < 0.5]
        kw = dict(solve=solve, cand_slots=cands, cand_tags=tags, cand_ground=[self.gflag.get(s, False) for s in cands],
                  max_window=self.dr.window // 2, tracklets=trk, label_classes=CLASSES, outliers=sorted(self.outl & self.act),
                  shrubbery_weight=0.25, draws=rng.integers(0, 2**31 - 1, len(cands) + 1), voxel_size=(0.5, 0.5, 0.3),
                  scale_weight=-1.0, scale_value=1.5, depth=[(0, 20), (2, 20)], max_near=int(rng.choice([5, 300])), max_middle=30,
                  max_far=80)
        if self.ground:
            kw.update(ground=True, plane_reg_weight=-1.0)
        return kw

    def lists(self, kw, step):
        """the chain's post-push list from the frame step's outputs"""
        sel, fl = step["selected"], step["flags"]
        keep = [t == -2 or (sel and (t == -1 or (t >= 0 and fl[t] & 1))) for t in kw["cand_tags"]]
        idx = np.cumsum(keep) - 1
        return [s for s, f in zip(kw["cand_slots"], keep) if f], np.where(keep, idx, -1).astype(np.int32), \
            [g for g, f in zip(kw["cand_ground"], keep) if f]

    def chain_solve(self, t, r, kw, step, opt):
        due = kw["solve"] == "always" or (kw["solve"] == "if_selected" and step["selected"])
        if not due:
            return None, None
        lms, idx, gr = self.lists(kw, step)
        kf = list(r["kf_slots"]) + ([r["kf_new"]] if step["selected"] else [])
        skw = {k: v for k, v in kw.items() if k not in ("solve", "cand_slots", "cand_tags", "cand_ground")}
        return t.keyframe_solve(kf_slots=kf, lm_slots=lms, lm_ground=gr, opt=opt, **skw), idx

    def after(self, tracks, r, run_ids, kw, one, k):
        step = one["step"]
        c = self.cover
        c["not_created"] += step["selected"] and bool((step["flags"] & 1 == 0).any())
        c["reactivated"] += step["selected"] and any(t == -1 for t in kw["cand_tags"]) and self.cover["solved"] > 0
        was = [s for s, _ in self.active]
        self.advance(tracks, r, run_ids, step, k)
        if not one["solved"]:
            c["ifsel_skipped"] += kw["solve"] == "if_selected"
            self.act &= set(self.slot_of.values())
            return
        c["solved"] += 1
        c["solved_unselected"] += not step["selected"]
        c["ifsel_solved"] += kw["solve"] == "if_selected"
        lms, _, _ = self.lists(kw, step)
        s = one["solve"]
        self.act = {x for x, f in zip(lms, s["lm_active"]) if f}
        self.outl = {x for x, f in zip(lms, s["lm_outlier"]) if f}
        self.gflag.update({x: bool(g) for x, g in zip(lms, s["lm_ground"])})
        kf = was + ([r["kf_new"]] if step["selected"] else [])
        gone = [x for x, f in zip(kf, s["kf_active"]) if not f and x in {a for a, _ in self.active}]
        if gone:
            self.drop(tracks, gone)
        self.act &= set(self.slot_of.values())


def _same_solve(one, ref, where):
    for key in ("kf_active", "kf_common", "lm_active", "lm_outlier", "lm_ground", "trk_outlier", "cand", "category"):
        n = len(ref[key])
        assert np.array_equal(np.asarray(one[key])[:n], np.asarray(ref[key])), (where, key)
    assert (one["n_ground"], one["n_draws"]) == (ref["n_ground"], ref["n_draws"]), where
    _same_result(one["result"], ref["result"])


DRIVES = [dict(seed=1, window=12, rig=False), dict(seed=2, window=12, rig=True, lidar=True),
          dict(seed=3, window=20, rig=False, n_frames=70, ground=True, win_rows=201), dict(seed=4, window=20, rig=True, n_frames=60, lidar=True)]


def _cloud_args(dr, seed, k):
    from tests.test_track_frame_step_lidar import _frame_cloud, _rig_lidar
    T, lo = _rig_lidar(len(dr.cam_intr))
    return dict(cloud=_frame_cloud(seed, k, empty=k % 9 == 4), T_cam_lidar=T, lidar_opt=lo, depths=True)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", DRIVES, ids=lambda kw: "w%d_%s%s" % (kw["window"], "rig" if kw["rig"] else "mono",
                                                                     "_lidar" if kw.get("lidar") else ""))
def test_camera_step_equals_the_chain(kw):
    kw = dict(kw)
    lidar, ground, win_rows = kw.pop("lidar", False), kw.pop("ground", False), kw.pop("win_rows", 0)
    dr = KeyframeDrive(**kw)
    h = capi.Handle(0)
    probe, rows = _track(h, dr, 1)
    probe.close()
    m_cap = (dr.window // 2 + 1) * rows + rows // 2  # small: the arena compacts inside steps
    a, _ = _track(h, dr, m_cap, ground, win_rows)
    b = a.clone()
    loop = CamLoop(dr, kw["seed"], dr.n_lm + 1, ground)
    loop.first([a, b])
    loop.act = set(loop.slot_of[i] for i in loop.created)
    oa, os_ = _options(), _options()
    os_.final_solver_iterations = 8
    for k in range(1, dr.n_frames):
        r, run_ids = loop.request(k)
        if lidar:
            r = {x: y for x, y in r.items() if x != "d"}
            r.update(_cloud_args(dr, kw["seed"], k))
        skw = loop.camera_request(k, r, run_ids)
        step = a.frame_step(opt=oa, **r)
        ref, idx = loop.chain_solve(a, r, skw, step, os_)
        one = b.camera_step(opt_adjust=oa, opt_solve=os_, **r, **skw)
        _same_step(one["step"], step, k)
        if lidar:
            assert np.array_equal(one["step"]["depth"].view(np.uint32), step["depth"].view(np.uint32)), k
        assert one["solved"] == (ref is not None), k
        if ref is not None:
            assert one["n_lm"] == int((idx >= 0).sum()) and np.array_equal(one["lm_index"], idx), k
            _same_solve(one["solve"], ref, k)
        assert bytes(a.snapshot()) == bytes(b.snapshot()), k
        loop.after([a, b], r, run_ids, skw, one, k)
    assert loop.pushed_rows > m_cap, (loop.pushed_rows, m_cap)  # some frame step compacted the arena
    # IF_SELECTED comes up when a window holds two keyframes; the mono drives see both of its outcomes, the rig drives one
    need = [x for x in loop.cover if not x.startswith("ifsel")] + (["ifsel_solved", "ifsel_skipped"] if not kw["rig"] else [])
    assert all(loop.cover[x] > 0 for x in need) and loop.cover["ifsel_solved"] + loop.cover["ifsel_skipped"] > 0, loop.cover
    a.close(); b.close(); h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("lidar", [False, True], ids=["d", "lidar"])
def test_group_camera_step_equals_single_calls(lidar):
    """8 mono tracks of different drives: sit-outs, frame-step-only and solving tracks, per-track adjust and solve options"""
    h = capi.Handle(0)
    n = 8
    drs = [KeyframeDrive(10 + i, n_frames=16, window=12, rig=False) for i in range(n)]
    loops, singles, grouped = [], [], []
    for i, dr in enumerate(drs):
        probe, rows = _track(h, dr, 1)
        probe.close()
        t, _ = _track(h, dr, (dr.window // 2 + 1) * rows + rows // 2)
        loops.append(CamLoop(dr, 10 + i, dr.n_lm + 1, False))
        loops[-1].first([t])
        loops[-1].act = set(loops[-1].slot_of[x] for x in loops[-1].created)
        singles.append(t)
        grouped.append(t.clone())
    g = capi.TrackGroup(h, grouped)
    oas, oss = [_options() for _ in range(n)], [_options() for _ in range(n)]
    for i in range(n):
        oas[i].reprojection_thres, oss[i].reprojection_thres = 1.1 + 0.1 * i, 2.0 - 0.1 * i
    kinds = dict(sat=0, stepped=0, solved=0)
    for k in range(1, 16):
        reqs, rs = [], []
        for i in range(n):
            if (k + i) % 5 == 0:
                reqs.append(None); rs.append(None)
                continue
            r, run_ids = loops[i].request(k)
            if lidar:
                r = {x: y for x, y in r.items() if x != "d"}
                r.update(_cloud_args(drs[i], 10 + i, k))
            skw = loops[i].camera_request(k, r, run_ids)
            reqs.append(dict(r, **skw)); rs.append((r, run_ids, skw))
        got = g.camera_step(reqs, opt_adjust=oas, opt_solve=oss)
        for i in range(n):
            if reqs[i] is None:
                assert got[i] is None
                kinds["sat"] += 1
                continue
            one = singles[i].camera_step(opt_adjust=oas[i], opt_solve=oss[i], **reqs[i])
            _same_step(got[i]["step"], one["step"], (k, i))
            assert got[i]["solved"] == one["solved"], (k, i)
            kinds["solved" if one["solved"] else "stepped"] += 1
            if one["solved"]:
                assert got[i]["n_lm"] == one["n_lm"] and np.array_equal(got[i]["lm_index"], one["lm_index"]), (k, i)
                _same_solve(got[i]["solve"], one["solve"], (k, i))
            assert bytes(singles[i].snapshot()) == bytes(grouped[i].snapshot()), (k, i)
            r, run_ids, skw = rs[i]
            loops[i].after([singles[i], grouped[i]], r, run_ids, skw, one, k)
    assert all(v > 0 for v in kinds.values()), kinds
    g.close()
    for t in singles + grouped:
        t.close()
    h.close()


def _setup(seed=21):
    dr = KeyframeDrive(seed, n_frames=30, window=12, rig=False)
    h = capi.Handle(0)
    probe, rows = _track(h, dr, 1)
    probe.close()
    a, _ = _track(h, dr, (dr.window // 2 + 1) * rows + rows // 2)
    loop = CamLoop(dr, seed, dr.n_lm + 1, False)
    loop.first([a])
    loop.act = set(loop.slot_of[x] for x in loop.created)
    return dr, h, a, loop


@pytest.mark.gpu
def test_refusals():
    dr, h, a, loop = _setup()
    opt = _options()
    # run until the window has three keyframes, so that the next frame's solve is ALWAYS
    k = 1
    while len(loop.active) < 3 or k % 3 == 0:
        r, run_ids = loop.request(k)
        skw = loop.camera_request(k, r, run_ids)
        one = a.camera_step(opt_adjust=opt, opt_solve=opt, **r, **skw)
        loop.after([a], r, run_ids, skw, one, k)
        k += 1
    r, run_ids = loop.request(k)
    skw = loop.camera_request(k, r, run_ids)
    assert skw["solve"] == "always"
    snap = bytes(a.snapshot())
    # early refusals: nothing written, no store changed
    bad_tags = list(skw["cand_tags"])
    bad_tags[0] = len(r["new_slots"])
    for bad in (dict(skw, cand_tags=bad_tags), dict(skw, outliers=[dr.n_lm + 5])):
        with pytest.raises(capi.KbaError):
            a.camera_step(opt_adjust=opt, opt_solve=opt, **r, **bad)
        assert bytes(a.snapshot()) == snap
    # a late refusal: the failing draw function; the store holds the frame step's writes, as the chain's after its frame step
    b = a.clone()
    step = b.frame_step(opt=opt, **r)
    chain_snap = bytes(b.snapshot())
    lms, _, _ = loop.lists(skw, step)
    if len(lms) > 2:
        late = dict(skw, draws=lambda n, out: 1, max_middle=5)
        req = (KbaCameraStepRequest * 1)()
        with pytest.raises(capi.KbaError, match="draw function failed"):
            a.camera_step(opt_adjust=opt, opt_solve=opt, **r, **late)
        assert bytes(a.snapshot()) == chain_snap
        del req
    b.close(); a.close(); h.close()


@pytest.mark.gpu
def test_transfers_follow_the_formula():
    """the camera step's transfers minus the frame step's (measured on a clone) against the header's terms: a request that never
    solves moves exactly the frame step's bytes, one whose IF_SELECTED is unmet adds exactly its lists' upload"""
    dr, h, a, loop = _setup(22)
    opt = _options()
    seen = unsolved = 0
    for k in range(1, 30):
        r, run_ids = loop.request(k)
        skw = loop.camera_request(k, r, run_ids)
        if k % 4 == 2:  # a frame no scheme selects, with IF_SELECTED: the lists go up and nothing else
            r.update(time_difference_ns=2**62, critical_quaternion_diff=10.0)
            skw["solve"] = "if_selected"
        b, c = a.clone(), a.clone()  # a clone packs the arena: both calls run on clones, so that they compact alike
        b.frame_step(opt=opt, **r)
        fs_up, fs_down, _ = b.transfer_bytes()
        b.close()
        one = c.camera_step(opt_adjust=opt, opt_solve=opt, **r, **skw)
        up, down, _ = c.transfer_bytes()
        a.close()
        a = c
        if skw["solve"] == "never":
            assert (up, down) == (fs_up, fs_down), k
        elif not one["solved"]:  # the lists went up, nothing else
            L, K, T = len(skw["cand_slots"]), len(r["kf_slots"]) + 1, len(skw["tracklets"])
            lists = 8 * len(skw["depth"]) + 4 * (K + 2 * L + len(skw["outliers"]) + T) + L + T
            assert up - fs_up == lists, k
            assert down == fs_down, k
            unsolved += 1
        else:
            seen += 1
            assert up > fs_up and down > fs_down, k
        loop.after([a], r, run_ids, skw, one, k)
    assert seen > 0 and unsolved > 0, (seen, unsolved)
    a.close(); h.close()
