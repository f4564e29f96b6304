"""Evaluation of the stored window (kba_track_evaluate / kba_track_group_evaluate(_opts)): residuals, losses, trimming values and
decisions and the cost parts of the window kba_track_solve would build, at the store's state, without changing the store.

Without a GPU: the ctypes mirror of kba_evaluate_out against the header, the exported symbols, and the request and output builders
of the binding.
On the GPU, with the drives of tests/test_track_group.py and tests/test_track_ground.py (mono with depth, a two-camera rig, ground
points attached on the device, 12 keyframes and 20 on a win_rows > 184 track), evaluated after several pushes and solves:
  - every raw residual row equals the CPU oracle's on the window rebuilt on the host from the store's snapshot, the losses
    numpy's scaled Cauchy, the trimming values and decisions their numpy / oracle recomputation from the returned rows, and the
    total cost the oracle's first initial cost and that of the track's solve of the same request;
  - the device attachment equals the host attachment bit for bit, the store is untouched, and a solve after an evaluation equals
    the solve of a clone that was never evaluated;
  - groups of 1, 3 and 32 equal single calls bit for bit, sit-outs, failing requests, per-track options and errors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from limo_b200.capi_types import Window
from tests.test_track_ground import _GroundDrive, _attach, _requests
from tests.test_track_group import ROOT, _Drive, _equal

KEYS = ("obs_lm", "obs_kf", "obs_cam", "residual", "rho", "trim_repr", "trim_depth", "rejected_repr", "rejected_depth", "gp_lm",
        "gp_kf", "gp_weight", "gp_residual", "cost")


# ---- CPU --------------------------------------------------------------------------------------------------------------------------
def test_evaluate_out_matches_ctypes_mirror(tmp_path):
    """sizeof(kba_evaluate_out) and every field offset as gcc compiles them == the ctypes mirror's"""
    from limo_b200 import capi_types as T
    fields = [f for f, _ in T.KbaEvaluateOut._fields_]
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "kba_b200.h"\nint main(){printf("%zu' + ' %zu' * len(fields) +
                    '\\n",sizeof(kba_evaluate_out)' + "".join(",offsetof(kba_evaluate_out,%s)" % f for f in fields) + ');return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(T.KbaEvaluateOut)] + [getattr(T.KbaEvaluateOut, f).offset for f in fields]


def test_evaluate_symbols_exported():
    from limo_b200 import capi
    L = capi.lib()
    for s in ("kba_track_evaluate", "kba_track_group_evaluate", "kba_track_group_evaluate_opts"):
        assert s in capi.SYMBOLS
        getattr(L, s)
    assert L.kba_version() == 5


def test_evaluate_request_builder():
    """Track._evaluate_request is the solve's request (the shared builder) with outputs sized for the capacities; the result
    function slices them by the counts the library writes"""
    from limo_b200 import capi
    from limo_b200.capi_types import KbaTrackCaps
    t = capi.Track.__new__(capi.Track)
    t.caps = KbaTrackCaps(8, 100, 1000, 6, 50, 400, 16, 0)
    kf, fx, lm = [3, 1, 2], np.array([1, 0, 0], np.uint8), np.arange(7, dtype=np.int32)
    q, o, keep, done = t._evaluate_request(kf, fx, lm, scale_weight=-1.0, gp_lm=np.array([1, 4], np.int32), plane_reg_weight=-1.0)
    qs, _, _, _ = t._solve_request(1, kf, fx, lm, scale_weight=-1.0, gp_lm=np.array([1, 4], np.int32), plane_reg_weight=-1.0)
    assert (q.n_kf, q.n_lm) == (qs.n_kf, qs.n_lm) == (3, 7)
    assert q.sel.contents.scale_weight == -1.0 and q.sel.contents.n_gp == 2 and not q.sel.contents.gp_kf
    assert list(np.ctypeslib.as_array(q.kf_slot, (3,))) == kf and list(np.ctypeslib.as_array(q.lm_slot, (7,))) == list(lm)
    assert o.obs_capacity == 400
    assert t._evaluate_request(kf, fx, lm, obs_capacity=9)[1].obs_capacity == 9
    # what the library would write: 5 observations, 1 ground-plane residual
    np.ctypeslib.as_array(o.residual, (400 * 3,))[:15] = np.arange(15.0)
    np.ctypeslib.as_array(o.rejected_repr, (7,))[:] = [0, 1, 0, 0, 0, 0, 1]
    o.n_obs, o.n_gp, o.failed = 5, 1, 0
    o.cost[:] = [1, 2, 3, 4, 5, 15]
    r = done(o)
    assert r["n_obs"] == 5 and r["residual"].shape == (5, 3) and r["residual"][4, 2] == 14.0
    assert r["rho"].shape == (5, 2) and r["obs_lm"].shape == (5,) and r["trim_repr"].shape == (7,)
    assert r["gp_residual"].shape == (1,) and list(r["rejected_repr"]) == [False, True] + [False] * 4 + [True]
    assert list(r["cost"]) == [1, 2, 3, 4, 5, 15] and capi.COST_PARTS[-1] == "total" and r["failed"] is False


# ---- GPU helpers --------------------------------------------------------------------------------------------------------------------
def _host_window(sn, req, ev, opt):
    """the window of req rebuilt on the host from the store's snapshot sn: per selected landmark its entries of the listed
    keyframes in (keyframe, arena) order; the ground-plane lists are the evaluation's (checked separately), the scale and plane
    rules resolved as the reference does"""
    row = {int(s): i for i, s in enumerate(sn["slot"])}
    off = np.concatenate([[0], np.cumsum(sn["count"])])
    kf, lm = [int(s) for s in req["kf_slots"]], np.asarray(req["lm_slots"], np.int64)
    index = {int(j): i for i, j in enumerate(lm)}
    rows = [[] for _ in lm]
    for k, s in enumerate(kf):
        for a in range(off[row[s]], off[row[s] + 1]):
            i = index.get(int(sn["lm"][a]))
            if i is not None:
                rows[i].append((k, int(sn["cam"][a]), sn["u"][a], sn["v"][a], sn["d"][a]))
    flat = [x for r in rows for x in r]
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    col = lambda i, dt: np.array([x[i] for x in flat], dtype=dt)  # noqa: E731
    od = col(4, np.float32)
    n_depth, n_gp = int((od > 0).sum()), ev["n_gp"]
    sc = {k: req[k] for k in ("scale_kf0", "scale_kf1", "scale_weight", "scale_value")}
    dist_fixed = bool(req.get("plane_dist_fixed", False))
    if sc["scale_weight"] < 0:  # cpp:703-716, 722-728
        sc["scale_weight"] = (1000.0 / (n_depth + n_gp) if n_gp < 30 else 0.0) if (n_depth > 10 or n_gp > 10) else 1000.0
        dist_fixed = n_depth < 10
    prw = req.get("plane_reg_weight", 0.0)
    prw = (10.0 if n_gp > 0 else 0.0) if prw < 0 else prw
    sel = [row[s] for s in kf]
    gp = dict(gp_lm=ev["gp_lm"], gp_kf=ev["gp_kf"], gp_weight=ev["gp_weight"]) if n_gp else {}
    return Window(sn["pose"][sel], req["kf_fixed"], sn["cam_intr"], sn["cam_pose"], sn["pos"][lm], sn["weight"][lm], ptr, col(0, np.int32),
                  col(2, np.float32), col(3, np.float32), od, obs_cam=col(1, np.int32), kf_plane=sn["plane"][sel], plane_reg_weight=prw,
                  plane_dist_fixed=dist_fixed, **sc, **gp)


def _close(a, b, rtol, atol, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, what
    bad = np.abs(a - b) > rtol * np.abs(b) + atol
    assert not bad.any(), "%s: %d of %d differ, worst %s vs %s" % (what, bad.sum(), bad.size, a[bad][:3], b[bad][:3])


def _check_oracle(ev, win, opt, what):
    """ev against the CPU oracle on the host-built window win.  An observation the oracle cannot evaluate (|z_cam| < 0.01) must
    have NaN rows and losses and set `failed`; the costs are compared when every observation evaluates (else the solve fails)."""
    from oracle import oracle as orc
    n = win.n_obs
    assert ev["n_obs"] == n, what
    lm_of = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr))
    assert np.array_equal(ev["obs_lm"], lm_of) and np.array_equal(ev["obs_kf"], win.obs_kf), what
    assert np.array_equal(ev["obs_cam"], win.obs_cam), what
    ref, ok = np.zeros((n, 3)), np.ones(n, bool)
    for o in range(n):
        k, c, j = win.obs_kf[o], win.obs_cam[o], lm_of[o]
        ok[o], r2, _, _ = orc.reprojection(win.kf_pose[k], win.cam_pose[c], win.cam_intr[c], win.lm_pos[j], win.obs_u[o], win.obs_v[o],
                                           jac=False)
        ref[o, :2] = r2
        if win.obs_d[o] > 0:
            ref[o, 2] = orc.depth(win.kf_pose[k], win.cam_pose[c], win.lm_pos[j], win.obs_d[o])[0][0]
    assert ev["failed"] == (not ok.all()), what
    r = ev["residual"]
    assert np.isnan(r[~ok]).all() and np.isnan(ev["rho"][~ok]).all(), what
    _close(r[ok], ref[ok], 1e-12, 1e-12, what + ": residual rows")
    # scaled Cauchy w b log(1 + s / b) of each block, from the returned rows
    w = win.lm_weight[lm_of]
    b_r, b_d = opt.reprojection_thres ** 2, opt.depth_thres ** 2
    has_d = win.obs_d > 0
    rho = np.stack([w * b_r * np.log1p((r[:, 0] ** 2 + r[:, 1] ** 2) / b_r), np.where(has_d, w * b_d * np.log1p(r[:, 2] ** 2 / b_d), 0.0)], 1)
    _close(ev["rho"][ok], rho[ok], 1e-12, 1e-12, what + ": rho")
    # trimming values: per landmark the largest raw block norm over the observations that evaluate (k_trim_eval), -1 without one
    tr, td = np.full(win.n_lm, -1.0), np.full(win.n_lm, -1.0)
    np.maximum.at(tr, lm_of[ok], np.sqrt(r[ok, 0] * r[ok, 0] + r[ok, 1] * r[ok, 1]))
    dd = ok & has_d
    np.maximum.at(td, lm_of[dd], np.abs(r[dd, 2]))
    _close(ev["trim_repr"], tr, 1e-15, 0.0, what + ": trim_repr")
    assert np.array_equal(ev["trim_depth"], td), what
    # decisions: TrimmerQuantile over the landmarks that have the group, none below min_residual_groups
    for key, vals, q in (("rejected_repr", ev["trim_repr"], opt.reprojection_quantile), ("rejected_depth", ev["trim_depth"], opt.depth_quantile)):
        want = np.zeros(win.n_lm, bool)
        has = vals >= 0
        if has.sum() and has.sum() >= opt.min_residual_groups:
            want[has] = orc.trimmer_quantile(vals[has], q)[1]
        assert np.array_equal(ev[key], want), what + ": " + key
    if not ok.all():
        return False
    # ground-plane height residuals and their Huber cost, scale regulariser and plane chain from the oracle's residual functions
    g_r = np.array([orc.gp_height(win.kf_pose[k], win.kf_plane[k, :3], win.kf_plane[k, 3], win.lm_pos[j])[0][0]
                    for j, k in zip(ev["gp_lm"], ev["gp_kf"])])
    _close(ev["gp_residual"], g_r, 1e-12, 1e-12, what + ": gp_residual")
    a2 = opt.gp_huber ** 2
    s2 = g_r * g_r
    huber = np.where(s2 > a2, 2.0 * opt.gp_huber * np.sqrt(s2) - a2, s2)
    c = ev["cost"]
    _close(c[2], 0.5 * (ev["gp_weight"] * huber).sum(), 1e-12, 1e-15, what + ": ground-plane cost")
    c_s = 0.0
    if win.scale_weight > 0:
        r_s = orc.scale_reg(win.kf_pose[win.scale_kf1], win.kf_pose[win.scale_kf0], win.scale_value)[0][0]
        c_s = 0.5 * win.scale_weight * r_s * r_s
    _close(c[3], c_s, 1e-9, 1e-20, what + ": scale-regulariser cost")
    c_p, wp = 0.0, win.plane_reg_weight
    if wp > 0 and win.n_kf > 1:
        P = win.kf_plane
        for k in range(win.n_kf - 1):
            c_p += 0.5 * 3 * wp * np.sum((P[k + 1, :3] - P[k, :3]) ** 2) + 0.5 * wp * (P[k + 1, 3] - P[k, 3]) ** 2
            c_p += 0.5 * 2 * wp * orc.gp_motion(win.kf_pose[k], win.kf_pose[k + 1], P[k, :3])[0][0] ** 2
        c_p += 0.5 * wp * np.sum((np.array([0.0, 0.0, 1.0]) - P[:, :3]) ** 2)
    _close(c[4], c_p, 1e-10, 1e-15, what + ": plane-chain cost")
    _close(c[:2], [0.5 * ev["rho"][:, 0].sum(), 0.5 * ev["rho"][:, 1].sum()], 1e-12, 0.0, what + ": cost parts")
    _close(c[5], c[:5].sum(), 1e-15, 0.0, what + ": total")
    ro = orc.solve_window(win, opt)
    _close(c[5], ro.solves[0].initial_cost, 1e-10, 0.0, what + ": total against the oracle's initial cost")
    return True


def _same(a, b, what):
    assert a["n_obs"] == b["n_obs"] and a["n_gp"] == b["n_gp"] and a["failed"] == b["failed"], what
    for k in KEYS:
        assert np.array_equal(a[k], b[k]), what + ": " + k


def _large_ground(h):
    """a 20-keyframe ground window of candidates on a win_rows = 301 track (the large-window solver)"""
    from tests.test_track_large import _candidates, _sub, _track
    dr = _GroundDrive(seed=331, W=20, n_lm=1400, n_obs=13000, steps=1)
    t = _track(dr, h, 301)
    req = _sub(dr, 0, 20)
    cand, gp, n_att = _candidates(dr, 15)
    assert n_att > 0
    return dr, t, dict(req, gp_lm=cand, plane_reg_weight=-1.0), gp


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["mono", "rig", "ground", "large"])
def test_evaluate_against_oracle_and_solver(kind):
    """after several pushes and solves: the evaluation against the oracle on the host-rebuilt window, its total cost against the
    track's next solve of the same request, the device attachment against the host's, the store untouched, and the solve after
    it equal to that of a clone that was never evaluated"""
    from limo_b200 import capi
    from limo_b200.capi_types import parse_snapshot
    h = capi.Handle(0)
    opt = capi.default_options()
    if kind == "large":
        dr, t, req, gp = _large_ground(h)
    else:
        dr = _Drive(seed=401, W=12, n_lm=900, n_obs=9000, rig=kind == "rig") if kind != "ground" else \
            _GroundDrive(seed=402, W=12, n_lm=900, n_obs=8000, steps=4)
        t = dr.make_track(h)
    n_checked = 0
    for step in range(3 if kind != "large" else 1):
        if kind != "large":
            if step:
                dr.advance(t, step)
            req = _requests(dr, step, 20)[0] if kind == "ground" else dr.request(step)
        what = "%s step %d" % (kind, step)
        before = t.snapshot()
        twin = t.clone()
        ev = t.evaluate(**req)
        assert np.array_equal(before, t.snapshot()), what + ": the store changed"
        sn = parse_snapshot(before)
        if kind in ("ground", "large"):  # the device attachment at the stored state equals the host's, bit for bit
            lm = np.asarray(req["lm_slots"])
            row = {int(s): i for i, s in enumerate(sn["slot"])}
            sel = [row[int(s)] for s in req["kf_slots"]]
            keep, best, wgt = _attach(sn["pose"][sel], sn["plane"][sel], sn["pos"][lm])
            cand = req["gp_lm"]
            k = keep[cand]
            assert ev["n_gp"] == int(k.sum()) > 0, what
            assert np.array_equal(ev["gp_lm"], cand[k]) and np.array_equal(ev["gp_kf"], best[cand][k]), what
            assert np.array_equal(ev["gp_weight"], wgt[cand][k]), what
        evaluated = _check_oracle(ev, _host_window(sn, req, ev, opt), opt, what)
        n_checked += evaluated
        ra, rb = t.solve(**req), twin.solve(**req)
        _equal(ra, rb, len(req["lm_slots"]), what + ": solve after an evaluation")
        assert np.array_equal(t.snapshot(), twin.snapshot()), what
        if evaluated:
            _close(ev["cost"][5], ra.solves[0].initial_cost, 1e-12, 0.0, what + ": total against the solve's initial cost")
        twin.close()
        dr.record(ra)
        print("%s: %d observations, %d ground points, failed %s, cost %s" % (what, ev["n_obs"], ev["n_gp"], ev["failed"], ev["cost"]))
    assert n_checked >= 1, kind  # the costs were compared at least once
    t.close(); h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 3, 32])
def test_group_equals_single_calls(G):
    """group outputs bit-equal to single calls; a sit-out leaves its output unwritten; a failing request in position k names
    track k and changes nothing; with _opts each track gets its own quantiles"""
    from limo_b200 import capi
    h = capi.Handle(0)
    base = [_Drive(seed=411 + i, W=5 + i, n_lm=300, n_obs=2500, rig=i == 2) for i in range(4)]
    drives = [base[i % 4] for i in range(G)]
    tracks = [d.make_track(h) for d in drives]
    for i, (d, t) in enumerate(zip(drives, tracks)):  # a different state per track: some solves
        for step in range(1, 1 + i % 3):
            d.advance(t, step)
            t.solve(**d.request(step))
    reqs = [d.request(i % 3) for i, d in enumerate(drives)]
    grp = capi.TrackGroup(h, tracks)
    evs = grp.evaluate(reqs)
    for i, t in enumerate(tracks):
        _same(evs[i], t.evaluate(**reqs[i]), "G %d track %d" % (G, i))
    # per-track quantiles
    opts = []
    for i in range(G):
        o = capi.default_options()
        o.reprojection_quantile, o.depth_quantile, o.min_residual_groups = 0.5 + 0.4 * i / max(G - 1, 1), 0.7, 5
        opts.append(o)
    evo = grp.evaluate(reqs, opt=opts)
    for i, t in enumerate(tracks):
        _same(evo[i], t.evaluate(**reqs[i], opt=opts[i]), "G %d _opts track %d" % (G, i))
    if G > 1:
        assert sum(e["rejected_repr"].sum() for e in evo) != sum(e["rejected_repr"].sum() for e in evs)
        # sit-outs: output structs untouched
        from limo_b200.capi_types import KbaEvaluateOut, KbaOptions, KbaTrackRequest
        n = len(tracks)
        q = (KbaTrackRequest * n)()
        out = (KbaEvaluateOut * n)()
        keep, done = [], []
        for i in range(n):
            if i % 2:
                out[i].n_obs, out[i].n_gp = -7, -7
                continue
            qi, oi, k, d = tracks[i]._evaluate_request(**reqs[i])
            q[i], out[i] = qi, oi
            keep.append(k); done.append((i, d))
        capi._check(capi.lib().kba_track_group_evaluate(grp._p, q, C.byref(capi.default_options()), out))
        for i in range(n):
            if i % 2:
                assert out[i].n_obs == -7 and out[i].n_gp == -7
        for i, d in done:
            _same(d(out[i]), evs[i], "G %d sitting out around track %d" % (G, i))
        # one FP32 option set is refused also when track 0 sits out; a request without keyframes is refused as the single call does
        o32 = capi.default_options()
        o32.precision = 1
        with pytest.raises(capi.KbaError, match="error 1.*FP64"):
            grp.evaluate([None] + reqs[1:], opt=o32)
        with pytest.raises(capi.KbaError, match="track 0: fewer than 3 keyframes"):
            grp.evaluate([dict(reqs[0], kf_slots=[], kf_fixed=[])] + reqs[1:])
        assert grp.evaluate([None] + reqs[1:])[0] is None
        # a bad request in the last position fails the call, names its track and changes nothing
        snaps = [t.snapshot() for t in tracks]
        bad = list(reqs)
        bad[-1] = dict(reqs[-1], kf_slots=[drives[-1].W + 5] + list(reqs[-1]["kf_slots"])[1:])
        with pytest.raises(capi.KbaError, match="error 1.*track %d" % (G - 1)):
            grp.evaluate(bad)
        assert all(np.array_equal(a, t.snapshot()) for a, t in zip(snaps, tracks))
    grp.close()
    for t in tracks:
        t.close()
    h.close()


@pytest.mark.gpu
def test_evaluate_errors():
    """a short observation capacity is KBA_ERR_CAPACITY with n_obs written; FP32 options are refused; transfers are counted"""
    from limo_b200 import capi
    h = capi.Handle(0)
    dr = _Drive(seed=421, W=6, n_lm=400, n_obs=3000)
    t = dr.make_track(h)
    req = dr.request(0)
    ev = t.evaluate(**req)
    up, down, _ = t.transfer_bytes()
    assert 0 < up < 4096 and down > 40 * ev["n_obs"], (up, down)
    q, o, _keep, _ = t._evaluate_request(obs_capacity=ev["n_obs"] - 1, **req)
    rc = capi.lib().kba_track_evaluate(t._p, C.byref(q), C.byref(capi.default_options()), C.byref(o))
    assert rc == 4 and o.n_obs == ev["n_obs"] and o.n_gp == 0
    assert b"obs_capacity" in capi.lib().kba_last_error()
    assert t.evaluate(obs_capacity=ev["n_obs"], **req)["n_obs"] == ev["n_obs"]
    o32 = capi.default_options()
    o32.precision = 1
    with pytest.raises(capi.KbaError, match="error 1.*FP64"):
        t.evaluate(**req, opt=o32)
    with pytest.raises(capi.KbaError, match="error 3"):
        t.evaluate(**dict(req, kf_slots=req["kf_slots"][:2], kf_fixed=req["kf_fixed"][:2]))
    t.close(); h.close()


def test_facade_evaluate_host():
    """tests/cpp/test_facade_evaluate.cpp, host mode: evaluateResiduals() throws naming the reason with the persistent window off and
    before the first solve(); the keying of the outputs by (landmark id, keyframe timestamp, camera id) and by landmark id, and the
    refusal of an output in another order"""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])
    out = subprocess.run([os.path.join(ROOT, "tests", "cpp", "test_facade_evaluate"), "host"], capture_output=True, text=True)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr


@pytest.mark.gpu
def test_facade_evaluate():
    """tests/cpp/test_facade_evaluate.cpp on the device: after every solve() of a two-camera drive, evaluateResiduals() gives one
    residual per measurement of a selected landmark in an active keyframe, each equal to a host computation from the facade's state,
    losses and trimming values that agree with them, and changes no pose or selection"""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])
    out = subprocess.run([os.path.join(ROOT, "tests", "cpp", "test_facade_evaluate")], capture_output=True, text=True)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
