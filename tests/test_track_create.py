"""push()'s landmark creation on the device-resident store (kba_track_create_landmarks / kba_track_group_create_landmarks) against a
restatement of the facade's host code.

For every landmark a pushed keyframe measures for the first time, the facade back-projects its first measurement with a lidar depth
(calculateLandmark(kf, id)) or triangulates the rays of every active keyframe and camera that measure it (calculateLandmark(id),
triangulate_rays).  The restatement below follows facade/bundle_adjuster_keyframes.cpp and internal/mini_eigen.hpp operation for
operation (numpy float64 scalars are IEEE doubles and divide by zero like the host), and test_restatement_equals_facade pins it to
the facade's own push() without a GPU (tests/cpp/test_facade_create.cpp, host mode).  On the GPU the device must then equal it bit
for bit: positions (NaN where the host has NaN), flags, and the store."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.create_drive import Drive
from tests.test_track_select import _apply, _iso

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_create")
D = np.float64
NAN3 = (float("nan"),) * 3


# ---- the host code, restated ---------------------------------------------------------------------------------------------------
def _mul(A, B):
    """Isometry3d product: R = Ra Rb (each entry summed from 0), t = Ra tb + ta"""
    (Ra, _), (Rb, tb) = A, B
    R = [[((0.0 + Ra[i][0] * Rb[0][j]) + Ra[i][1] * Rb[1][j]) + Ra[i][2] * Rb[2][j] for j in range(3)] for i in range(3)]
    return R, _apply(A, tb)


def _inv(T):
    R, t = T
    Rt = [[R[j][i] for j in range(3)] for i in range(3)]
    return Rt, [-((Rt[i][0] * t[0] + Rt[i][1] * t[1]) + Rt[i][2] * t[2]) for i in range(3)]


def _mv(m, p):
    """Matrix3d * Vector3d, m row-major flat"""
    return [(m[3 * i] * p[0] + m[3 * i + 1] * p[1]) + m[3 * i + 2] * p[2] for i in range(3)]


def _inverse3(m):
    """mini_eigen's Matrix3d::inverse(): cofactors over the determinant"""
    m = [D(x) for x in m]
    d = (m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6])) + m[2] * (m[3] * m[7] - m[4] * m[6])
    return [(m[4] * m[8] - m[5] * m[7]) / d, (m[2] * m[7] - m[1] * m[8]) / d, (m[1] * m[5] - m[2] * m[4]) / d,
            (m[5] * m[6] - m[3] * m[8]) / d, (m[0] * m[8] - m[2] * m[6]) / d, (m[2] * m[3] - m[0] * m[5]) / d,
            (m[3] * m[7] - m[4] * m[6]) / d, (m[1] * m[6] - m[0] * m[7]) / d, (m[0] * m[4] - m[1] * m[3]) / d]


def host_create(dr, active, kf_new, lm_ids):
    """push()'s creation of landmarks lm_ids, keyframe kf_new just pushed, keyframes `active` (ascending id) active.
    Returns [(flags, (x, y, z))] with flags bit 0 created, bit 1 has depth; NaN positions where not created."""
    camT = [_iso(c) for c in dr.cam_pose]
    ray_T = {(k, c): _inv(_mul(camT[c], _iso(dr.kf_pose[k]))) for k in active for c in range(len(camT))}
    intr_inv = [_inverse3([f, 0.0, cx, 0.0, f, cy, 0.0, 0.0, 1.0]) for f, cx, cy in dr.cam_intr]
    out = []
    with np.errstate(all="ignore"):
        for lid in lm_ids:
            obs = dr.meas[kf_new].get(lid, [])
            if any(o[3] >= 0 for o in obs):                                   # containsDepth: a NaN is no depth
                # calculateLandmark(kf, id) skips entries with d < 0 only: a NaN before the depth is taken
                c, u, v, d = next(o for o in obs if not o[3] < 0)
                f, cx, cy = dr.cam_intr[c]
                z = float(d)
                x, y = ((float(u) - cx) * z) / f, ((float(v) - cy) * z) / f
                out.append((3, tuple(_apply(ray_T[(kf_new, c)], [x, y, z]))))
                continue
            S, rhs, n = [0.0] * 9, [0.0] * 3, 0                               # calculateLandmark(id), triangulate_rays
            for k in active:
                for c, u, v, _ in dr.meas[k].get(lid, []):
                    ray = _mv(intr_inv[c], [float(u), float(v), 1.0])
                    nrm = np.sqrt((ray[0] * ray[0] + ray[1] * ray[1]) + ray[2] * ray[2])
                    ray = [r / nrm for r in ray]
                    R, t = ray_T[(k, c)]
                    r = _mv([x for row in R for x in row], ray)
                    cur = [(1.0 if i == j else 0.0) - r[i] * r[j] for i in range(3) for j in range(3)]
                    S = [S[q] + cur[q] for q in range(9)]
                    ct = _mv(cur, t)
                    rhs = [rhs[i] + ct[i] for i in range(3)]
                    n += 1
            out.append((1, tuple(_mv(_inverse3(S), rhs))) if n >= 2 else (0, NAN3))
    return out


def drive_requests(dr):
    """what the facade drive does at each push (tests/cpp/test_facade_create.cpp): keyframes max(0, k - window) .. k active, the
    landmarks push() has to create plus every fourth landmark of the keyframe that exists already.  Yields
    (k, active, request ids in ascending order, host_create's result)."""
    created = set()
    for k in range(dr.n_push):
        active = list(range(max(0, k - dr.window), k + 1))
        ids = sorted(lid for lid in dr.meas[k] if lid not in created or lid % 4 == 0)
        res = host_create(dr, active, k, ids)
        created |= {lid for lid, (fl, _) in zip(ids, res) if fl & 1}
        yield k, active, ids, res


def _same(a, b):
    a, b = np.asarray(a, D).ravel(), np.asarray(b, D).ravel()
    nan = np.isnan(b)
    return np.array_equal(np.isnan(a), nan) and np.array_equal(a[~nan].view(np.int64), b[~nan].view(np.int64))


DRIVES = [dict(seed=1, window=12, rig=True), dict(seed=2, window=12, rig=False), dict(seed=3, window=20, rig=True),
          dict(seed=4, window=20, rig=False)]


def _build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])


# ---- CPU: the restatement against the facade's push() --------------------------------------------------------------------------
@pytest.mark.parametrize("kw", DRIVES, ids=lambda kw: "w%d_%s" % (kw["window"], "rig" if kw["rig"] else "mono"))
def test_restatement_equals_facade(kw, tmp_path):
    _build()
    dr = Drive(**kw)
    path = tmp_path / "drive.txt"
    dr.write(path)
    r = subprocess.run([EXE, "host", str(path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    facade = {}
    for line in r.stdout.split("\n"):
        if line:
            k, lid, cr, dp, x, y, z = line.split()
            facade[(int(k), int(lid))] = (int(cr) | 2 * int(dp), tuple(float.fromhex(s) if "n" not in s else float("nan") for s in (x, y, z)))
    seen = dict(depth=0, depth_second_cam=0, nan_then_depth=0, nan_depth=0, two_rays=0, many_rays=0, one_ray=0, degenerate=0, total=0)
    for k, active, ids, res in drive_requests(dr):
        for lid, (fl, pos) in zip(ids, res):
            ffl, fpos = facade.pop((k, lid))
            assert ffl == fl, (k, lid, ffl, fl)
            assert _same(pos, fpos), (k, lid, pos, fpos)
            seen["total"] += 1
            obs = dr.meas[k][lid]
            seen["depth"] += fl == 3
            seen["depth_second_cam"] += fl == 3 and obs[0][3] < 0
            seen["nan_then_depth"] += fl == 3 and bool(np.isnan(obs[0][3])) and bool(np.isnan(pos).all())
            seen["nan_depth"] += bool(np.isnan([o[3] for o in obs]).any()) and fl == 1
            rays = sum(len(dr.meas[a].get(lid, [])) for a in active)
            seen["two_rays"] += fl == 1 and rays == 2
            seen["many_rays"] += fl == 1 and rays > 2
            seen["one_ray"] += fl == 0
            seen["degenerate"] += fl == 1 and not np.isfinite(pos).all()
    assert not facade, "lines the restatement did not produce: %s" % list(facade)[:5]
    need = ["depth", "two_rays", "many_rays", "one_ray", "degenerate"] + (["depth_second_cam", "nan_then_depth"] if kw["rig"] else [])
    assert all(seen[n] > 0 for n in need), seen


def test_create_struct_sizes_match_header(tmp_path):
    """sizeof() of the creation structs as the C compiler sees them == size of the ctypes mirrors"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu\\n",'
                    'sizeof(kba_create_request),sizeof(kba_create_out));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(T.KbaCreateRequest), C.sizeof(T.KbaCreateOut)]


# ---- GPU: the device against the restatement -----------------------------------------------------------------------------------
def _track(h, dr, sentinel=None, solves=True):
    """a track sized for the drive; keyframe k goes to slot k % (window + 2).  sentinel: positions every landmark slot starts from;
    solves=False: the smallest solve capacities (a track that only creates landmarks)"""
    from limo_b200 import capi
    n_meas = sum(len(o) for m in dr.meas for o in m.values())
    t = capi.Track(h, dr.cam_intr, dr.cam_pose, max_keyframes=dr.window + 2, max_landmarks=dr.n_lm, max_measurements=n_meas,
                   win_keyframes=min(dr.window + 1, 30), win_landmarks=max(dr.n_lm, 64) if solves else 64,
                   win_observations=n_meas if solves else 64)
    if sentinel is not None:
        t.set_landmarks(np.arange(dr.n_lm), pos=sentinel, weight=np.full(dr.n_lm, 0.5))
    return t


def _push(t, dr, k):
    S = dr.window + 2
    if k >= dr.window + 1:
        t.drop_keyframe((k - dr.window - 1) % S)
    lm, cam, u, v, d = dr.arena(k)
    t.push_keyframe(k % S, dr.kf_pose[k], lm, u, v, d, cam=cam)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", DRIVES, ids=lambda kw: "w%d_%s" % (kw["window"], "rig" if kw["rig"] else "mono"))
def test_create_matches_host(kw):
    from limo_b200 import capi
    dr = Drive(**kw)
    h = capi.Handle(0)
    t = _track(h, dr, solves=False)
    S = dr.window + 2
    for k, active, ids, res in drive_requests(dr):
        _push(t, dr, k)
        pos, flags = t.create_landmarks([a % S for a in active], len(active) - 1, ids)
        assert np.array_equal(flags, [fl for fl, _ in res]), k
        assert _same(pos, [p for _, p in res]), k
        h2d, d2h, _ = t.transfer_bytes()
        assert (h2d, d2h) == (4 * (len(active) + len(ids)), 25 * len(ids))
    t.close(); h.close()


@pytest.mark.gpu
def test_solve_after_create_equals_solve_after_set():
    """the store after create_landmarks: created slots hold the restated positions with weight 1, the others are untouched --
    a solve over every slot then equals, bit for bit, the solve of a track that got the same values through set_landmarks"""
    from limo_b200 import capi
    dr = Drive(5, n_push=8, window=6, rig=True, new_per_push=40)
    rng = np.random.default_rng(0)
    sentinel = rng.uniform(-1, 1, (dr.n_lm, 3)) + np.array([30.0, 0.0, 1.0])
    h = capi.Handle(0)
    a, b = _track(h, dr, sentinel), _track(h, dr, sentinel)
    S = dr.window + 2
    for k, active, ids, res in drive_requests(dr):
        _push(a, dr, k); _push(b, dr, k)
        a.create_landmarks([x % S for x in active], len(active) - 1, ids)
        made = [(lid, p) for lid, (fl, p) in zip(ids, res) if fl & 1]
        if made:
            b.set_landmarks([lid for lid, _ in made], pos=np.array([p for _, p in made]), weight=np.ones(len(made)))
    active = list(range(dr.n_push - dr.window, dr.n_push))
    lms = sorted({lid for k in active for lid in dr.meas[k]})
    fixed = [1, 1] + [0] * (len(active) - 2)
    opt = capi.default_options()
    ra = a.solve([k % S for k in active], fixed, lms, opt=opt)
    rb = b.solve([k % S for k in active], fixed, lms, opt=opt)
    assert ra.c.status == 0 and rb.c.status == 0
    assert np.array_equal(ra.lm_pos.view(np.int64), rb.lm_pos.view(np.int64))
    assert np.array_equal(ra.kf_pose.view(np.int64), rb.kf_pose.view(np.int64))
    a.close(); b.close(); h.close()


def _group_setup(h):
    drives = [Drive(11, n_push=6, window=4, rig=True, new_per_push=50), Drive(12, n_push=7, window=5, rig=False, new_per_push=80),
              Drive(13, n_push=6, window=4, rig=True, new_per_push=30, depth=False)]
    tracks = [_track(h, dr, solves=False) for dr in drives]
    steps = [list(drive_requests(dr)) for dr in drives]
    return drives, tracks, steps


@pytest.mark.gpu
def test_group_equals_single_calls():
    """a group of heterogeneous tracks (rigs, sizes, with and without depth) with requests sitting out equals the single calls
    and the restatement; a group of one equals the single call"""
    from limo_b200 import capi
    h = capi.Handle(0)
    drives, tracks, steps = _group_setup(h)
    g = capi.TrackGroup(h, tracks)
    singles = [_track(h, dr, solves=False) for dr in drives]
    one = capi.TrackGroup(h, [singles[0]])
    n_steps = max(len(s) for s in steps)
    for k in range(n_steps):
        req = []
        for i, dr in enumerate(drives):
            if k >= len(steps[i]) or (k + i) % 3 == 2:  # this track sits the call out (its keyframe is pushed all the same)
                if k < len(steps[i]):
                    _push(tracks[i], dr, k); _push(singles[i], dr, k)
                    steps[i][k] = None
                req.append(None)
                continue
            _, active, ids, _ = steps[i][k]
            _push(tracks[i], dr, k); _push(singles[i], dr, k)
            S = dr.window + 2
            req.append(dict(kf_slots=[a % S for a in active], kf_new=len(active) - 1, lm_slots=ids))
        out = g.create_landmarks(req)
        for i, r in enumerate(req):
            if r is None:
                assert out[i] is None
                continue
            res = steps[i][k][3]
            pos, flags = singles[i].create_landmarks(**r) if i else one.create_landmarks([r])[0]
            assert np.array_equal(out[i][1], flags) and _same(out[i][0], pos)
            assert np.array_equal(flags, [fl for fl, _ in res]) and _same(pos, [p for _, p in res])
        act = [r for r in req if r is not None]
        h2d, d2h = g.transfer_bytes()
        assert d2h == 25 * sum(len(r["lm_slots"]) for r in act)
        R = h2d - 4 * sum(len(r["kf_slots"]) + len(r["lm_slots"]) for r in act)
        assert (R == 0) if len(act) <= 1 else (R > 0 and R % (len(act) - 1) == 0)
    assert g.create_landmarks([None] * len(tracks)) == [None] * len(tracks) and g.transfer_bytes() == (0, 0)
    for x in (g, one, *tracks, *singles):
        x.close()
    h.close()


@pytest.mark.gpu
def test_create_rejects_bad_requests_and_changes_nothing():
    """every invalid request fails with its code before anything is written: every store, the group's other track's included,
    still holds its sentinel positions and weights -- a solve over all its landmarks equals, bit for bit, the solve of a track that
    saw no failed call -- and the valid call afterwards gives what that track gives"""
    from limo_b200 import capi
    dr = Drive(21, n_push=4, window=3, rig=True, new_per_push=30)
    sentinel = np.random.default_rng(1).uniform(-1, 1, (dr.n_lm, 3)) + np.array([30.0, 0.0, 1.0])
    h = capi.Handle(0)
    t, other, ref = (_track(h, dr, sentinel) for _ in range(3))
    g = capi.TrackGroup(h, [other, t])
    steps = list(drive_requests(dr))
    for k in range(3):
        _push(t, dr, k); _push(other, dr, k); _push(ref, dr, k)
    _, active, ids, _ = steps[2]
    kf = [a % (dr.window + 2) for a in active]
    good = dict(kf_slots=kf, kf_new=len(kf) - 1, lm_slots=ids)
    bad = [(dict(good, kf_slots=[]), "no keyframes"), (dict(good, kf_new=len(kf)), "kf_new"), (dict(good, kf_new=-1), "kf_new"),
           (dict(good, kf_slots=kf + kf[:1]), "listed twice"), (dict(good, kf_slots=kf + [4]), "not pushed"),
           (dict(good, kf_slots=kf + [99]), "not pushed"), (dict(good, lm_slots=ids + ids[:1]), "listed twice"),
           (dict(good, lm_slots=ids + [dr.n_lm]), "out of range"), (dict(good, lm_slots=ids + [-1]), "out of range")]
    for r, msg in bad:
        with pytest.raises(capi.KbaError, match="error 1: .*" + msg):  # KBA_ERR_BAD_ARG
            t.create_landmarks(**r)
        if r["kf_slots"]:
            with pytest.raises(capi.KbaError, match="error 1: .*track 1: .*" + msg):
                g.create_landmarks([good, r])
    too_many = dict(good, lm_slots=np.arange(dr.n_lm + 1) % dr.n_lm)
    with pytest.raises(capi.KbaError, match="error 4: .*more keyframes or landmarks"):  # KBA_ERR_CAPACITY
        t.create_landmarks(**too_many)
    L = capi.lib()
    q = capi.KbaCreateRequest(n_kf=len(kf), kf_new=0, n_new=len(ids))
    o = capi.KbaCreateOut()
    assert L.kba_track_create_landmarks(t._p, C.byref(q), C.byref(o)) == 1  # null output arrays: KBA_ERR_BAD_ARG
    assert L.kba_track_create_landmarks(t._p, None, C.byref(o)) == 1
    lms = sorted({lid for k in range(3) for lid in dr.meas[k]})
    opt = capi.default_options()
    r0 = ref.solve(kf, [1, 1, 0], lms, opt=opt)
    assert r0.c.status == 0
    for x in (t, other):  # nothing was written by the failed calls: the stores solve as the untouched one does
        rx = x.solve(kf, [1, 1, 0], lms, opt=opt)
        assert rx.c.status == 0
        assert np.array_equal(rx.lm_pos.view(np.int64), r0.lm_pos.view(np.int64))
        assert np.array_equal(rx.kf_pose.view(np.int64), r0.kf_pose.view(np.int64))
    pos0, flags0 = ref.create_landmarks(**good)  # the solves moved the poses: the valid call now agrees with the untouched track's
    for x in (t, other):
        pos, flags = x.create_landmarks(**good)
        assert np.array_equal(flags, flags0) and _same(pos, pos0)
    g.close(); t.close(); other.close(); ref.close(); h.close()


@pytest.mark.gpu
def test_facade_device_creation_equals_push(tmp_path):
    """tests/cpp/test_facade_create: facade drives (two-camera and mono rigs, 12- and 20-keyframe windows, 30 pushes) mirrored
    into a track; after every push kba_track_create_landmarks equals the facade's own push() bit for bit"""
    _build()
    for kw in DRIVES:
        path = tmp_path / "drive.txt"
        Drive(**kw).write(path)
        r = subprocess.run([EXE, "device", str(path)], capture_output=True, text=True, timeout=1200)
        print(r.stdout)
        assert r.returncode == 0, r.stdout + r.stderr
