"""Landmark selection on the device-resident store (kba_track_select_landmarks) against a restatement of the facade's host code.

The device computes the per-landmark quantities of limo's selection chain -- cheirality, the voxel scheme's bins, the near order,
pixel flow and the seen counts -- from the poses, the arena and the positions in a track's store.  The restatement below follows
facade/landmark_selection.cpp and internal/mini_eigen.hpp operation for operation (Python floats are IEEE doubles, numpy float32
rounds like the host's float), so the outputs must be equal: exactly for the integers, bit for bit for the flows.  The facade
test (tests/cpp/test_facade_select.cpp) then checks the whole selection through LandmarkSelector against the host select()."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
DBL_MAX = float(np.finfo(np.float64).max)


# ---- the host code, restated ---------------------------------------------------------------------------------------------------
def _iso(q):
    """convert(Pose): Identity().translate(t).rotate(q) with Eigen's un-normalised toRotationMatrix -> (R rows, t)"""
    qw, qx, qy, qz = (float(x) for x in q[:4])
    tx, ty, tz = 2.0 * qx, 2.0 * qy, 2.0 * qz
    twx, twy, twz = tx * qw, ty * qw, tz * qw
    txx, txy, txz, tyy, tyz, tzz = tx * qx, ty * qx, tz * qx, ty * qy, tz * qy, tz * qz
    Rq = [[1.0 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1.0 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]
    e = lambda i, k: 1.0 if i == k else 0.0
    R = [[((0.0 + e(i, 0) * Rq[0][j]) + e(i, 1) * Rq[1][j]) + e(i, 2) * Rq[2][j] for j in range(3)] for i in range(3)]
    t = [0.0 + ((e(i, 0) * float(q[4]) + e(i, 1) * float(q[5])) + e(i, 2) * float(q[6])) for i in range(3)]
    return R, t


def _apply(T, p):
    R, t = T
    return [((R[i][0] * p[0] + R[i][1] * p[1]) + R[i][2] * p[2]) + t[i] for i in range(3)]


def _sq(v):
    return (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]


def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _dist_path(q, path):
    if len(path) == 1:
        return math.sqrt(_sq(_sub(q, path[0])))
    best = DBL_MAX
    for i in range(len(path) - 1):
        v, w = _sub(path[i + 1], path[i]), _sub(q, path[i])
        c1 = (w[0] * v[0] + w[1] * v[1]) + w[2] * v[2]
        c2 = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
        if c1 <= 0.0:
            d2 = _sq(w)
        elif c2 <= c1:
            d2 = _sq(_sub(q, path[i + 1]))
        else:
            t = c1 / c2
            d2 = _sq(_sub(q, [path[i][a] + v[a] * t for a in range(3)]))
        best = d2 if d2 < best else best
    return math.sqrt(best)


def host_select(scene, kf_list, cand, voxel, roi_far, roi_middle):
    """cheirality + voxel steps 1-5 + flow + seen, candidate-indexed like kba_select_out"""
    kfT = [_iso(scene.kf_pose[k]) for k in kf_list]
    camT = [_iso(c) for c in scene.cam_pose]
    n = len(cand)
    cheiral = np.ones(n, np.uint8)
    seen = np.zeros(n, np.int32)
    for c, lm in enumerate(cand):
        for ki, k in enumerate(kf_list):
            ms = scene.meas[k].get(lm)
            if not ms:
                continue
            seen[c] += 1
            pv = _apply(kfT[ki], scene.lm_pos[lm])
            for cam, _, _ in ms:
                if _apply(camT[cam], pv)[2] < 0.0:
                    cheiral[c] = 0
    cur = kfT[-1]
    path = []
    for T in kfT:
        R, t = T
        inv_t = [-((R[0][i] * t[0] + R[1][i] * t[1]) + R[2][i] * t[2]) for i in range(3)]
        path.append(_apply(cur, inv_t))
    bin_ = np.full(n, -1, np.int8)
    inside = []                                    # (candidate, float point)
    for c, lm in enumerate(cand):
        if not cheiral[c]:
            continue
        p = [F32(x) for x in _apply(cur, scene.lm_pos[lm])]
        if not (np.isfinite(p[2]) and p[2] >= F32(-20.0) and p[2] <= F32(100.0)):
            continue
        if _dist_path([float(x) for x in p], path) < roi_far:
            inside.append((c, p))
        else:
            bin_[c] = 2
    near = []
    if inside:
        inv = [F32(1.0) / F32(v) for v in voxel]
        mn = list(inside[0][1]); mx = list(inside[0][1])
        for _, p in inside:
            for a in range(3):
                mn[a] = p[a] if p[a] < mn[a] else mn[a]
                mx[a] = p[a] if mx[a] < p[a] else mx[a]
        min_b = [int(np.floor(F32(mn[a] * inv[a]))) for a in range(3)]
        div_b = [int(np.floor(F32(mx[a] * inv[a]))) - min_b[a] + 1 for a in range(3)]
        mul = [1, div_b[0], div_b[0] * div_b[1]]
        idx = []
        for i, (c, p) in enumerate(inside):
            v = 0
            for a in range(3):
                v += int(F32(np.floor(F32(p[a] * inv[a]))) - F32(min_b[a])) * mul[a]
            idx.append((v, i))
        idx.sort()
        a0 = 0
        while a0 < len(idx):
            b0 = a0
            s = [F32(0.0)] * 3
            while b0 < len(idx) and idx[b0][0] == idx[a0][0]:
                p = inside[idx[b0][1]][1]
                s = [F32(s[q] + p[q]) for q in range(3)]
                b0 += 1
            cnt = F32(b0 - a0)
            cen = [float(F32(s[q] / cnt)) for q in range(3)]
            c = inside[idx[a0][1]][0]
            if _dist_path(cen, path) < roi_middle:
                bin_[c] = 0
                near.append(c)
            else:
                bin_[c] = 1
            a0 = b0
    flow = np.full(n, np.nan)
    for c in near:
        lm = cand[c]
        last, fl = {}, {}
        for k in kf_list:
            for cam, u, v in scene.meas[k].get(lm, []):
                if cam in last:
                    du, dv = float(last[cam][0]) - float(u), float(last[cam][1]) - float(v)
                    fl[cam] = fl.get(cam, 0.0) + math.sqrt(du * du + dv * dv)
                last[cam] = (u, v)
        if fl:
            best = None
            for cam in sorted(fl):
                if best is None or best < fl[cam]:
                    best = fl[cam]
            flow[c] = best
    return dict(cheiral=cheiral, bin=bin_, near_order=np.array(near, np.int32), flow=flow, seen=seen)


# ---- seeded track stores -------------------------------------------------------------------------------------------------------
def _quat(yaw, pitch=0.0, roll=0.0):
    cy, sy, cp, sp, cr, sr = (math.cos(yaw / 2), math.sin(yaw / 2), math.cos(pitch / 2), math.sin(pitch / 2), math.cos(roll / 2),
                              math.sin(roll / 2))
    return [cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy]


class Scene:
    """keyframes driving along x (vehicle <- origin poses, z up), a rig of one or two cameras (z forward), landmarks ahead of and
    around the path: clusters that share a voxel, points above / below the PassThrough band, points far from the path, tracks
    seen once, points that fall behind the cameras of the last keyframes that still measure them"""

    def __init__(self, seed, n_kf=8, n_lm=600, rig=True):
        rng = np.random.default_rng(seed)
        self.n_kf = n_kf
        self.kf_pose = []
        for k in range(n_kf):
            q = _quat(0.01 * k + rng.normal(0, 0.003), rng.normal(0, 0.002), rng.normal(0, 0.002))
            self.kf_pose.append(np.array(q + [-1.5 * k + rng.normal(0, 0.01), rng.normal(0, 0.05), rng.normal(0, 0.02)]))  # at x = 1.5 k
        cams = [np.array([0.5, 0.5, -0.5, 0.5, 0.0, 0.0, 0.0])]  # camera <- vehicle: camera z = vehicle x, camera y = -vehicle z
        if rig:  # a second camera turned a little, with a quaternion that is not normalised (Eigen does not normalise either)
            cams.append(np.array([0.52, 0.48, -0.5, 0.5, 0.3, -0.1, 0.05]))
        self.cam_pose = cams
        self.cam_intr = [[700.0, 600.0, 190.0]] * len(cams)
        pos = np.column_stack([rng.uniform(-2, 70, n_lm), rng.uniform(-25, 25, n_lm), rng.uniform(-3, 6, n_lm)])
        m = n_lm // 10
        pos[:m] = pos[m:2 * m] + rng.uniform(-0.05, 0.05, (m, 3))          # pairs inside one voxel
        pos[2 * m:2 * m + 8, 2] = rng.choice([-40.0, 130.0], 8)              # outside the PassThrough band
        pos[2 * m + 8:2 * m + 20, 1] = rng.choice([-1.0, 1.0], 12) * rng.uniform(60, 90, 12)  # far from the path
        pos[2 * m + 20:2 * m + 40, 0] = rng.uniform(-14, -4, 20)            # behind the vehicle
        self.lm_pos = [list(map(float, p)) for p in pos]
        self.meas = [dict() for _ in range(n_kf)]  # keyframe -> landmark id -> [(camera, u, v)] in camera order
        for lm in range(n_lm):
            if lm % 17 == 0:                       # a track seen once
                span = [int(rng.integers(0, n_kf))]
            else:
                a = int(rng.integers(0, n_kf - 1))
                span = list(range(a, min(n_kf, a + int(rng.integers(2, n_kf + 1)))))
            for k in span:
                cams_k = [0] if not rig else [c for c in (0, 1) if rng.random() < 0.7] or [int(rng.integers(0, 2))]
                if lm % 17 == 0:
                    cams_k = cams_k[:1]
                self.meas[k][lm] = [(c, F32(rng.uniform(0, 1200)), F32(rng.uniform(0, 380))) for c in cams_k]
        self.slot = rng.permutation(n_lm).astype(np.int32)  # landmark id -> store slot: not in id order

    def make_track(self, h):
        from limo_b200 import capi
        n_meas = sum(len(ms) for d in self.meas for ms in d.values())
        t = capi.Track(h, self.cam_intr, self.cam_pose, max_keyframes=self.n_kf + 2, max_landmarks=len(self.lm_pos),
                       max_measurements=n_meas, win_keyframes=8, win_landmarks=64, win_observations=64)
        order = np.argsort(self.slot)            # slot -> landmark id
        t.set_landmarks(np.arange(len(self.lm_pos), dtype=np.int32), pos=np.array(self.lm_pos)[order])
        for k in range(self.n_kf):
            lm, cam, u, v = [], [], [], []
            for lid in sorted(self.meas[k]):
                for c, uu, vv in self.meas[k][lid]:
                    lm.append(self.slot[lid]); cam.append(c); u.append(uu); v.append(vv)
            t.push_keyframe(k, self.kf_pose[k], lm, u, v, np.full(len(lm), -1.0, np.float32), cam=cam)
        return t


PARAMS = [dict(voxel_size=(0.5, 0.5, 0.3), roi_far=40.0, roi_middle=15.0),   # limo's mono-lidar values
          dict(voxel_size=(2.0, 2.0, 1.0), roi_far=30.0, roi_middle=8.0)]


def _candidates(scene, kf_list, drop_every=23):
    """active landmarks (measured by a listed keyframe) minus every drop_every-th (the outliers), ascending id"""
    ids = sorted({lm for k in kf_list for lm in scene.meas[k]})
    return [lm for lm in ids if lm % drop_every != 5]


def _check(dev, ref):
    for key in ("cheiral", "bin", "near_order", "seen"):
        assert np.array_equal(dev[key], ref[key]), key
    nan = np.isnan(ref["flow"])
    assert np.array_equal(np.isnan(dev["flow"]), nan), "flow: which candidates have a value"
    assert np.array_equal(dev["flow"][~nan].view(np.int64), ref["flow"][~nan].view(np.int64)), "flow: bit patterns"


@pytest.mark.gpu
@pytest.mark.parametrize("seed,rig,n_lm", [(1, True, 600), (2, False, 600), (3, True, 4000)])
def test_select_matches_host(seed, rig, n_lm):
    from limo_b200 import capi
    sc = Scene(seed, n_lm=n_lm, rig=rig)
    h = capi.Handle(0)
    t = sc.make_track(h)
    kf_list = list(range(1, sc.n_kf))                # keyframe 0 stays in the store, inactive
    cand = _candidates(sc, kf_list)
    covered = dict(behind=0, multi_voxel=0, passthrough=0, no_flow=0, seen_ties=0)
    for p in PARAMS:
        dev = t.select_landmarks(kf_list, sc.slot[cand], **p)
        ref = host_select(sc, kf_list, cand, p["voxel_size"], p["roi_far"], p["roi_middle"])
        _check(dev, ref)
        assert len(ref["near_order"]) > 0 and (ref["bin"] == 1).any() and (ref["bin"] == 2).any()
        covered["behind"] += int((ref["cheiral"] == 0).sum())
        covered["multi_voxel"] += int(((ref["bin"] == -1) & (ref["cheiral"] == 1)).sum())
        covered["no_flow"] += int(np.isnan(ref["flow"][ref["near_order"]]).sum())
        far = ref["bin"] == 2
        covered["seen_ties"] += int(len(ref["seen"][far]) - len(np.unique(ref["seen"][far])))
        h2d, d2h, _ = t.transfer_bytes()
        assert h2d == 4 * (len(kf_list) + len(cand)) and d2h >= 18 * len(cand)
    covered["passthrough"] = sum(1 for lm in cand if abs(sc.lm_pos[lm][2]) > 30)
    assert all(v > 0 for v in covered.values()), covered
    t.close(); h.close()


@pytest.mark.gpu
def test_select_behind_one_keyframe_only():
    """a landmark that only the newest keyframe sees from behind is rejected; the same landmark is kept once that keyframe is not
    in the request, and a landmark the newest keyframe does not measure is not affected by it"""
    from limo_b200 import capi
    sc = Scene(5, n_lm=300, rig=True)
    lid = 7
    sc.lm_pos[lid] = [1.5 * (sc.n_kf - 1) - 3.0, 0.5, 1.0]   # 3 m behind the newest keyframe, ahead of keyframe 1
    for k in range(sc.n_kf):
        sc.meas[k].pop(lid, None)
    sc.meas[sc.n_kf - 1][lid] = [(0, F32(600.0), F32(190.0))]
    sc.meas[1][lid] = [(1, F32(610.0), F32(180.0))]
    h = capi.Handle(0)
    t = sc.make_track(h)
    for kf_list in (list(range(1, sc.n_kf)), list(range(1, sc.n_kf - 1))):
        cand = _candidates(sc, kf_list)
        dev = t.select_landmarks(kf_list, sc.slot[cand], **PARAMS[0])
        ref = host_select(sc, kf_list, cand, (0.5, 0.5, 0.3), 40.0, 15.0)
        _check(dev, ref)
        c = cand.index(lid)
        assert dev["cheiral"][c] == (0 if kf_list[-1] == sc.n_kf - 1 else 1)
    t.close(); h.close()


@pytest.mark.gpu
def test_select_rejects_bad_requests():
    from limo_b200 import capi
    sc = Scene(4, n_lm=200, rig=False)
    h = capi.Handle(0)
    t = sc.make_track(h)
    cand = sc.slot[_candidates(sc, [1, 2, 3])]
    for kf, lm, msg in (([], cand, "no keyframes"), ([1, 1, 2], cand, "listed twice"), ([1, 2, 20], cand, "not pushed"),
                        ([1, 2], np.r_[cand, cand[:1]], "listed twice"), ([1, 2], np.r_[cand, [10 ** 6]], "out of range")):
        with pytest.raises(capi.KbaError, match=msg):
            t.select_landmarks(kf, lm)
    with pytest.raises(capi.KbaError, match="voxel"):
        t.select_landmarks([1, 2], cand, voxel_size=(0.5, 0.0, 0.3))
    t.drop_keyframe(2)
    with pytest.raises(capi.KbaError, match="not pushed"):
        t.select_landmarks([1, 2], cand)
    t.close(); h.close()


def test_select_struct_sizes_match_header(tmp_path):
    """sizeof() of the selection structs as the C compiler sees them == size of the ctypes mirrors"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu\\n",'
                    'sizeof(kba_select_params),sizeof(kba_select_out));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(T.KbaSelectParams), C.sizeof(T.KbaSelectOut)]


@pytest.mark.gpu
def test_facade_device_selection_equals_host():
    """tests/cpp/test_facade_select: limo's mono-lidar selection chain (cheirality, voxel, AddDepth) over 12- and 20-keyframe
    drives; at every solve() the device-backed selection equals the host select(), and the end states are bit-identical"""
    exe = os.path.join(ROOT, "tests", "cpp", "test_facade_select")
    assert os.path.exists(exe), "build it with make -C limo_b200/csrc facade"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
