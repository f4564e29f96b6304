"""Window upkeep on the device-resident store -- deactivateKeyframes (kba_track_deactivate_keyframes) and the AddDepth scheme's
costs (kba_track_depth_costs), with their group forms -- against a restatement of the facade's host code.

The restatement below follows BundleAdjusterKeyframes::push() / deactivateKeyframes() and LandmarkSelectionSchemeAddDepth::
getSelection() with limo's comparator and sorter (is_ground_plane, float(local.norm())), and ranks the costs with a restatement
of libstdc++'s std::partial_sort (heap select), so that ties fall as on the host.  test_restatement_equals_facade pins it to the
facade's own calls without a GPU (tests/cpp/test_facade_upkeep.cpp, host mode).  On the GPU the device must equal it bit for bit:
common counts, flags, offsets, eligible indices and cost bits."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tests.test_track_create import host_create
from tests.test_track_select import _apply, _iso
from tests.upkeep_drive import UpkeepDrive

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_upkeep")
NEG = -np.finfo(np.float64).max
WANTED = 50


# ---- the host code, restated ---------------------------------------------------------------------------------------------------
def partial_sort_set(c, n):
    """the ids std::partial_sort(c.begin(), c.begin() + n, c.end(), cost <) leaves in front (libstdc++: __heap_select)"""
    a = list(c)
    less = lambda x, y: x[1] < y[1]  # noqa: E731

    def push_heap(hole, top, value):
        parent = (hole - 1) // 2
        while hole > top and less(a[parent], value):
            a[hole] = a[parent]
            hole = parent
            parent = (hole - 1) // 2
        a[hole] = value

    def adjust_heap(hole, length, value):
        top = second = hole
        while second < (length - 1) // 2:
            second = 2 * (second + 1)
            if less(a[second], a[second - 1]):
                second -= 1
            a[hole] = a[second]
            hole = second
        if (length & 1) == 0 and second == (length - 2) // 2:
            second = 2 * (second + 1)
            a[hole] = a[second - 1]
            hole = second - 1
        push_heap(hole, top, value)

    if n <= 0:
        return set()
    if n >= 2:
        parent = (n - 2) // 2
        while True:
            adjust_heap(parent, n, a[parent])
            if parent == 0:
                break
            parent -= 1
    for i in range(n, len(a)):
        if less(a[i], a[0]):
            v = a[i]
            a[i] = a[0]
            adjust_heap(0, n, v)
    return {x[0] for x in a[:n]}


def cost_of(kf_pose, pos):
    """std::max(-DBL_MAX, double(float(|kf * pos|))): a NaN norm leaves -DBL_MAX"""
    x, y, z = _apply(_iso(kf_pose), [float(v) for v in pos])
    with np.errstate(all="ignore"):
        v = float(np.float32(np.sqrt((x * x + y * y) + z * z)))
    return v if NEG < v else NEG


def drive_steps(dr):
    """the facade drive of tests/cpp/test_facade_upkeep.cpp: push() (landmarks created over the active keyframes), then from the
    fourth push deactivateKeyframes(3, 4, W), the labels and AddDepth over the active landmarks that exist and have id % 13 != 5.
    Yields one dict per step: k, the lists before deactivation (kf, lm), its outputs (common, kf_active, lm_active), the active
    keyframes after it, the eligible landmarks, the cost vectors as (off, cand, cost) and the selection."""
    W = dr.window
    active, active_lm, pos = [], set(), {}
    for k in range(dr.n_push):
        active.append(k)
        fresh = sorted(lid for lid in dr.meas[k] if lid not in pos)
        for lid, (fl, p) in zip(fresh, host_create(dr, active, k, fresh)):
            if fl & 1:
                pos[lid] = p
        active_lm |= {lid for lid in dr.meas[k] if lid in pos}  # push() skips the landmarks it could not create
        if k < 3:
            continue
        kf, lm = list(active), sorted(active_lm)
        newest = set(dr.meas[k])
        common = [len(set(dr.meas[a]) & newest) for a in kf]
        kf_active = []
        for i, c in enumerate(common):
            n = len(kf) - 1 - i
            kf_active.append(0 if n > W - 1 else (1 if n < 4 - 1 else int(c > 3)))
        active = [a for a, f in zip(kf, kf_active) if f]
        measured = set().union(*(dr.meas[a] for a in active))
        lm_active = [int(lid in measured) for lid in lm]
        active_lm = {lid for lid in active_lm if lid in measured}
        elig = sorted(lid for lid in active_lm if lid in pos and dr.ground[lid] and lid % 13 != 5)
        index = {lid: j for j, lid in enumerate(elig)}
        off, cand, cost = [0], [], []
        for a in active:
            for lid in sorted(dr.meas[a]):
                if lid in index:
                    cand.append(index[lid])
                    cost.append(cost_of(dr.kf_pose[a], pos[lid]))
            off.append(len(cand))
        sel = set()
        for ind in range(min(W, len(active))):
            c = [(elig[cand[i]], cost[i]) for i in range(off[ind], off[ind + 1])]
            sel |= partial_sort_set(c, min(WANTED, len(c)))
        yield dict(k=k, kf=kf, lm=lm, common=common, kf_active=kf_active, lm_active=lm_active, active=list(active), elig=elig, pos=dict(pos),
                   off=np.array(off, np.int32), cand=np.array(cand, np.int32), cost=np.array(cost, np.float64), sel=sel)


DRIVES = [dict(seed=1, window=12, rig=True), dict(seed=2, window=12, rig=False), dict(seed=3, window=20, rig=True),
          dict(seed=4, window=20, rig=False)]
IDS = lambda kw: "w%d_%s" % (kw["window"], "rig" if kw["rig"] else "mono")  # noqa: E731


def _build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])


# ---- CPU: the restatement against the facade -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", DRIVES, ids=IDS)
def test_restatement_equals_facade(kw, tmp_path):
    _build()
    dr = UpkeepDrive(**kw)
    path = tmp_path / "drive.txt"
    dr.write(path)
    r = subprocess.run([EXE, "host", str(path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    facade = {}
    for line in r.stdout.split("\n"):
        if line:
            tag, k, *ids = line.split()
            facade[(tag, int(k))] = [int(x) for x in ids]
    seen = dict(steps=0, by_rule=0, by_window=0, neg=0, tie=0, no_elig=0)
    for st in drive_steps(dr):
        k = st["k"]
        assert facade.pop(("D", k)) == st["active"], k
        assert facade.pop(("L", k)) == [lid for lid, f in zip(st["lm"], st["lm_active"]) if f], k
        assert set(facade.pop(("S", k))) == st["sel"], k
        seen["steps"] += 1
        n_kf = len(st["kf"])
        seen["by_rule"] += sum(1 for i, f in enumerate(st["kf_active"]) if not f and n_kf - 1 - i <= dr.window - 1)
        seen["by_window"] += sum(1 for i, f in enumerate(st["kf_active"]) if not f and n_kf - 1 - i > dr.window - 1)
        seen["neg"] += int((st["cost"] == NEG).sum())
        seen["no_elig"] += int((np.diff(st["off"]) == 0).sum())
        el = set(st["elig"])
        seen["tie"] += sum(1 for a, b in dr.ties if a in el and b in el and st["pos"][a] == st["pos"][b])
    assert not facade, "lines the restatement did not produce: %s" % list(facade)[:5]
    assert all(v > 0 for v in seen.values()), seen


def test_upkeep_struct_sizes_match_header(tmp_path):
    """sizeof() of the upkeep structs as the C compiler sees them == size of the ctypes mirrors"""
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n",sizeof(kba_deactivate_request),'
                    'sizeof(kba_deactivate_out),sizeof(kba_depth_request),sizeof(kba_depth_out));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(T.KbaDeactivateRequest), C.sizeof(T.KbaDeactivateOut), C.sizeof(T.KbaDepthRequest), C.sizeof(T.KbaDepthOut)]


def test_upkeep_null_arguments_need_no_device():
    """a null track, group, request or output is KBA_ERR_BAD_ARG before any device work"""
    _build()
    from limo_b200 import capi
    L = capi.lib()
    dq, do, cq, co = capi.KbaDeactivateRequest(), capi.KbaDeactivateOut(), capi.KbaDepthRequest(), capi.KbaDepthOut()
    for fn, q, o in ((L.kba_track_deactivate_keyframes, dq, do), (L.kba_track_group_deactivate_keyframes, dq, do),
                     (L.kba_track_depth_costs, cq, co), (L.kba_track_group_depth_costs, cq, co)):
        assert fn(None, C.byref(q), C.byref(o)) == 1
        assert "null argument" in capi.lib().kba_last_error().decode()


def test_partial_sort_restatement_keeps_heap_order_on_ties():
    """the heap select keeps libstdc++'s tied elements, not the first ones: pinned on a case where the two differ"""
    c = list(enumerate([1.0, 2.0, 1.0, 1.0, 1.0, 1.0, 0.0, 1.0, 2.0]))
    assert partial_sort_set(c, 5) == {0, 3, 4, 5, 6}  # what libstdc++ keeps; a stable sort would keep {0, 2, 3, 4, 6}
    assert partial_sort_set(c, 0) == set() and partial_sort_set(c, 9) == set(range(9))


# ---- GPU: the device against the restatement -----------------------------------------------------------------------------------
def _track(h, dr):
    from limo_b200 import capi
    n_meas = sum(len(o) for m in dr.meas for o in m.values())
    return capi.Track(h, dr.cam_intr, dr.cam_pose, max_keyframes=dr.window + 2, max_landmarks=dr.n_lm, max_measurements=n_meas,
                      win_keyframes=min(dr.window + 1, 30), win_landmarks=64, win_observations=64)


def _push(t, dr, k, pos, done):
    """keyframe k into slot k % (W + 2) (the keyframe that held it is inactive by then) and the positions created so far"""
    S = dr.window + 2
    if k >= S:
        t.drop_keyframe((k - S) % S)
    lm, cam, u, v, d = dr.arena(k)
    t.push_keyframe(k % S, dr.kf_pose[k], lm, u, v, d, cam=cam)
    new = sorted(set(pos) - done)
    if new:
        t.set_landmarks(new, pos=np.array([pos[i] for i in new]), weight=np.ones(len(new)))
        done |= set(new)


def _steps(dr):
    """every push with the restated step after it (None for the first three pushes)"""
    it = {st["k"]: st for st in drive_steps(dr)}
    return [it.get(k) for k in range(dr.n_push)]


def _bound(dr, st):
    return sum(min(len(st["elig"]), sum(len(o) for o in dr.meas[a].values())) for a in st["active"])


def _check_step(dr, st, deact, costs):
    kf_active, kf_common, lm_active = deact
    assert np.array_equal(kf_common, st["common"]) and np.array_equal(kf_active, st["kf_active"]), st["k"]
    assert np.array_equal(lm_active, st["lm_active"]), st["k"]
    off, cand, cost = costs
    assert np.array_equal(off, st["off"]) and np.array_equal(cand, st["cand"]), st["k"]
    assert np.array_equal(cost.view(np.int64), st["cost"].view(np.int64)), st["k"]


@pytest.mark.gpu
@pytest.mark.parametrize("kw", DRIVES, ids=IDS)
def test_upkeep_matches_restatement(kw):
    from limo_b200 import capi
    dr = UpkeepDrive(**kw)
    h = capi.Handle(0)
    t = _track(h, dr)
    S, done = dr.window + 2, set()
    for k, st in enumerate(_steps(dr)):
        pos = st["pos"] if st else {}
        _push(t, dr, k, pos, done)
        if st is None:
            continue
        deact = t.deactivate_keyframes([a % S for a in st["kf"]], st["lm"], 3, 4, dr.window)
        h2d, d2h, _ = t.transfer_bytes()
        assert (h2d, d2h) == (4 * (len(st["kf"]) + len(st["lm"])), 5 * len(st["kf"]) + len(st["lm"]))
        costs = t.depth_costs([a % S for a in st["active"]], st["elig"])
        h2d, d2h, _ = t.transfer_bytes()
        assert (h2d, d2h) == (4 * (len(st["active"]) + len(st["elig"])), 4 * len(st["active"]) + 12 * _bound(dr, st))
        _check_step(dr, st, deact, costs)
    t.close(); h.close()


@pytest.mark.gpu
def test_group_equals_single_calls():
    """a group of heterogeneous tracks (rigs, windows, sizes) with requests sitting out equals the single calls and the
    restatement; a group of one equals the single call; the transfer counts follow the header's formulas"""
    from limo_b200 import capi
    h = capi.Handle(0)
    drives = [UpkeepDrive(31, n_push=14, window=6, rig=True), UpkeepDrive(32, n_push=16, window=8, rig=False, new_per_push=70),
              UpkeepDrive(33, n_push=12, window=5, rig=True, new_per_push=25)]
    steps = [_steps(dr) for dr in drives]
    tracks, singles = [_track(h, dr) for dr in drives], [_track(h, dr) for dr in drives]
    done = [[set(), set()] for _ in drives]
    g = capi.TrackGroup(h, tracks)
    one = capi.TrackGroup(h, [singles[0]])
    for k in range(max(dr.n_push for dr in drives)):
        dreq, creq = [], []
        for i, dr in enumerate(drives):
            st = steps[i][k] if k < dr.n_push else None
            if k < dr.n_push:
                pos = st["pos"] if st else {}
                _push(tracks[i], dr, k, pos, done[i][0]); _push(singles[i], dr, k, pos, done[i][1])
            if st is None or (k + i) % 3 == 2:  # sits the call out
                dreq.append(None); creq.append(None)
                continue
            S = dr.window + 2
            dreq.append(dict(kf_slots=[a % S for a in st["kf"]], lm_slots=st["lm"], min_connecting=3, min_window=4, max_window=dr.window))
            creq.append(dict(kf_slots=[a % S for a in st["active"]], lm_slots=st["elig"]))
        dout = g.deactivate_keyframes(dreq)
        dbytes = g.transfer_bytes()
        cout = g.depth_costs(creq)
        cbytes = g.transfer_bytes()
        act = [i for i, r in enumerate(dreq) if r is not None]
        for i in range(len(drives)):
            if i not in act:
                assert dout[i] is None and cout[i] is None
                continue
            st = steps[i][k]
            if i == 0:
                sd, sc = one.deactivate_keyframes([dreq[0]])[0], one.depth_costs([creq[0]])[0]
            else:
                sd, sc = singles[i].deactivate_keyframes(**dreq[i]), singles[i].depth_costs(**creq[i])
            for a, b in zip(dout[i] + cout[i], sd + sc):
                assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
            _check_step(drives[i], st, dout[i], cout[i])
        if not act:
            assert dbytes == (0, 0) and cbytes == (0, 0)
            continue
        R = dbytes[0] - 4 * sum(len(dreq[i]["kf_slots"]) + len(dreq[i]["lm_slots"]) for i in act)
        assert (R == 0) if len(act) == 1 else (R > 0 and R % (len(act) - 1) == 0)
        assert dbytes[1] == sum(5 * len(dreq[i]["kf_slots"]) + len(dreq[i]["lm_slots"]) for i in act)
        assert cbytes[0] == R + 4 * sum(len(creq[i]["kf_slots"]) + len(creq[i]["lm_slots"]) for i in act)
        assert cbytes[1] == sum(4 * len(creq[i]["kf_slots"]) + 12 * _bound(drives[i], steps[i][k]) for i in act)
    assert g.depth_costs([None] * 3) == [None] * 3 and g.transfer_bytes() == (0, 0)
    for x in (g, one, *tracks, *singles):
        x.close()
    h.close()


@pytest.mark.gpu
def test_upkeep_errors_write_nothing():
    """every invalid request fails with its code before anything is written: sentinel outputs of the single call and of every
    request of a group stay as they were; the valid call afterwards equals the restatement"""
    from limo_b200 import capi
    dr = UpkeepDrive(41, n_push=6, window=4, rig=True, new_per_push=30)
    steps = _steps(dr)
    h = capi.Handle(0)
    t, other = _track(h, dr), _track(h, dr)
    g = capi.TrackGroup(h, [other, t])
    done = [set(), set()]
    for k in range(dr.n_push):
        pos = steps[k]["pos"] if steps[k] else {}
        _push(t, dr, k, pos, done[0]); _push(other, dr, k, pos, done[1])
    st = steps[-1]
    S = dr.window + 2
    kf, lm = [a % S for a in st["kf"]], st["lm"]
    ak, el = [a % S for a in st["active"]], st["elig"]
    good_d = dict(kf_slots=kf, lm_slots=lm, min_connecting=3, min_window=4, max_window=dr.window)
    good_c = dict(kf_slots=ak, lm_slots=el)
    B = _bound(dr, st)
    bad = [(dict(good_d, kf_slots=kf + kf[:1]), dict(good_c, kf_slots=ak + ak[:1]), 1, "listed twice"),
           (dict(good_d, kf_slots=kf + [S]), dict(good_c, kf_slots=ak + [S]), 1, "not pushed"),
           (dict(good_d, kf_slots=kf + [-1]), dict(good_c, kf_slots=ak + [-1]), 1, "not pushed"),
           (dict(good_d, lm_slots=lm + lm[:1]), dict(good_c, lm_slots=el + el[:1]), 1, "listed twice"),
           (dict(good_d, lm_slots=lm + [dr.n_lm]), dict(good_c, lm_slots=el + [dr.n_lm]), 1, "out of range"),
           (dict(good_d, lm_slots=list(range(dr.n_lm)) + [0]), dict(good_c, lm_slots=list(range(dr.n_lm)) + [0]), 4, "more keyframes"),
           (None, dict(good_c, cap=B - 1), 4, "cap below"), (None, dict(good_c, cap=-1), 1, "negative size"),
           (dict(good_d, kf_slots=[]), dict(good_c, kf_slots=[]), 1, "no keyframes")]
    L = capi.lib()

    def sentinel(res):
        for a in res:
            a.view(np.uint8)[:] = 0xA5
        return [a.copy() for a in res]

    for rd, rc_, code, msg in bad:
        for r, args, fn, gfn, Req, Out, good in ((rd, t._deactivate_request, L.kba_track_deactivate_keyframes,
                                                   L.kba_track_group_deactivate_keyframes, capi.KbaDeactivateRequest, capi.KbaDeactivateOut,
                                                   good_d),
                                                  (rc_, t._depth_request, L.kba_track_depth_costs, L.kba_track_group_depth_costs,
                                                   capi.KbaDepthRequest, capi.KbaDepthOut, good_c)):
            if r is None:
                continue
            q, o, (*res, _kf, _lm), _done = args(**r)
            before = sentinel(res)
            assert fn(t._p, C.byref(q), C.byref(o)) == code
            assert msg in L.kba_last_error().decode()
            assert all(np.array_equal(a, b) for a, b in zip(res, before))
            if not r["kf_slots"]:
                continue  # n_kf = 0 sits a group call out
            q0, o0, (*res0, _kf0, _lm0), _done0 = args(**good)
            before0 = sentinel(res0)
            reqs, outs = (Req * 2)(q0, q), (Out * 2)(o0, o)
            assert gfn(g._p, reqs, outs) == code
            assert re.search("track 1: .*" + msg, L.kba_last_error().decode())
            assert all(np.array_equal(a, b) for a, b in zip(res + res0, before + before0))
    for fn, args, good in ((L.kba_track_deactivate_keyframes, t._deactivate_request, good_d), (L.kba_track_depth_costs, t._depth_request, good_c)):
        q, o, _keep, _done = args(**good)
        o2 = type(o)()  # null output arrays
        assert fn(t._p, C.byref(q), C.byref(o2)) == 1
    for x in (t, other):
        _check_step(dr, st, x.deactivate_keyframes(**good_d), x.depth_costs(**good_c))
    g.close(); t.close(); other.close(); h.close()


@pytest.mark.gpu
def test_facade_device_upkeep_equals_facade(tmp_path):
    """tests/cpp/test_facade_upkeep: facade drives (two-camera and mono rigs, 12- and 20-keyframe windows, 30 pushes) mirrored
    into a track that creates its own landmarks; after every step the device deactivation equals the facade's
    active_keyframe_ids_ / active_landmark_ids_ and std::partial_sort over the device costs equals the AddDepth selection"""
    _build()
    for kw in DRIVES:
        path = tmp_path / "drive.txt"
        UpkeepDrive(**kw).write(path)
        r = subprocess.run([EXE, "device", str(path)], capture_output=True, text=True, timeout=1200)
        print(r.stdout)
        assert r.returncode == 0, r.stdout + r.stderr
