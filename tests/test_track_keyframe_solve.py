"""limo's solve block as one store call -- kba_track_keyframe_solve and its group forms -- against the chain of store calls it
replaces: deactivate_keyframes, the host's compaction and updateLabels, set_landmarks (shrubbery weights), rank_landmarks and
solve_ranked, exactly as the tests of those calls drive them.  Two copies of each store (Track.clone) go through the drives of
tests/upkeep_drive.py; after every keyframe step the outputs and the snapshots of the two stores must be equal byte for byte."""
import numpy as np
import pytest

from tests.test_track_rank import _same_result
from tests.test_track_upkeep import drive_steps
from tests.upkeep_drive import UpkeepDrive

VOX = dict(voxel_size=(0.5, 0.5, 0.3), roi_far=40.0, roi_middle=15.0)
OUTLIER, SHRUB, GROUND = 1, 2, 4
CLASSES = {1: OUTLIER, 2: SHRUB, 3: GROUND, 5: SHRUB | GROUND, 6: OUTLIER | GROUND}  # label 0 and 4: no class
SHRUB_W = 0.25


class Host:
    """a caller's bookkeeping of one track: the active keyframes and landmarks, the outlier set, the ground flags"""

    def __init__(self, dr):
        self.dr, self.S = dr, dr.window + 4
        self.kf, self.lm, self.outliers, self.done = [], set(), set(), set()
        self.ground = {lid: bool(g) for lid, g in enumerate(dr.ground)}
        self.pos = {st["k"]: st["pos"] for st in drive_steps(dr)}

    def push(self, tracks, k):
        """keyframe k into slot k % S of every copy, the positions created so far, and its landmarks into the active set"""
        dr = self.dr
        lm, cam, u, v, d = dr.arena(k)
        pos = self.pos.get(k, {})
        new = sorted(set(pos) - self.done)
        for t in tracks:
            if k >= self.S:
                t.drop_keyframe((k - self.S) % self.S)
            t.push_keyframe(k % self.S, dr.kf_pose[k], lm, u, v, d, cam=cam)
            if new:
                t.set_landmarks(new, pos=np.array([pos[i] for i in new]), weight=np.ones(len(new)))
        self.done |= set(new)
        self.kf.append(k)
        self.lm |= {lid for lid in dr.meas[k] if lid in self.done}
        for a in self.kf:
            self.lm |= {lid for lid in dr.meas[a] if lid in self.done}

    def request(self, rng, ground, step):
        """the keywords of a keyframe solve: the lists, this frame's tracklets and the ranking's and solve's keywords"""
        lm = sorted(self.lm)
        newest = sorted(self.dr.meas[self.kf[-1]])
        trk = []
        for lid in newest:
            if rng.random() < 0.6:
                label = int(rng.choice([0, 1, 2, 3, 4, 5, 6], p=[0.4, 0.08, 0.15, 0.2, 0.05, 0.07, 0.05]))
                trk.append((lid if lid in self.done else -1, label, int(rng.random() < 0.03)))
        trk.append((-1, 1, 1))  # an id without a slot
        small = step % 4 == 1  # a selection below the trimming threshold
        caps = dict(max_near=3, max_middle=2, max_far=3) if small else dict(max_near=int(rng.choice([40, 300])), max_middle=30, max_far=80)
        depth = [(i, 2 if small else 40) for i in range(0, self.dr.window + 1, 3)]
        scal = dict(scale_weight=-1.0, scale_value=1.5)
        if ground:
            scal.update(ground=True, plane_reg_weight=-1.0)
        return dict(kf_slots=[a % self.S for a in self.kf], lm_slots=lm, min_connecting=3, min_window=4, max_window=self.dr.window,
                    lm_ground=[self.ground[i] for i in lm], tracklets=trk, label_classes=CLASSES, outliers=sorted(self.outliers),
                    shrubbery_weight=SHRUB_W, depth=depth, draws=rng.integers(0, 2**31 - 1, len(lm) + 1), **caps, **VOX, **scal)

    def chain(self, t, r, opt):
        """the chain of store calls a caller runs today on track t for request r, with the facade's updateLabels on the host"""
        kf_active, kf_common, lm_active = t.deactivate_keyframes(r["kf_slots"], r["lm_slots"], r["min_connecting"], r["min_window"],
                                                                 r["max_window"])
        kf = [s for s, f in zip(r["kf_slots"], kf_active) if f]
        active = {s for s, f in zip(r["lm_slots"], lm_active) if f}
        outl = {s for s in r["outliers"] if s in active}
        ground = dict(zip(r["lm_slots"], [bool(g) for g in r["lm_ground"]]))
        shrub = []
        for slot, label, iso in r["tracklets"]:
            c = CLASSES.get(label, 0)
            if slot >= 0 and (iso or c & OUTLIER):
                outl.add(slot)
            if slot < 0 or slot not in active:
                continue
            if c & SHRUB:
                shrub.append(slot)
            ground[slot] = bool(c & GROUND)
        if shrub:
            t.set_landmarks(shrub, weight=np.full(len(shrub), r["shrubbery_weight"]))
        cand = [s for s in r["lm_slots"] if s in active and s not in outl]
        elig = np.array([ground[s] for s in cand], np.uint8)
        keys = ("max_near", "max_middle", "max_far", "depth", "draws", *VOX)
        rk = t.rank_landmarks(kf, cand, elig=elig, **{k: r[k] for k in keys})
        fixed = np.r_[[1], np.zeros(len(kf) - 1)].astype(np.uint8)
        scal = {k: r[k] for k in ("scale_weight", "scale_value", "ground", "plane_reg_weight") if k in r}
        res = t.solve_ranked(kf, fixed, opt=opt, **scal)
        trk_out = [int(iso or bool(CLASSES.get(label, 0) & OUTLIER) or (slot >= 0 and slot in outl and slot in ground))
                   for slot, label, iso in r["tracklets"]]
        return dict(kf_active=kf_active, kf_common=kf_common, lm_active=lm_active,
                    lm_outlier=np.array([s in outl for s in r["lm_slots"]], np.uint8),
                    lm_ground=np.array([ground[s] for s in r["lm_slots"]], np.uint8), trk_outlier=np.array(trk_out, np.uint8),
                    result=res, shrub=shrub, outl=outl, ground=ground, **rk)

    def advance(self, r, out):
        """the bookkeeping after a solve block, from the call's outputs"""
        self.kf = [a for a, f in zip(self.kf, out["kf_active"]) if f]
        self.lm = {s for s, f in zip(r["lm_slots"], out["lm_active"]) if f}
        self.outliers = {s for s, f in zip(r["lm_slots"], out["lm_outlier"]) if f}
        self.outliers |= {slot for (slot, _l, _o), f in zip(r["tracklets"], out["trk_outlier"]) if f and slot >= 0}
        for s, g in zip(r["lm_slots"], out["lm_ground"]):
            self.ground[s] = bool(g)


def _same(one, ref, where):
    for key in ("kf_active", "kf_common", "lm_active", "lm_outlier", "lm_ground", "trk_outlier", "cand", "category"):
        assert np.array_equal(np.asarray(one[key]), np.asarray(ref[key])), (where, key)
    assert (one["n_ground"], one["n_draws"]) == (ref["n_ground"], ref["n_draws"]), where
    _same_result(one["result"], ref["result"])


def _track(h, dr, ground, win_rows=0):
    from limo_b200 import capi
    n_meas = sum(len(o) for m in dr.meas for o in m.values())
    return capi.Track(h, dr.cam_intr, dr.cam_pose, max_keyframes=dr.window + 4, max_landmarks=dr.n_lm, max_measurements=n_meas,
                      win_keyframes=min(dr.window + 2, 30), win_landmarks=dr.n_lm, win_observations=n_meas,
                      win_ground=dr.n_lm if ground else 0, win_rows=win_rows)


def _options():
    from limo_b200 import capi
    opt = capi.default_options()
    opt.solver_time_sec = 0.0  # no time limit: both copies run the same iterations
    return opt


CONFIGS = [dict(seed=1, window=12, rig=False, ground=False, win_rows=0), dict(seed=2, window=12, rig=True, ground=True, win_rows=0),
           dict(seed=3, window=20, rig=False, ground=True, win_rows=201)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: "w%d_%s_%s" % (c["window"], "rig" if c["rig"] else "mono",
                                                                       "ground" if c["ground"] else "plain"))
def test_keyframe_solve_equals_the_chain(cfg):
    from limo_b200 import capi
    dr = UpkeepDrive(cfg["seed"], n_push=34, window=cfg["window"], rig=cfg["rig"], new_per_push=40)
    h = capi.Handle(0)
    a = _track(h, dr, cfg["ground"], cfg["win_rows"])
    b = a.clone()
    host = Host(dr)
    rng = np.random.default_rng(cfg["seed"])
    opt = _options()
    seen = dict(deactivated=0, trimmed=0, untrimmed=0, shrub=0, ground=0, outlier=0, left=0, large=0)
    for k in range(dr.n_push):
        host.push([a, b], k)
        if k < 3:
            continue
        r = host.request(rng, cfg["ground"], k)
        ref = host.chain(a, r, opt)
        one = b.keyframe_solve(opt=opt, **r)
        _same(one, ref, k)
        assert bytes(a.snapshot()) == bytes(b.snapshot()), k
        h2d, d2h, _ = b.transfer_bytes()
        assert h2d > 0 and d2h > 0
        n_kept = int(one["kf_active"].sum())
        seen["deactivated"] += int(n_kept < len(r["kf_slots"]))
        seen["trimmed" if len(one["cand"]) > 100 else "untrimmed"] += int(one["result"].c.num_solves > 0)
        seen["shrub"] += len(ref["shrub"])
        seen["ground"] += int(one["n_ground"] > 0)
        seen["outlier"] += int(one["lm_outlier"].sum())
        # outliers whose landmarks this deactivation removed: they leave the set
        seen["left"] += len(set(r["outliers"]) - {s for s, f in zip(r["lm_slots"], one["lm_active"]) if f})
        # the solve's reduced rows as track_check counts them: plane blocks iff ground candidates were attached (the ranking's
        # n_ground; plane_reg_weight -1 is not > 0); above 184 rows the solve runs on the large-window solver
        rows = (10 if one["n_ground"] > 0 and cfg["ground"] else 6) * n_kept + 1
        seen["large"] += int(rows > 184)
        host.advance(r, one)
    need = ["deactivated", "trimmed", "untrimmed", "shrub", "outlier", "left"] + (["ground"] if cfg["ground"] else [])
    need += ["large"] if cfg["win_rows"] else []
    assert all(seen[n] > 0 for n in need), seen
    a.close(); b.close(); h.close()


@pytest.mark.gpu
def test_group_keyframe_solve_equals_single_calls():
    """a group of 8 mono tracks of different stores, one request sitting out per step, per-track options: every track's outputs
    and snapshot equal its single call's on a clone"""
    from limo_b200 import capi
    h = capi.Handle(0)
    drs = [UpkeepDrive(50 + i, n_push=14, window=6 + (i % 3), rig=False, new_per_push=25 + 5 * i) for i in range(8)]
    gt = [_track(h, dr, False) for dr in drs]
    st = [t.clone() for t in gt]
    g = capi.TrackGroup(h, gt)
    hosts = [Host(dr) for dr in drs]
    rng = np.random.default_rng(7)
    opts = [_options() for _ in drs]
    for i, o in enumerate(opts):
        o.reprojection_thres = 1.2 + 0.1 * i
    for k in range(14):
        for i, host in enumerate(hosts):
            host.push([gt[i], st[i]], k)
        if k < 3:
            continue
        reqs = [None if i == k % 8 else hosts[i].request(rng, False, k) for i in range(8)]
        outs = g.keyframe_solve(reqs, opt=opts)
        assert outs[k % 8] is None
        for i, r in enumerate(reqs):
            if r is None:
                continue
            one = st[i].keyframe_solve(opt=opts[i], **r)
            _same(outs[i], one, (k, i))
            hosts[i].advance(r, one)
        snaps_g, snaps_s = g.snapshot(), [t.snapshot() for t in st]
        for i in range(8):
            assert bytes(snaps_g[i]) == bytes(snaps_s[i]), (k, i)
    g.close()
    for t in gt + st:
        t.close()
    h.close()


@pytest.mark.gpu
def test_refused_requests_write_nothing():
    """a malformed slot, capacity overflows, too few keyframes after the deactivation and a failing draw function: each call
    fails with the underlying call's code and message, writes no output, and leaves the store's snapshot as it was"""
    from limo_b200 import capi
    dr = UpkeepDrive(9, n_push=10, window=8, rig=False, new_per_push=40)
    h = capi.Handle(0)
    t = _track(h, dr, False)
    host = Host(dr)
    rng = np.random.default_rng(9)
    for k in range(8):
        host.push([t], k)
        if k >= 3:
            r = host.request(rng, False, k)
            host.advance(r, t.keyframe_solve(opt=_options(), **r))
    host.push([t], 8)
    base = host.request(rng, False, 8)
    base["tracklets"] = [(s, 2, 0) for s in sorted(host.lm)[:20]]  # shrubbery on active landmarks: a refused call writes no weight
    before = bytes(t.snapshot())
    bad_slot = [list(base["kf_slots"]) + [base["kf_slots"][-1]], base["tracklets"] + [(dr.n_lm, 0, 0)]]
    cases = [(dict(kf_slots=bad_slot[0]), 1, "listed twice"), (dict(tracklets=bad_slot[1]), 1, "tracklet landmark slot"),
             (dict(depth=[(0, 1)] * 1025), 4, "1024"), (dict(max_window=2), 3, "fewer than 3 keyframes"),
             (dict(draws=np.zeros(0, np.int64), max_middle=300), 1, "draw function failed")]
    for kw, code, msg in cases:
        q, o, keep, _done, rc = t._keyframe_solve_request(256, **dict(base, **kw))
        for arr in keep[:8]:
            arr[...] = 7
        o.rank.n_sel = o.rank.n_ground = o.rank.n_draws = -7
        got = capi.lib().kba_track_keyframe_solve(t._p, q, _options(), o, rc)
        assert got == code, (kw.keys(), got, capi.lib().kba_last_error())
        assert msg in capi.lib().kba_last_error().decode(), msg
        assert all((arr == 7).all() for arr in keep[:8]), msg
        assert (o.rank.n_sel, o.rank.n_ground, o.rank.n_draws) == (-7, -7, -7), msg
        assert bytes(t.snapshot()) == before, msg
    t.keyframe_solve(opt=_options(), **base)  # the request itself is fine
    assert bytes(t.snapshot()) != before
    t.close(); h.close()


@pytest.mark.gpu
def test_group_refusal_writes_nothing():
    """a group of three (track 1 sitting out) in which track 2's draw function fails, then one in which track 0's tracklet slot is
    out of range: each call names the failing track, writes no output of any track and leaves every snapshot as it was"""
    from limo_b200 import capi
    h = capi.Handle(0)
    drs = [UpkeepDrive(60 + i, n_push=9, window=6, rig=False, new_per_push=40) for i in range(3)]
    ts = [_track(h, dr, False) for dr in drs]
    g = capi.TrackGroup(h, ts)
    hosts = [Host(dr) for dr in drs]
    rng = np.random.default_rng(3)
    for k in range(8):
        for i in range(3):
            hosts[i].push([ts[i]], k)
        if k >= 3:
            reqs = [hosts[i].request(rng, False, k) for i in range(3)]
            for i, o in enumerate(g.keyframe_solve(reqs, opt=_options())):
                hosts[i].advance(reqs[i], o)
    for i in range(3):
        hosts[i].push([ts[i]], 8)
    base = []
    for i in range(3):
        r = hosts[i].request(rng, False, 8)
        r.update(tracklets=[(s, 2, 0) for s in sorted(hosts[i].lm)[:20]], max_middle=300)
        base.append(r)
    before = [bytes(b) for b in g.snapshot()]
    bad_draws = dict(draws=np.zeros(0, np.int64))
    bad_slot = dict(tracklets=base[0]["tracklets"] + [(drs[0].n_lm, 0, 0)])
    for fix, track, msg in (({2: bad_draws}, 2, "draw function failed"), ({0: bad_slot}, 0, "tracklet landmark slot")):
        reqs, outs, ress = (capi.KbaKfsolveRequest * 3)(), (capi.KbaKfsolveOut * 3)(), (capi.KbaResult * 3)()
        keep = []
        for i in (0, 2):
            q, o, k, _done, rc = ts[i]._keyframe_solve_request(256, **dict(base[i], **fix.get(i, {})))
            for arr in k[:8]:
                arr[...] = 7
            o.rank.n_sel = o.rank.n_ground = o.rank.n_draws = -7
            reqs[i], outs[i], ress[i] = q, o, rc
            keep.append(k)
        outs[1].rank.n_sel = -7
        got = capi.lib().kba_track_group_keyframe_solve(g._p, reqs, _options(), outs, ress)
        err = capi.lib().kba_last_error().decode()
        assert got == 1 and "kba_track_group_keyframe_solve" in err and "track %d: " % track in err and msg in err, err
        for k in keep:
            assert all((arr == 7).all() for arr in k[:8]), msg
        assert all(outs[i].rank.n_sel == -7 for i in range(3)), msg
        assert [bytes(b) for b in g.snapshot()] == before, msg
    g.close()
    for t in ts:
        t.close()
    h.close()
