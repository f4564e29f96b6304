"""Snapshots of the device-resident store (kba_track_save / kba_track_load / kba_track_clone / kba_track_group_save).

Without a GPU: the header struct against its ctypes mirror, the exported symbols, and capi_types.parse_snapshot on a hand-built
buffer, malformed ones included.
On the GPU, with the drives of tests/test_track_group_store.py and tests/test_track_group.py:
  - continuation: a track saved in the middle of a drive and loaded on a fresh handle gives, at every later step, the source's
    outputs bit for bit through every store call, and the same final snapshot;
  - canonical form: a compacting arena and one that never compacts, group and single writes, give the same bytes; a fresh
    track's landmarks are zero;
  - a save changes nothing (a ranking made before it is solved after it), a clone is load(save(src)) and independent of src;
  - caps at load, group saves, corrupted input, and a load on a second device when one is visible."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_track_group import PLANE, _Drive
from tests.test_track_group_store import _same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPS_AT = 16   # byte offset of kba_snapshot_header.caps


# ---- CPU --------------------------------------------------------------------------------------------------------------------------
def test_snapshot_header_matches_ctypes_mirror(tmp_path):
    """sizeof(kba_snapshot_header) and every field offset as gcc compiles them == the ctypes mirror's"""
    from limo_b200 import capi_types as T
    fields = [f for f, _ in T.KbaSnapshotHeader._fields_]
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "kba_b200.h"\nint main(){printf("%zu' + ' %zu' * len(fields) +
                    '\\n",sizeof(kba_snapshot_header)' + "".join(",offsetof(kba_snapshot_header,%s)" % f for f in fields) +
                    ');return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(T.KbaSnapshotHeader)] + [getattr(T.KbaSnapshotHeader, f).offset for f in fields]
    assert T.KbaSnapshotHeader.caps.offset == CAPS_AT and C.sizeof(T.KbaSnapshotHeader) == 128


def test_snapshot_symbols_exported():
    from limo_b200 import capi
    L = capi.lib()
    for n in ("kba_track_snapshot_size", "kba_track_save", "kba_track_load", "kba_track_clone", "kba_track_group_snapshot_sizes",
              "kba_track_group_save"):
        assert n in capi.SYMBOLS and hasattr(L, n), n


def _hand_built():
    """a two-camera snapshot of 3 live keyframes (slots 0, 2, 5; counts 2, 0, 3) and 4 landmark slots, built from the format's
    statement in include/kba_b200.h"""
    from limo_b200 import capi_types as T
    n_cam, slot, cnt, L = 2, [0, 2, 5], [2, 0, 3], 4
    K, M = len(slot), sum(cnt)
    a8 = lambda b: (b + 7) // 8 * 8  # noqa: E731
    hd = T.KbaSnapshotHeader(magic=T.SNAPSHOT_MAGIC, format_version=1, writer_version=4, n_cam=n_cam,
                             caps=T.KbaTrackCaps(8, L, 16, 4, 4, 16, 0, 0), n_keyframes=K, n_entries=M, lm_cap=L)
    parts = [bytes(hd)]
    cam = np.arange(10 * n_cam, dtype=np.float64)
    parts.append(cam.tobytes())
    for a in (np.array(slot, np.int32), np.array(cnt, np.int32)):
        parts.append(a.tobytes() + b"\0" * (a8(4 * K) - 4 * K))
    parts += [np.arange(7 * K, dtype=np.float64).tobytes(), np.arange(4 * K, dtype=np.float64).tobytes()]
    cols = [np.array([0, 3, 1, 1, 2], np.int32), np.array([0, 1, 1, 0, 1], np.int32)] + [np.arange(M, dtype=np.float32) + q for q in range(3)]
    for c in cols:
        parts.append(c.tobytes() + b"\0" * (a8(4 * M) - 4 * M))
    parts += [np.arange(3 * L, dtype=np.float64).tobytes(), np.ones(L).tobytes()]
    o = [C.sizeof(hd), C.sizeof(hd) + 80 * n_cam]
    o.append(o[1] + 2 * a8(4 * K) + 88 * K)
    o.append(o[2] + 5 * a8(4 * M))
    hd.cam_offset, hd.cam_bytes, hd.kf_offset, hd.kf_bytes = o[0], o[1] - o[0], o[1], o[2] - o[1]
    hd.meas_offset, hd.meas_bytes, hd.lm_offset, hd.lm_bytes = o[2], o[3] - o[2], o[3], 32 * L
    parts[0] = bytes(hd)
    return bytearray(b"".join(parts))


def test_parse_snapshot_reads_a_hand_built_buffer():
    from limo_b200 import capi_types as T
    s = T.parse_snapshot(np.frombuffer(bytes(_hand_built()), np.uint8))
    assert s["header"].n_cam == 2 and s["cam_intr"].shape == (2, 3) and s["cam_pose"][1, 6] == 19.0
    assert s["slot"].tolist() == [0, 2, 5] and s["count"].tolist() == [2, 0, 3]
    assert s["pose"].shape == (3, 7) and s["plane"][2, 3] == 11.0
    assert s["lm"].tolist() == [0, 3, 1, 1, 2] and s["cam"].tolist() == [0, 1, 1, 0, 1] and s["d"][4] == 6.0
    assert s["pos"].shape == (4, 3) and s["weight"].tolist() == [1.0] * 4


def test_parse_snapshot_rejects_malformed_buffers():
    from limo_b200 import capi_types as T
    good = _hand_built()
    hd = T.KbaSnapshotHeader.from_buffer_copy(bytes(good[:128]))

    def with_header(**kw):
        h = T.KbaSnapshotHeader.from_buffer_copy(bytes(hd))
        for k, v in kw.items():
            setattr(h, k, v)
        b = bytearray(good)
        b[:128] = bytes(h)
        return b

    def poke(off, dtype, value):
        b = bytearray(good)
        b[off:off + np.dtype(dtype).itemsize] = np.array([value], dtype).tobytes()
        return b
    cases = [(with_header(magic=0x12345678), "magic"), (with_header(format_version=2), "format_version"),
             (good[:-8], "truncated"), (good[:100], "truncated"), (with_header(meas_bytes=hd.meas_bytes + 8), "meas_bytes"),
             (with_header(n_entries=4), "cam_bytes|kf_bytes|meas_offset|meas_bytes|lm_offset"),
             (poke(hd.kf_offset + 4, np.int32, 9), "slots"), (poke(hd.kf_offset + 4, np.int32, 0), "slots"),
             (poke(hd.kf_offset + 16 + 4, np.int32, 1), "counts"), (poke(hd.meas_offset, np.int32, 4), "landmark slot"),
             (poke(hd.meas_offset + 24, np.int32, 2), "camera")]
    for buf, what in cases:
        with pytest.raises(ValueError, match=what):
            T.parse_snapshot(bytes(buf))


def test_snapshot_bench_dry_run():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "snapshot_bench.py"), "--dry-run"], capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr
    assert '"dry_run": true' in out.stdout


# ---- GPU: the drive ----------------------------------------------------------------------------------------------------------
class _Run:
    """a track of a _Drive (keyframe k in slot k % (W + 1)) and the keyframe step applied to it: drop, push, then every store
    call on the window (frame flow, selection, creation, upkeep, depth costs, pose-only tracking, reclaim with the freed slots
    written again, a solve, a ranking and its solve).  Outputs are returned for comparison; the solve's poses feed the host's
    mirror once per step (record)."""

    def __init__(self, seed, W=6, steps=12, rig=False, ground=False, mono_cam=False, tight=False, device_gp=False, win_rows=0):
        self.W, self.steps, self.mono_cam, self.device_gp, self.win_rows = W, steps, mono_cam, device_gp, win_rows
        self.d = _Drive(seed=seed, W=W, n_lm=500, n_obs=(W + steps) * 160, config=3 if ground else 2, rig=rig, ground=ground,
                        steps=steps)
        c = self.d.counts()
        self.m_cap = max(sum(c[s:s + W + 1]) for s in range(len(c) - W)) + 8 if tight else 2 * sum(c)

    def make(self, h, **caps):
        from limo_b200 import capi
        d = self.d
        kw = dict(max_keyframes=self.W + 1, max_landmarks=d.win.n_lm, max_measurements=self.m_cap, win_keyframes=self.W,
                  win_landmarks=d.win.n_lm, win_observations=d.window_obs()[0], win_ground=len(d.gp) if d.ground else 0,
                  win_rows=self.win_rows)
        kw.update(caps)
        t = capi.Track(h, d.cam_intr, d.cam_pose, **kw)
        t.set_landmarks(np.arange(d.win.n_lm, dtype=np.int32), pos=d.win.lm_pos, weight=d.win.lm_weight)
        for k in range(self.W):
            t.push_keyframe(**self.push_args(k))
        return t

    def push_args(self, k):
        lm, u, v, d, cam = self.d.measurements(k)
        o = np.lexsort((cam, lm))
        return dict(slot=k % (self.W + 1), pose7=self.d.win.kf_pose[k], lm_slot=lm[o], u=u[o], v=v[o], d=d[o],
                    cam=None if self.mono_cam else cam[o], plane4=PLANE if self.d.ground else None)

    def request(self, s):
        req = self.d.request(s)
        if self.device_gp and "gp_lm" in req:  # every ground landmark of the window a candidate, attached on the device
            gi = np.array([i for i, j in enumerate(req["lm_slots"]) if int(j) in self.d.gp], np.int32)
            for k in ("gp_kf", "gp_weight"):
                req.pop(k)
            req.update(gp_lm=gi, plane_reg_weight=-1.0)
        return req

    def step(self, t, s, req):
        """step s >= 1 of the drive on track t, with the solve request req of the step; returns every output"""
        from limo_b200 import capi
        W, d = self.W, self.d
        k = W - 1 + s
        if k >= W + 1:
            t.drop_keyframe(k % (W + 1))
        t.push_keyframe(**self.push_args(k))
        slots = [j % (W + 1) for j in range(s, k + 1)]
        lms = np.unique(np.concatenate([d.per_kf[j][0] for j in range(s, k + 1)])).astype(np.int32)
        nxt = min(k + 1, d.n_kf - 1)
        lm, u, v, dd, cam = d.measurements(nxt)
        o = np.lexsort((cam, lm))
        out = dict(flow=t.frame_flow(k % (W + 1), lm[o], u[o], v[o], cam=cam[o]), sel=t.select_landmarks(slots, lms),
                   deact=t.deactivate_keyframes(slots, lms), depth=t.depth_costs(slots, lms))
        opt = capi.default_options()
        opt.solver_time_sec = 20.0
        out["pose"] = t.adjust_pose(d.win.kf_pose[nxt], lm[o], u[o], v[o], dd[o], cam=cam[o], opt=opt)
        out["solve"] = t.solve(opt=opt, **req)
        out["rank"] = t.rank_landmarks(slots, lms, draws=lambda n: (np.arange(n) * 7919) % 1000003)
        fixed = np.zeros(len(slots), np.uint8)
        fixed[:2] = 1
        out["ranked"] = t.solve_ranked(slots, fixed, opt=opt)
        out["create"] = t.create_landmarks(slots, len(slots) - 1, np.unique(d.per_kf[k][0])[:60])
        free, pos, wt = t.reclaim_landmarks(0, d.win.n_lm, evict=True)
        out["reclaim"] = (free, pos, wt)
        if len(free):  # a caller hands freed slots out again
            t.set_landmarks(free[:8], pos=pos[:8] + 0.5, weight=np.full(min(8, len(free)), 0.9))
        return out


def _res(r):
    return dict(status=r.c.status, iters=[s.num_iterations for s in r.solves], kf_pose=r.kf_pose, kf_plane=r.kf_plane,
                lm_pos=r.lm_pos, lm_rejected=r.lm_rejected, cost=(r.c.initial_cost, r.c.final_cost))


def _comparable(out):
    return {k: _res(v) if hasattr(v, "solves") else v for k, v in out.items()}


def _continue(run, pairs, s0, s1):
    """steps s0 .. s1 - 1 on every (source, copy) pair (copy None: the source alone): outputs bit-identical at every step"""
    for s in range(s0, s1):
        req = run.request(s)
        outs = [(run.step(a, s, req), b and run.step(b, s, req)) for a, b in pairs]
        for i, (oa, ob) in enumerate(outs):
            if ob is not None:
                _same(_comparable(oa), _comparable(ob), "step %d pair %d" % (s, i))
        assert outs[0][0]["solve"].c.status == 0
        run.d.record(outs[0][0]["solve"])


def _bytes_equal(a, b, what, skip_caps=False):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, what
    if skip_caps:
        a, b = a.copy(), b.copy()
        a[CAPS_AT:CAPS_AT + 32] = b[CAPS_AT:CAPS_AT + 32] = 0
    assert a.tobytes() == b.tobytes(), what


RUNS = dict(mono=dict(seed=71), rig=dict(seed=72, rig=True), compacting=dict(seed=74, mono_cam=True, tight=True),
            ground_large=dict(seed=73, ground=True, device_gp=True, win_rows=301))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(RUNS))
def test_loaded_track_continues_bit_identically(kind):
    """save at the middle step, load on a fresh handle, continue both: every output bit-identical, the final snapshots equal"""
    from limo_b200 import capi
    run = _Run(**RUNS[kind])
    h, h2 = capi.Handle(0), capi.Handle(0)
    src = run.make(h)
    mid = run.steps // 2
    _continue(run, [(src, None)], 1, mid)
    snap = src.snapshot()
    dst = capi.Track.load(h2, snap)
    _bytes_equal(dst.snapshot(), snap, "loaded track's snapshot")
    _continue(run, [(src, dst)], mid, run.steps)
    _bytes_equal(dst.snapshot(), src.snapshot(), "final snapshots")
    if kind == "compacting":
        assert src.snapshot()[CAPS_AT + 8:CAPS_AT + 12].view(np.int32)[0] == run.m_cap
    for t in (src, dst):
        t.close()
    h.close()
    h2.close()


@pytest.mark.gpu
def test_large_window_ground_track_continues_after_a_load():
    """a 20-keyframe ground-plane window (201 reduced rows, the large-window solver of a win_rows = 301 track) with device
    attachment: loaded mid-drive, the copy solves bit-identically"""
    from limo_b200 import capi
    run = _Run(seed=75, W=20, steps=4, ground=True, device_gp=True, win_rows=301)
    h = capi.Handle(0)
    src = run.make(h)
    _continue(run, [(src, None)], 1, 2)
    dst = capi.Track.load(h, src.snapshot())
    _continue(run, [(src, dst)], 2, run.steps)
    _bytes_equal(dst.snapshot(), src.snapshot(), "final snapshots")
    for t in (src, dst):
        t.close()
    h.close()


@pytest.mark.gpu
def test_snapshots_are_canonical():
    """a compacting arena and one that never compacts, and group and single writes, give the same bytes; a fresh track's
    landmark section is zero"""
    from limo_b200 import capi
    from limo_b200 import capi_types as T
    h = capi.Handle(0)
    run = _Run(seed=74, mono_cam=True, tight=True, steps=14)
    tight, roomy = run.make(h), run.make(h, max_measurements=4 * sum(run.d.counts()))
    ga_t = [run.make(h) for _ in range(2)]
    ga = capi.TrackGroup(h, ga_t)
    for s in range(1, run.steps):
        k = run.W - 1 + s
        drop = k % (run.W + 1) if k >= run.W + 1 else None
        for t in (tight, roomy):
            if drop is not None:
                t.drop_keyframe(drop)
            t.push_keyframe(**run.push_args(k))
        ga.drop_keyframes([drop, drop])
        ga.push_keyframes([run.push_args(k), run.push_args(k)])
        wr = dict(lm_slot=np.arange(s, 400, 37, dtype=np.int32), pos=np.full((len(range(s, 400, 37)), 3), 0.1 * s), weight=None)
        tight.set_landmarks(**wr)
        roomy.set_landmarks(**wr)
        ga.set_landmarks([wr, wr])
        sa, sb = tight.snapshot(), roomy.snapshot()
        _bytes_equal(sa, sb, "step %d: compacting against never compacting" % s, skip_caps=True)
        g = ga.snapshot()
        _bytes_equal(g[0], sa, "step %d: group writes against single writes" % s)
        _bytes_equal(g[1], sa, "step %d: group writes against single writes" % s)
    caps = dict(max_measurements=4 * sum(run.d.counts()))
    _bytes_equal(capi.Track.load(h, tight.snapshot(), caps).snapshot(), roomy.snapshot(), "loaded with the same caps")
    fresh = capi.Track(h, run.d.cam_intr, run.d.cam_pose, max_keyframes=4, max_landmarks=1000, max_measurements=10, win_keyframes=3,
                       win_landmarks=10, win_observations=10)
    p = T.parse_snapshot(fresh.snapshot())
    assert len(p["slot"]) == 0 and not p["pos"].any() and not p["weight"].any()
    assert p["header"].writer_version == capi.lib().kba_version() >= 4
    ga.close()
    for t in [tight, roomy, fresh] + ga_t:
        t.close()
    h.close()


@pytest.mark.gpu
def test_save_changes_nothing():
    """rank, save, solve_ranked: accepted, and equal to rank, solve_ranked on a twin that was not saved"""
    from limo_b200 import capi
    run = _Run(seed=72, rig=True)
    h = capi.Handle(0)
    a, b = run.make(h), run.make(h)
    slots = list(range(run.W))
    lms = np.unique(np.concatenate([run.d.per_kf[j][0] for j in range(run.W)])).astype(np.int32)
    fixed = np.r_[1, 1, np.zeros(run.W - 2)].astype(np.uint8)
    for t in (a, b):
        t.rank_landmarks(slots, lms, draws=lambda n: np.arange(n))
    snap = a.snapshot()
    ra, rb = a.solve_ranked(slots, fixed), b.solve_ranked(slots, fixed)
    _same(_res(ra), _res(rb), "solve_ranked after a save")
    assert ra.c.status == 0
    assert a.snapshot().tobytes() != snap.tobytes()  # the solve wrote the store
    _bytes_equal(a.snapshot(), b.snapshot(), "stores after the solve")
    for t in (a, b):
        t.close()
    h.close()


@pytest.mark.gpu
def test_clone_is_load_of_save_and_independent():
    from limo_b200 import capi
    run = _Run(seed=73, ground=True)
    h, h2 = capi.Handle(0), capi.Handle(0)
    src = run.make(h)
    _continue(run, [(src, None)], 1, 3)
    snap = src.snapshot()
    for hh in (h, h2):
        c = src.clone(hh)
        _bytes_equal(c.snapshot(), capi.Track.load(hh, snap).snapshot(), "clone on %s handle" % ("the same" if hh is h else "a second"))
        c.close()
    c = src.clone(h2)
    c.set_landmarks([0, 1], pos=[[1.0, 2.0, 3.0]] * 2, weight=[0.25, 0.5])
    c.drop_keyframe(2)
    _bytes_equal(src.snapshot(), snap, "source after writes to its clone")
    c_snap = c.snapshot()
    src.set_keyframe_poses([1], [run.d.win.kf_pose[1] + np.r_[0, 0, 0, 0, 0.5, 0, 0]])
    _bytes_equal(c.snapshot(), c_snap, "clone after writes to its source")
    assert c_snap.tobytes() != snap.tobytes()
    for t in (src, c):
        t.close()
    h.close()
    h2.close()


@pytest.mark.gpu
def test_caps_at_load():
    """larger caps continue bit-identically on the windows both hold; caps that cannot hold the content are KBA_ERR_CAPACITY"""
    from limo_b200 import capi
    run = _Run(seed=71, steps=8)
    h = capi.Handle(0)
    src = run.make(h)
    _continue(run, [(src, None)], 1, 3)
    snap = src.snapshot()
    n_lm = run.d.win.n_lm
    big = capi.Track.load(h, snap, dict(win_keyframes=run.W + 8, max_landmarks=2 * n_lm, max_keyframes=run.W + 3))
    from limo_b200 import capi_types as T
    p, q = T.parse_snapshot(big.snapshot()), T.parse_snapshot(snap)
    assert p["header"].caps.win_keyframes == run.W + 8 and p["header"].lm_cap == 2 * n_lm
    assert np.array_equal(p["pos"][:n_lm], q["pos"]) and not p["pos"][n_lm:].any() and np.array_equal(p["lm"], q["lm"])
    _continue(run, [(src, big)], 3, run.steps)
    for caps, what in [(dict(max_landmarks=n_lm - 1), "max_landmarks"), (dict(max_measurements=10), "max_measurements"),
                       (dict(max_keyframes=3), "max_keyframes")]:
        with pytest.raises(capi.KbaError, match="error 4: kba_track_load: caps.%s" % what):
            capi.Track.load(h, snap, caps)
        with pytest.raises(capi.KbaError, match="error 4: kba_track_clone: caps.%s" % what):
            src.clone(**caps)
    for t in (src, big):
        t.close()
    h.close()


@pytest.mark.gpu
def test_group_save():
    """each buffer equals the single save; a NULL buffer sits out; a too-small buffer fails naming its track, nothing written"""
    from limo_b200 import capi
    h = capi.Handle(0)
    runs = [_Run(seed=71), _Run(seed=72, rig=True), _Run(seed=73, ground=True)]
    ts = [r.make(h) for r in runs]
    g = capi.TrackGroup(h, ts)
    snaps = g.snapshot()
    for t, s in zip(ts, snaps):
        _bytes_equal(s, t.snapshot(), "group save against the single save")
    part = g.snapshot(which=[0, 2])
    assert part[1] is None
    _bytes_equal(part[2], snaps[2], "track 2 with track 1 sitting out")
    assert g.transfer_bytes()[1] == len(snaps[0]) + len(snaps[2])
    L = capi.lib()
    bufs = [np.full(len(s) + 8, 0xAB, np.uint8) for s in snaps]
    sizes = np.array([len(s) + 8 for s in snaps], np.int64)
    sizes[1] = len(snaps[1]) - 1
    ptrs = (C.c_void_p * 3)(*[b.ctypes.data for b in bufs])
    assert L.kba_track_group_save(g._p, ptrs, sizes.ctypes.data_as(C.POINTER(C.c_int64))) == 4
    assert "kba_track_group_save: track 1: " in L.kba_last_error().decode()
    assert all((b == 0xAB).all() for b in bufs)
    g.close()
    for t in ts:
        t.close()
    h.close()


@pytest.mark.gpu
def test_corrupted_snapshot_is_refused():
    from limo_b200 import capi
    from limo_b200 import capi_types as T
    run = _Run(seed=72, rig=True)
    h = capi.Handle(0)
    src = run.make(h)
    snap = src.snapshot()
    hd = T.parse_snapshot(snap)["header"]
    flipped = snap.copy()
    flipped[hd.kf_offset:hd.kf_offset + 8] = np.frombuffer(snap[hd.kf_offset:hd.kf_offset + 8].tobytes(), np.int32)[::-1].copy().view(np.uint8)
    bad_cam = snap.copy()
    bad_cam[hd.meas_offset + hd.meas_bytes // 5 + 12:][:4] = np.array([2], np.int32).view(np.uint8)
    version = snap.copy()
    version[4:8] = np.array([2], np.uint32).view(np.uint8)
    for buf, what in [(flipped, "keyframe slot"), (bad_cam, "camera"), (snap[:-1], "truncated"), (snap[:64], "truncated"),
                      (version, "format_version")]:
        with pytest.raises(capi.KbaError, match="error 1: kba_track_load: .*%s" % what):
            capi.Track.load(h, buf)
    src.close()
    h.close()


@pytest.mark.gpu
def test_load_on_a_second_device():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    from limo_b200 import capi
    run = _Run(seed=72, rig=True, steps=8)
    h0, h1 = capi.Handle(0), capi.Handle(1)
    src = run.make(h0)
    _continue(run, [(src, None)], 1, 4)
    dst = capi.Track.load(h1, src.snapshot())
    cl = src.clone(h1)
    _continue(run, [(src, dst), (src.clone(h0), cl)], 4, run.steps)
    _bytes_equal(dst.snapshot(), src.snapshot(), "final snapshots across devices")
    for t in (src, dst, cl):
        t.close()
    h0.close()
    h1.close()
