"""One kba_options per window, track or frame: a parameter sweep runs as one launch.

Window i of a per-window solve equals window i of the same batch solved with opts[i] for every window, bit for bit, on every
solver path (asserted through the plan driver of tests/test_launch_plan.py); the options reach the kernels (the CPU oracle with
each window's options); a track group with per-track options equals each track solved or tracked alone with its own; an
options array of equal entries equals the single-options call; bad entries fail before anything is uploaded; and changing only
the options re-launches the solve's CUDA graph without rebuilding it."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import sweep_drive as sw
from tests.test_first_step_dense import WINDOWS, assert_path
from tests.test_launch_plan import driver  # noqa: F401  (the plan driver fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _opts(n, precision=0, min_lm=100):
    """n option sets that differ in the Cauchy scales (limo's grid), the quantiles, the trimming rounds (0, 1, 2, and -1 with
    different min_landmarks_for_trimming), the final iteration count and the function tolerance"""
    from limo_b200 import capi
    rounds = [(0, min_lm), (1, min_lm), (2, min_lm), (-1, min_lm), (-1, 100000), (2, min_lm)]
    out = []
    pts = sw.grid(110)[7::19]
    for i in range(n):
        d, r = pts[i % len(pts)]
        o = capi.default_options()
        o.depth_thres, o.reprojection_thres = d, r
        o.depth_quantile = (0.95, 0.9, 0.85)[i % 3]
        o.reprojection_quantile = (0.95, 0.8, 0.9, 0.85)[i % 4]
        o.num_trim_rounds, o.min_landmarks_for_trimming = rounds[i % len(rounds)]
        o.final_solver_iterations = (100, 40, 15)[i % 3]
        o.function_tolerance = (1e-6, 1e-8, 1e-4)[i % 3]
        o.precision = precision
        out.append(o)
    return out


def _same(a, b, what):
    assert a.c.status == b.c.status, what
    assert np.array_equal(a.kf_pose, b.kf_pose), what
    assert np.array_equal(a.kf_plane, b.kf_plane), what
    assert np.array_equal(a.lm_pos[:a.n_lm], b.lm_pos[:b.n_lm]), what
    assert np.array_equal(a.lm_rejected[:a.n_lm], b.lm_rejected[:b.n_lm]), what
    assert a.c.num_solves == b.c.num_solves and bytes(a.c.solves) == bytes(b.c.solves), what
    assert a.c.initial_cost == b.c.initial_cost and a.c.final_cost == b.c.final_cost, what
    assert a.c.num_iteration_records == b.c.num_iteration_records, what
    for x, y in zip(a.iterations, b.iterations):
        assert bytes(x) == bytes(y), what


def _same_frame(a, b, what):
    assert a.c.status == b.c.status and a.c.num_solves == b.c.num_solves, what
    assert np.array_equal(a.kf_pose, b.kf_pose), what
    assert np.array_equal(a.lm_rejected, b.lm_rejected), what
    assert bytes(a.c.solves) == bytes(b.c.solves), what
    assert a.c.num_iteration_records == b.c.num_iteration_records, what
    for x, y in zip(a.iterations, b.iterations):
        assert bytes(x) == bytes(y), what


def test_options_length_is_checked_before_any_call():
    from limo_b200 import capi
    b = capi.Batch.__new__(capi.Batch)
    b.windows, b._p = [None, None, None], None
    with pytest.raises(ValueError):
        b.solve([capi.default_options()] * 2)
    g = capi.TrackGroup.__new__(capi.TrackGroup)
    g.tracks, g._p = [None, None], None
    for call in (lambda: g.solve([None, None], opt=[capi.default_options()]),
                 lambda: g.solve_ranked([None, None], opt=[capi.default_options()] * 3),
                 lambda: g.adjust_pose([None, None], opt=[capi.default_options()])):
        with pytest.raises(ValueError):
            call()


# solver path -> (window of tests/test_first_step_dense.WINDOWS, windows in the batch, precision, launch plan fields)
PATHS = {
    "schur_fused6": ("config2_slice", 6, 0, dict(fused=1, fused_slots=6)),
    "schur_fused7": ("free_kf30_none_fixed", 4, 0, dict(fused=1, fused_slots=7)),
    "large_tiled": ("free_keyframes_30", 4, 0, dict(fused=0, solve_tiled=1, solve_split=0)),
    "large_split": ("config5_kf40_lm700", 4, 0, dict(fused=0, solve_tiled=0, solve_split=32)),
    "large_one_cta": ("config5_kf40_lm700", 17, 0, dict(fused=0, solve_tiled=0, solve_split=0)),
    "motion_only_speed_prior": ("motion_only_speed_prior", 6, 0, dict(fused=1, fused_slots=6)),
    "fp32": ("config2_slice", 4, 1, dict(fused=1, fused_slots=6)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("path", sorted(PATHS))
def test_per_window_equals_uniform(driver, path):  # noqa: F811
    from limo_b200 import capi
    name, n, precision, want = PATHS[path]
    wins = [WINDOWS[name][0]() for _ in range(n)]
    assert_path(driver, wins, want)
    opts = _opts(n, precision, min_lm=30 if name.startswith("motion") else 100)
    h = capi.Handle(0)
    b = h.batch(wins)
    b.solve(opts)
    per = b.download(iterations_capacity=160)
    for i, o in enumerate(opts):
        b.solve(o)
        uni = b.download(iterations_capacity=160)
        _same(per[i], uni[i], "%s window %d" % (path, i))
    b.close()
    h.close()


@pytest.mark.gpu
def test_options_reach_the_kernels():
    """each window of a mixed batch agrees with the oracle solved with its own options; a non-default window differs from its
    default-options solve"""
    from limo_b200 import capi, synth
    from oracle import oracle as orc
    wins = [synth.make_window(1, seed=s) for s in (3, 4, 5, 6)]
    opts = _opts(4)
    h = capi.Handle(0)
    res = h.solve_batch(wins, opts)
    dflt = h.solve_batch(wins)
    differs = []
    for i, (w, o) in enumerate(zip(wins, opts)):
        ref = orc.solve_window(w, o)
        dt = np.linalg.norm(res[i].kf_pose[:, 4:] - ref.kf_pose[:, 4:], axis=1).max()
        assert res[i].c.status == 0 and dt <= 1e-6, (i, dt)
        assert abs(res[i].c.final_cost - ref.c.final_cost) <= 1e-8 * ref.c.final_cost, i
        # negative control: the default options solve the window to another result than its own options
        d0 = np.linalg.norm(res[i].kf_pose[:, 4:] - dflt[i].kf_pose[:, 4:], axis=1).max()
        differs.append(d0 > 1e-6 or abs(res[i].c.final_cost - dflt[i].c.final_cost) > 1e-8 * dflt[i].c.final_cost)
    assert any(differs), differs
    h.close()


@pytest.mark.gpu
def test_equal_entries_equal_the_single_options_call():
    from limo_b200 import capi, synth
    wins = [synth.make_window(2, n_kf=12, n_lm=400, n_obs=3000, seed=s) for s in (1, 2, 3)]
    o = _opts(1)[0]
    h = capi.Handle(0)
    b = h.batch(wins)
    b.solve(o)
    one = b.download(iterations_capacity=160)
    b.solve([o] * 3)
    many = b.download(iterations_capacity=160)
    for i in range(3):
        _same(one[i], many[i], "window %d" % i)
    b.close()
    h.close()


@pytest.fixture
def sweep(monkeypatch):
    from limo_b200 import capi
    monkeypatch.setenv("KBA_P_SPLIT", "6")  # the same landmark split alone and in the group (tests/test_track_group.py)
    h = capi.Handle(0)
    dr = sw.SweepDrive(W=12, steps=4)
    yield h, dr
    h.close()


@pytest.mark.gpu
def test_sweep_drive_equals_tracks_alone(sweep):
    """12 tracks of limo's grid over a 12-keyframe ground-plane drive: adjust_pose, push, solve and write-back each step, as a
    group with per-track options and each track alone with its own"""
    from limo_b200 import capi
    h, dr = sweep
    G = 12
    opts = sw.options(sw.grid(110)[::9][:G])
    grp_t, alone_t = [dr.make(h) for _ in range(G)], [dr.make(h) for _ in range(G)]
    grp = capi.TrackGroup(h, [t for t, _ in grp_t])
    for step in range(dr.steps):
        if step:
            fr = grp.adjust_pose([dr.frame(m, step) for _, m in grp_t], opts)
            for i, ((ta, ma), o) in enumerate(zip(alone_t, opts)):
                fa = ta.adjust_pose(opt=o, **dr.frame(ma, step))
                _same_frame(fr[i], fa, "step %d track %d frame" % (step, i))
                dr.push(grp_t[i][0], grp_t[i][1], step, fr[i].kf_pose[0])
                dr.push(ta, ma, step, fa.kf_pose[0])
        reqs = [m.request(step) for _, m in grp_t]
        rg = grp.solve(reqs, opts)
        for i, ((ta, ma), o) in enumerate(zip(alone_t, opts)):
            ra = ta.solve(opt=o, **ma.request(step))
            _same(rg[i], ra, "step %d track %d" % (step, i))
            grp_t[i][1].record(rg[i]); ma.record(ra)
    grp.close()
    for t, _ in grp_t + alone_t:
        t.close()


@pytest.mark.gpu
def test_group_calls_equal_single_calls(sweep):
    """solve_ranked and a skipped track with per-track options; the group's stores equal the single tracks' afterwards (the next
    solve reads them)"""
    from limo_b200 import capi
    h, dr = sweep
    opts = sw.options(sw.grid(110)[3::37])
    ga, ta = [dr.make(h) for _ in opts], [dr.make(h) for _ in opts]
    grp = capi.TrackGroup(h, [t for t, _ in ga])
    reqs = [m.request(0) for _, m in ga]
    for (t, _), (u, _), r in zip(ga, ta, reqs):
        for x in (t, u):
            x.select_landmarks(r["kf_slots"], r["lm_slots"])
            x.rank_landmarks(r["kf_slots"], r["lm_slots"], draws=np.arange(100000) % 7)
    sel = [dict(kf_slots=r["kf_slots"], kf_fixed=r["kf_fixed"]) for r in reqs]
    rg = grp.solve_ranked(sel, opts)
    for i, ((u, _), o) in enumerate(zip(ta, opts)):
        _same(rg[i], u.solve_ranked(opt=o, **sel[i]), "ranked track %d" % i)
    reqs[1] = None  # sits out: its entry is not read
    bad = list(opts)
    bad[1] = capi.default_options()
    bad[1].num_trim_rounds = 7
    rg = grp.solve(reqs, bad)
    for i, ((u, m), o) in enumerate(zip(ta, opts)):
        if reqs[i] is not None:
            _same(rg[i], u.solve(opt=o, **m.request(0)), "solve track %d" % i)
    grp.close()
    for t, _ in ga + ta:
        t.close()


@pytest.mark.gpu
def test_bad_entries_change_nothing(sweep):
    from limo_b200 import capi
    h, dr = sweep
    opts = sw.options(sw.grid(3))
    tr = [dr.make(h) for _ in opts]
    grp = capi.TrackGroup(h, [t for t, _ in tr])
    reqs = [m.request(0) for _, m in tr]
    mixed = sw.options(sw.grid(3))
    mixed[2].precision = 1
    seven = sw.options(sw.grid(3))
    seven[1].num_trim_rounds = 7
    for bad, code, idx in ((mixed, "error 1:", "track 2"), (seven, "error 4:", "track 1")):
        for call in (lambda: grp.solve(reqs, bad), lambda: grp.adjust_pose([dr.frame(m, 1) for _, m in tr], bad)):
            with pytest.raises(capi.KbaError) as e:
                call()
            assert code in str(e.value) and idx in str(e.value), str(e.value)
    wins = [dr.base.win] * 3
    with pytest.raises(capi.KbaError) as e:
        h.solve_batch(wins, mixed)
    assert "window 2" in str(e.value)
    # nothing was written: a solve now equals a solve of fresh tracks
    fresh = [dr.make(h) for _ in opts]
    rg = grp.solve(reqs, opts)
    for i, ((t, m), o) in enumerate(zip(fresh, opts)):
        _same(rg[i], t.solve(opt=o, **m.request(0)), "track %d" % i)
    grp.close()
    for t, _ in tr + fresh:
        t.close()


@pytest.mark.gpu
def test_changing_only_the_options_keeps_the_graph(tmp_path):
    """two solves of one batch with different options: no graph rebuild reported, results equal the stream path's"""
    script = tmp_path / "w.py"
    script.write_text("""
import sys
import numpy as np
sys.path.insert(0, %r)
from limo_b200 import capi, synth
from tests.test_window_options import _opts
h = capi.Handle(0)
b = h.batch([synth.make_window(2, n_kf=12, n_lm=400, n_obs=3000, seed=s) for s in (1, 2, 3)])
out = []
for o in (_opts(3), _opts(6)[3:]):
    b.solve(o)
    out += [np.concatenate([r.kf_pose.ravel(), r.lm_pos.ravel(), [r.c.final_cost]]) for r in b.download()]
np.save(sys.argv[1], np.stack(out))
""" % ROOT)
    outs = {}
    for mode in ("2", "0"):
        env = dict(os.environ, KBA_GRAPH=mode, KBA_GRAPH_VERBOSE="1")
        p = subprocess.run([sys.executable, str(script), str(tmp_path / ("o%s.npy" % mode))], env=env, capture_output=True,
                           text=True, cwd=ROOT)
        assert p.returncode == 0, p.stderr
        outs[mode] = np.load(tmp_path / ("o%s.npy" % mode))
        if mode == "2":
            assert p.stderr.count("solve graph built") == 1, p.stderr
    assert np.array_equal(outs["2"], outs["0"])


def test_sweep_bench_dry_run():
    p = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "sweep_bench.py"), "--dry-run", "--groups", "110"],
                       capture_output=True, text=True, cwd=ROOT)
    assert p.returncode == 0, p.stderr
