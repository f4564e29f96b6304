"""The landmark-sharded solve of windows with ground-plane residuals, and the in-process exchange that runs several ranks on one
GPU (capi.ShardComm.local, parallel.solve_sharded_local).

A ground-plane residual belongs to the rank owning its landmark; the per-keyframe (pose | normal | distance) blocks, the
ground-plane cost and the plane layout are window-wide.  World 1 must reproduce the plain solve bit for bit, over NCCL and over
the in-process exchange.  World 2 and 3 on one GPU are the check of the cross-rank sums: the order of the additions changes, so
they agree with the plain solve (and the oracle) to the north-star tolerances, and all ranks return the same bits.
"""
import numpy as np
import pytest

from limo_b200 import parallel, synth
from limo_b200.capi_types import Window

TRANSLATION_TOL = 1e-6   # metres
COST_REL_TOL = 1e-8


def _with(win, **kw):
    """a copy of `win` with some fields replaced"""
    f = dict(kf_pose=win.kf_pose, kf_fixed=win.kf_fixed, cam_intr=win.cam_intr, cam_pose=win.cam_pose, lm_pos=win.lm_pos,
             lm_weight=win.lm_weight, lm_obs_ptr=win.lm_obs_ptr, obs_kf=win.obs_kf, obs_u=win.obs_u, obs_v=win.obs_v,
             obs_d=win.obs_d, obs_cam=win.obs_cam, kf_plane=win.kf_plane, gp_lm=win.gp_lm, gp_kf=win.gp_kf,
             gp_weight=win.gp_weight, scale_kf0=win.scale_kf0, scale_kf1=win.scale_kf1, scale_weight=win.scale_weight,
             scale_value=win.scale_value, plane_reg_weight=win.plane_reg_weight, plane_dist_fixed=win.plane_dist_fixed,
             landmarks_fixed=win.landmarks_fixed, speed_kf=win.speed_kf, speed_weight=win.speed_weight, speed_dt=win.speed_dt,
             speed_v_before=win.speed_v_before, speed_T_origin_before=win.speed_T_origin_before)
    f.update(kw)
    return Window(**f)


def _ground_window(n_kf=40, seed=None):
    win = synth.make_window(3, n_kf=n_kf, seed=seed)
    assert win.n_gp > 0 and win.plane_reg_weight == 10.0
    return win


def _plane_free_window():
    return synth.make_window(5, n_kf=40, n_lm=3000, n_obs=45000)


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the partition of the ground-plane lists
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_shards_tile_the_ground_plane_lists(world):
    win = _ground_window()
    lm, kf, wt = [], [], []
    prev_j1 = 0
    for r in range(world):
        sub, j0, j1 = parallel.shard_window(win, r, world)
        assert j0 == prev_j1
        prev_j1 = j1
        if sub.n_gp:
            assert ((sub.gp_lm >= 0) & (sub.gp_lm < j1 - j0)).all()
            lm.append(sub.gp_lm + j0); kf.append(sub.gp_kf); wt.append(sub.gp_weight)
        # the window's scalars travel with every shard
        for name in ("scale_kf0", "scale_kf1", "scale_weight", "scale_value", "plane_reg_weight", "plane_dist_fixed",
                     "landmarks_fixed", "speed_kf", "speed_weight", "speed_dt"):
            assert getattr(sub, name) == getattr(win, name), name
        assert np.array_equal(sub.kf_plane, win.kf_plane) and np.array_equal(sub.kf_fixed, win.kf_fixed)
    assert prev_j1 == win.n_lm
    assert np.array_equal(np.concatenate(lm), win.gp_lm)
    assert np.array_equal(np.concatenate(kf), win.gp_kf)
    assert np.array_equal(np.concatenate(wt), win.gp_weight)


def test_ground_window_takes_the_large_path_shapes():
    """the windows below: 391 and 591 reduced rows (10 per free keyframe plus one; keyframe 0 is fixed), past the fused path"""
    for n_kf, rows in ((40, 391), (60, 591)):
        win = _ground_window(n_kf)
        assert 10 * int((win.kf_fixed == 0).sum()) + 1 == rows


# ---------------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


def _nccl_world1(handle, win, opt=None):
    from limo_b200 import capi
    sub, j0, _ = parallel.shard_window(win, 0, 1)
    comm = capi.ShardComm(handle, 0, 1, capi.shard_unique_id())
    batch = handle.batch([sub])
    batch.set_shard(comm, j0, win.n_lm)
    batch.solve(opt or capi.default_options())
    res = batch.download(256)[0]
    batch.close()
    comm.close()
    return res


def _summary(res):
    return [(s.num_iterations, s.num_successful_steps, s.termination, s.num_landmarks) for s in res.solves]


def _assert_bit_equal(a, b, n_lm, counts=True):
    assert a.c.status == 0 and b.c.status == 0
    assert a.c.num_solves == b.c.num_solves
    if counts:
        assert _summary(a) == _summary(b)
    else:
        assert [s.num_iterations for s in a.solves] == [s.num_iterations for s in b.solves]
    assert [s.final_cost for s in a.solves] == [s.final_cost for s in b.solves]
    assert np.array_equal(a.kf_pose, b.kf_pose)
    assert np.array_equal(a.kf_plane, b.kf_plane)
    assert np.array_equal(a.lm_pos[:n_lm], b.lm_pos[:n_lm])
    assert np.array_equal(a.lm_rejected[:n_lm], b.lm_rejected[:n_lm])


def _assert_close(results, ref, win):
    """a W-rank solve against a one-process solve of the whole window (plain GPU solve or the oracle)"""
    kf_pose, kf_plane, lm_pos, rej = parallel.merge_shards(results, win.n_lm)
    for r, _, _ in results:  # the reduced solve is replicated: every rank holds the same bits
        assert r.c.status == 0
        assert np.array_equal(r.kf_pose, kf_pose) and np.array_equal(r.kf_plane, kf_plane)
        assert [s.num_iterations for s in r.solves] == [s.num_iterations for s in results[0][0].solves]
    r0 = results[0][0]
    assert r0.c.num_solves == ref.c.num_solves
    assert np.array_equal(rej, ref.lm_rejected[:win.n_lm])
    dt = np.linalg.norm(kf_pose[:, 4:] - ref.kf_pose[:, 4:], axis=1).max()
    assert dt <= TRANSLATION_TOL, dt
    assert r0.solves[-1].final_cost == pytest.approx(ref.solves[-1].final_cost, rel=COST_REL_TOL)
    assert r0.solves[0].initial_cost == pytest.approx(ref.solves[0].initial_cost, rel=COST_REL_TOL)


@pytest.mark.gpu
@pytest.mark.parametrize("plane_reg_weight", [10.0, 0.0])
def test_world1_nccl_ground_plane_equals_plain_solve(handle, plane_reg_weight):
    win = _with(_ground_window(), plane_reg_weight=plane_reg_weight)
    rp = handle.solve_window(win)
    rs = _nccl_world1(handle, win)
    # the summaries' landmark / residual counts are the rank's own; with one rank they are the window's
    _assert_bit_equal(rs, rp, win.n_lm)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ground", "plane_free"])
def test_world1_loopback_equals_nccl(handle, kind):
    win = _ground_window() if kind == "ground" else _plane_free_window()
    rn = _nccl_world1(handle, win)
    [(rl, j0, j1)] = parallel.solve_sharded_local(win, 1)
    assert (j0, j1) == (0, win.n_lm)
    _assert_bit_equal(rl, rn, win.n_lm)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_loopback_ground_plane_matches_plain_solve(handle, world):
    win = _ground_window()
    rp = handle.solve_window(win)
    res = parallel.solve_sharded_local(win, world)
    assert all(j1 > j0 for _, j0, j1 in res)
    assert sum(r.solves[0].num_residual_blocks for r, _, _ in res) > 0
    _assert_close(res, rp, win)


@pytest.mark.gpu
def test_loopback_ground_plane_matches_oracle(handle, oracle):
    win = _ground_window()
    rc = oracle.solve_window(win)
    for world in (2, 3):
        _assert_close(parallel.solve_sharded_local(win, world), rc, win)


@pytest.mark.gpu
def test_loopback_ground_plane_60_keyframes(handle):
    win = _ground_window(60)
    rp = handle.solve_window(win)
    _assert_close(parallel.solve_sharded_local(win, 2), rp, win)


@pytest.mark.gpu
def test_loopback_world2_plane_free(handle):
    """the path that existed before ground-plane residuals, with more than one rank"""
    win = _plane_free_window()
    rp = handle.solve_window(win)
    _assert_close(parallel.solve_sharded_local(win, 2), rp, win)


@pytest.mark.gpu
def test_shard_without_ground_points(handle):
    """all ground points in rank 0's landmark range: rank 1 holds none, yet adds rank 0's ground-plane blocks and costs.  At
    plane_reg_weight 10 the regularisation chain makes every free plane variable, so the layout itself is checked below, at 0."""
    base = _ground_window()
    _, j0, j1 = parallel.shard_window(base, 0, 2)
    keep = base.gp_lm < j1
    win = _with(base, gp_lm=base.gp_lm[keep], gp_kf=base.gp_kf[keep], gp_weight=base.gp_weight[keep])
    assert win.n_gp > 0
    assert parallel.shard_window(win, 1, 2)[0].n_gp == 0
    rp = handle.solve_window(win)
    res = parallel.solve_sharded_local(win, 2)
    _assert_close(res, rp, win)
    # the plane blocks moved: planes are variable on both ranks
    assert not np.array_equal(res[1][0].kf_plane, win.kf_plane)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_window_wide_plane_layout_without_chain(handle, world):
    """plane_reg_weight 0: a keyframe's plane blocks are variable only through its ground points.  Every shard holds ground
    points, but those of some keyframes sit on the last rank only, so the other ranks must take those keyframes' plane rows
    from the window-wide gather (k_shard_gp_gather, k_shard_planes) and keep them as trimming goes on (act_glob)."""
    base = _ground_window()
    last = parallel.shard_window(base, world - 1, world)[1]   # first landmark of the last rank
    only_last = (base.gp_kf % 4 == 1) & (base.gp_lm < last)    # drop these keyframes' ground points outside the last rank
    win = _with(base, gp_lm=base.gp_lm[~only_last], gp_kf=base.gp_kf[~only_last], gp_weight=base.gp_weight[~only_last],
                plane_reg_weight=0.0)
    subs = [parallel.shard_window(win, r, world)[0] for r in range(world)]
    assert all(s.n_gp > 0 for s in subs)
    last_kf = set(subs[-1].gp_kf[subs[-1].gp_kf % 4 == 1].tolist())
    assert last_kf and all(not (set(s.gp_kf.tolist()) & last_kf) for s in subs[:-1])
    rp = handle.solve_window(win)
    res = parallel.solve_sharded_local(win, world)
    assert rp.c.num_solves > 1 and rp.lm_rejected[:win.n_lm].any()  # trimming is active
    _assert_close(res, rp, win)
    kf_plane = res[0][0].kf_plane
    # without the chain a keyframe's plane is fixed by its ground points alone (1 to 4 on most keyframes here), so it is nearly
    # unobservable along some directions, and rounding differences of the reordered sums show up there first (as for landmarks
    # seen with little parallax, tests/test_gpu_parity.py); poses and cost are held to the north-star tolerances above
    assert np.abs(kf_plane - rp.kf_plane).max() <= 1e-3
    # the keyframes whose ground points are on the last rank only moved their planes on every rank
    moved = [k for k in last_kf if not np.array_equal(kf_plane[k], win.kf_plane[k])]
    assert len(moved) == len(last_kf)
    # keyframes without ground points kept theirs: the planes of the layout are those of the plain solve
    none = [k for k in range(win.n_kf) if k not in set(win.gp_kf.tolist())]
    assert all(np.array_equal(kf_plane[k], win.kf_plane[k]) for k in none)


@pytest.mark.gpu
def test_loopback_rank_failure_releases_the_others(handle):
    """a rank whose set_shard fails (a batch of two windows) breaks the group: the other rank gets an error, no hang"""
    import threading

    from limo_b200 import capi
    win = _ground_window()
    subs = [parallel.shard_window(win, r, 2) for r in range(2)]
    hs = [capi.Handle(0) for _ in range(2)]
    comms = capi.ShardComm.local(hs)
    batches = [hs[0].batch([subs[0][0], subs[0][0]]), hs[1].batch([subs[1][0]])]
    errors = [None, None]

    def run(r):
        try:
            batches[r].set_shard(comms[r], subs[r][1], win.n_lm)
            batches[r].solve()
        except capi.KbaError as e:
            errors[r] = str(e)

    ts = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=120)
    assert not any(t.is_alive() for t in ts)
    assert errors[0] is not None and "exactly one window" in errors[0]
    assert errors[1] is not None and "in-process exchange" in errors[1]
    for b in batches:
        b.close()
    for c in comms:
        c.close()
    for h in hs:
        h.close()
