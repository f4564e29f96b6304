"""Iteration 1 of a window's first inner solve against a dense extended-precision Levenberg-Marquardt step.

tests/test_iteration_log.py holds the CUDA log to the oracle's, and so trusts the oracle's Schur elimination, Jacobi scaling,
damping, back substitution and controller arithmetic.  This file pins the first step of both to a reference that shares none
of that code: the damped normal equations of the WHOLE problem (poses and landmarks, no elimination), assembled and solved in
numpy.longdouble -- on the x86 hosts this suite runs on that is the 80-bit extended type (64-bit significand), which is what
the host provides; the test is skipped where longdouble is no wider than double.

From the implementation under test it takes the robustified blocks (r, J_pose, J_landmark, cost) of evaluate(), which
tests/test_gpu_parity.py::test_eval_matches_oracle and tests/test_oracle_jacobians.py pin on their own, and from the oracle
the two operators pose_plus and scale_reg, which tests/test_oracle_jacobians.py checks by finite differences.  Plane-free
windows only: the plane blocks and the regulariser chain of ground-plane windows have no dense reference here.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.linalg

from limo_b200 import synth
from tests import edge_windows as ew
from tests import iter_log as il

LD = np.longdouble
pytestmark = pytest.mark.skipif(np.finfo(LD).eps >= np.finfo(np.float64).eps, reason="numpy.longdouble is not an extended type here")

# Records 0 and 1 against the dense step, relative (cost_change in units of the cost).  Worst observed over the five windows,
# oracle: step_norm 2.4e-12 (ragged: landmarks seen once, held by the damping alone), cost 4.1e-13, cost_change 1.7e-13,
# relative_decrease 2.9e-13; CUDA path on an NVIDIA H100 80GB HBM3 (700 W): step_norm 1.2e-12, cost 4.2e-13, cost_change
# 1.7e-13, relative_decrease 3.0e-13 (scripts/iteration_log_agreement.py).  About 100 times the worst of them:
STEP_TOL = 1e-10


def _shapes(name):
    from tests import test_schur_fused_shapes as sf
    return getattr(sf, name)()


WINDOWS = {
    "config1": lambda: synth.make_window(1),
    "config2_slice": lambda: synth.make_window(2, n_kf=12, n_lm=400, n_obs=3000),
    "stereo_rig": lambda: _shapes("_stereo_rig"),
    "gap_over_fixed_keyframe": lambda: _shapes("_gap_over_fixed_keyframe"),
    "ragged": ew.CASES["ragged"],
}


def _solve_spd(A, b):
    """A y = b for a symmetric positive definite longdouble A: double-precision Cholesky, residuals and updates in longdouble
    (iterative refinement contracts by cond(A) * 2^-53 per round; the damped, Jacobi-scaled matrix has a condition of at most
    ~1e10, 5e4 on config 1).  It stops once a correction is below 1e-14 of the solution: the following one is smaller still,
    and the records it is compared with are held to 1e-9 .. 1e-11"""
    cf = scipy.linalg.cho_factor(A.astype(np.float64), lower=True)
    y = np.zeros_like(b)
    for _ in range(12):
        res = b - A @ y
        dy = scipy.linalg.cho_solve(cf, res.astype(np.float64)).astype(LD)
        y = y + dy
        if np.abs(dy).max() <= 1e-14 * np.abs(y).max():
            return y
    raise AssertionError("iterative refinement did not converge")


def dense_first_step(win, opt, blocks, evaluate, orc):
    """Records 0 and 1 of the first inner solve as a dense reference gives them.

    blocks: (r [n_obs, 3], jac_pose [n_obs, 3, 6], jac_lm [n_obs, 3, 3], cost) at the window's state; evaluate(window) returns
    the same tuple (the candidate's cost is taken from it); orc: the oracle binding (pose_plus, scale_reg).
    Unknowns: 6 columns per keyframe that is not constant, then 3 per landmark with an observation.  The Jacobian is never
    stored densely (18 000 x 2 100 longdoubles); J^T J and J^T r are summed from its blocks, which is the same matrix."""
    r, jp, jl = (np.asarray(a, dtype=LD) for a in blocks[:3])
    cost_x = LD(blocks[3])
    ptr = np.asarray(win.lm_obs_ptr)
    lm_of_obs = np.repeat(np.arange(win.n_lm), np.diff(ptr))
    kf_of_obs = np.asarray(win.obs_kf)
    has_scale = win.scale_weight > 0
    free_kf = [k for k in range(win.n_kf) if not win.kf_fixed[k] and
               ((kf_of_obs == k).any() or (has_scale and k in (win.scale_kf0, win.scale_kf1)))]
    col_kf = {k: 6 * i for i, k in enumerate(free_kf)}
    in_lm = np.flatnonzero(np.diff(ptr) > 0)
    n_p = 6 * len(free_kf)
    col_lm = np.full(win.n_lm, -1)
    col_lm[in_lm] = n_p + 3 * np.arange(len(in_lm))
    n = n_p + 3 * len(in_lm)

    # rows of the Jacobian as (columns, values, residual): observations, then the scale regulariser
    rows_c, rows_v, rows_r = [], [], []
    for o in range(win.n_obs):
        k, j = int(kf_of_obs[o]), int(lm_of_obs[o])
        cols = np.arange(col_lm[j], col_lm[j] + 3)
        vals = jl[o]
        if k in col_kf:
            cols = np.concatenate([np.arange(col_kf[k], col_kf[k] + 6), cols])
            vals = np.concatenate([jp[o], jl[o]], axis=1)
        rows_c.append(cols); rows_v.append(vals); rows_r.append(r[o])

    def scale_row(poses):
        """sqrt(weight) * (residual, Jacobian) of the scale regulariser |t(pose1 relative to pose0)| - scale_value: Ceres'
        ScaledLoss(TrivialLoss, weight) corrects a block by sqrt(rho') = sqrt(weight); its cost is weight * r^2 / 2"""
        res, j1, j0 = orc.scale_reg(poses[win.scale_kf1], poses[win.scale_kf0], win.scale_value)
        sw = np.sqrt(LD(win.scale_weight))
        cols, vals = [], []
        for k, jk in ((win.scale_kf1, j1), (win.scale_kf0, j0)):
            if k in col_kf:
                cols.append(np.arange(col_kf[k], col_kf[k] + 6)); vals.append(sw * jk.astype(LD))
        return np.concatenate(cols), np.concatenate(vals, axis=1), sw * res.astype(LD), LD(win.scale_weight) * LD(res[0]) ** 2 / 2

    reg_cost = LD(0)
    if has_scale:
        cols, vals, res, reg_cost = scale_row(win.kf_pose)
        rows_c.append(cols); rows_v.append(vals); rows_r.append(res)

    H, g = np.zeros((n, n), dtype=LD), np.zeros(n, dtype=LD)
    for cols, vals, res in zip(rows_c, rows_v, rows_r):
        H[np.ix_(cols, cols)] += vals.T @ vals
        g[cols] += vals.T @ res
    c = np.diag(H).copy()                                   # squared column norms
    s = 1 / (1 + np.sqrt(c))                                # Jacobi scaling, taken once at the first iterate
    radius = LD(opt.initial_trust_region_radius)
    D = np.clip(c * s * s, LD(opt.min_lm_diagonal), LD(opt.max_lm_diagonal)) / radius
    A = H * s[:, None] * s[None, :]
    A[np.diag_indices(n)] += D
    delta = s * _solve_spd(A, -s * g)
    model = LD(0)                                           # -(J delta)^T (r + J delta / 2)
    for cols, vals, res in zip(rows_c, rows_v, rows_r):
        jd = vals @ delta[cols]
        model -= jd @ (res + jd / 2)

    def plus(step):
        """x + step: pose_plus on the keyframes, addition on the landmarks; and the norms of the ambient difference"""
        step = step.astype(np.float64)
        poses, lms = win.kf_pose.copy(), win.lm_pos.copy()
        for k, c0 in col_kf.items():
            poses[k] = orc.pose_plus(win.kf_pose[k], step[c0:c0 + 6])
        lms[in_lm] += step[n_p:].reshape(-1, 3)
        diff = np.concatenate([(poses - win.kf_pose)[free_kf].ravel(), (lms - win.lm_pos)[in_lm].ravel()]).astype(LD)
        return poses, lms, np.sqrt(diff @ diff), np.abs(diff).max()

    out = SimpleNamespace(cost0=cost_x + reg_cost, radius0=radius, n_columns=n)
    out.gradient_max_norm0 = plus(-g)[3]
    poses, lms, out.step_norm, _ = plus(delta)
    cand = ew._rebuild(win, kf_pose=poses, lm_pos=lms)
    cand_blocks = evaluate(cand)
    assert cand_blocks[4] == 0
    cand_cost = LD(cand_blocks[3]) + (scale_row(poses)[3] if has_scale else 0)
    out.cost_change = out.cost0 - cand_cost
    out.relative_decrease = out.cost_change / model
    out.successful = bool(out.relative_decrease > opt.min_relative_decrease)
    # neither tolerance test fires on the first step of these windows (the record would be written differently)
    x = np.concatenate([win.kf_pose[free_kf].ravel(), win.lm_pos[in_lm].ravel()])
    assert out.step_norm > opt.parameter_tolerance * (np.linalg.norm(x) + opt.parameter_tolerance)
    assert abs(out.cost_change) > opt.function_tolerance * out.cost0
    out.cost1 = cand_cost                                   # the accepted iterate's cost, or the rejected candidate's
    rho = out.relative_decrease
    out.radius1 = min(LD(opt.max_trust_region_radius), radius / max(LD(1) / 3, 1 - (2 * rho - 1) ** 3)) if out.successful else radius / 2
    return out


def _check_first_step(res, ref, tol, label):
    """records 0 and 1 of `res` (first inner solve) against the dense step, every field at `tol` (relative; cost_change in
    units of the cost)"""
    recs = il.records(res)
    r0, r1 = recs[0], recs[1]
    assert (r0.solve_index, r0.iteration, r1.solve_index, r1.iteration) == (0, 0, 0, 1), label
    dev = {
        "cost 0": abs(r0.cost - ref.cost0) / ref.cost0,
        "gradient_max_norm 0": abs(r0.gradient_max_norm - ref.gradient_max_norm0) / ref.gradient_max_norm0,
        "radius 0": abs(r0.trust_region_radius - ref.radius0) / ref.radius0,
        "cost 1": abs(r1.cost - ref.cost1) / ref.cost1,
        "cost_change": abs(r1.cost_change - ref.cost_change) / ref.cost0,
        "step_norm": abs(r1.step_norm - ref.step_norm) / ref.step_norm,
        "relative_decrease": abs(r1.relative_decrease - ref.relative_decrease) / abs(ref.relative_decrease),
        "radius 1": abs(r1.trust_region_radius - ref.radius1) / ref.radius1,
    }
    assert r1.valid and r1.successful == ref.successful, label
    for name, d in dev.items():
        assert d <= tol, (label, name, float(d), tol)
    return {k: float(v) for k, v in dev.items()}


@pytest.mark.parametrize("name", list(WINDOWS))
def test_oracle_first_step_matches_dense_step(oracle, name):
    """the oracle's elimination, scaling, damping, back substitution and controller arithmetic, without a GPU"""
    win = WINDOWS[name]()
    opt = oracle.default_options()
    ref = dense_first_step(win, opt, oracle.evaluate(win), oracle.evaluate, oracle)
    assert ref.successful and ref.n_columns > 3 * 190
    _check_first_step(oracle.solve_window(win, opt), ref, STEP_TOL, name)


def test_dense_step_notices_a_wrong_block(oracle):
    """the reference can fail: the landmark Jacobian of ONE observation of 1000 off by 1e-6 moves the candidate cost by 1.4e-9"""
    win = WINDOWS["config1"]()
    opt = oracle.default_options()
    r, jp, jl, cost, failed = oracle.evaluate(win)
    jl = jl.copy()
    jl[5] *= 1 + 1e-6
    ref = dense_first_step(win, opt, (r, jp, jl, cost, failed), oracle.evaluate, oracle)
    with pytest.raises(AssertionError):
        _check_first_step(oracle.solve_window(win, opt), ref, STEP_TOL, "perturbed")


@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(WINDOWS))
def test_cuda_first_step_matches_dense_step(handle, oracle, name):
    """the CUDA pass chain of one LM iteration without the oracle's solver: blocks from kba_eval, the step from the dense
    reference, records 0 and 1 of kba_solve_window"""
    win = WINDOWS[name]()
    opt = handle.default_options()
    ref = dense_first_step(win, opt, handle.evaluate(win), handle.evaluate, oracle)
    _check_first_step(handle.solve_window(win, opt), ref, STEP_TOL, name)
