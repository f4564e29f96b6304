"""Helpers for the per-iteration log of a window solve (kba_result.iterations): invariants one log must satisfy on its own,
and the record-by-record comparison of two logs of the same window (CUDA path against CPU oracle).

A log is a sequence of runs.  A run is one Levenberg-Marquardt solve: a record with iteration == 0 (the cost, gradient and
radius the solve starts from), then one record per iteration.  An inner solve of solveTrimmed (solve_index) is one run, or two
when a trimming-round solve that did not decrease the cost was repeated with three times the iterations
(robust_solving.cpp:172-181): the summary solves[solve_index] then describes the second one.  A solve whose first evaluation
failed (initial_cost == -1, FAILURE) writes no record at all.
"""
import math
from collections import namedtuple

FIELDS = ("cost", "cost_change", "gradient_max_norm", "step_norm", "relative_decrease", "trust_region_radius")

# Largest deviation a field of a CUDA record may have from the oracle's record.  cost, step_norm, gradient_max_norm,
# relative_decrease and trust_region_radius are relative; cost_change is absolute in units of the record's cost (late in a
# solve it is the difference of two nearly equal sums, so its error is eps * cost, not eps * change).  A row without a field
# does not compare it.
#
# Two FP64 rows.  "fp64_head" holds the head of a log (log_deviations(head=True): iterations 0 .. 2 of the first inner solve),
# whose records both sides compute from the same iterate to rounding: this is the sharp per-step check.  "fp64" holds every
# record.  It is looser by orders of magnitude and cannot be otherwise: a rounding difference in one accepted iterate is
# amplified by the flat directions of the problem in every later step (landmarks seen once or twice, the plane blocks), so
# late records differ by 1e-6 between ANY two FP64 implementations -- the oracle against itself with its sums split over 4
# threads instead of 1 deviates as much as the CUDA path does (third column).  What "fp64" adds is the flags of every record
# and costs at 1e-8.
#
# Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W) by scripts/iteration_log_agreement.py: the worst record over the
# 17 windows of tests/test_iteration_log.py and the kernel variants (ground-plane windows under the prefix rule).  Each
# tolerance is about 100 times the worst FP64 value.
#   field                  head      whole log: CUDA vs oracle   oracle vs oracle (threads)
#   cost                   8.9e-12   1.2e-10                     1.1e-10
#   cost_change / cost     9.2e-12   1.2e-10                     1.1e-10
#   gradient_max_norm      1.7e-11   2.2e-06                     2.1e-05
#   step_norm              6.8e-12   8.5e-06                     8.4e-06
#   relative_decrease      1.5e-11   8.5e-07                     7.0e-07
#   trust_region_radius    0         9.0e-07                     6.2e-06
# (whole-log worst cases: ragged and stereo_rig for the gradient, step and radius, config3_kf8 for the costs.)
# precision = 1, first inner solve of config 2: cost 5.1e-06, step_norm 3.6e-05.
TOL = {
    "fp64_head": dict(cost=1e-9, cost_change=1e-9, gradient_max_norm=2e-9, step_norm=1e-9, relative_decrease=2e-9,
                      trust_region_radius=1e-9),
    "fp64": dict(cost=1e-8, cost_change=1e-8, gradient_max_norm=2e-4, step_norm=1e-3, relative_decrease=1e-4,
                 trust_region_radius=1e-4),
    # kba_options.precision = 1: residual / Jacobian blocks in single precision, FP64 accumulation (first inner solve only)
    "fp32_linearize": dict(cost=5e-4, step_norm=4e-3),
}

RADIUS_PREFIX_LIMIT = 1e12   # prefix rule: records are compared while every radius before them is at most this
TERM_FAILURE = 2

Rec = namedtuple("Rec", ("solve_index", "run", "iteration", "valid", "successful") + FIELDS)


def records(result):
    """the log as a list of Rec; `run` counts the iteration-0 records of the same solve_index seen so far (0 or 1)"""
    out, seen = [], {}
    for e in result.iterations:
        if e.iteration == 0:
            seen[e.solve_index] = seen.get(e.solve_index, -1) + 1
        out.append(Rec(e.solve_index, seen.get(e.solve_index, 0), e.iteration, bool(e.step_is_valid), bool(e.step_is_successful),
                       e.cost, e.cost_change, e.gradient_max_norm, e.step_norm, e.relative_decrease, e.trust_region_radius))
    return out


def runs(result):
    """{(solve_index, run): [Rec, ...]} in log order"""
    out = {}
    for r in records(result):
        out.setdefault((r.solve_index, r.run), []).append(r)
    return out


def _is_tolerance_record(r):
    """the last record of a solve that a parameter / function tolerance ended: the step was valid, it is not applied, and
    relative_decrease is written as 0 (a rejected step cannot have it: a cost change of exactly 0 fires the function tolerance)"""
    return r.valid and not r.successful and r.relative_decrease == 0.0


def check_log_invariants(result, opt, label=""):
    """what a log must satisfy whoever wrote it (CUDA path or oracle): see the module docstring and the comments below"""
    c = result.c
    assert 0 <= c.num_iteration_records <= c.iterations_capacity, (label, c.num_iteration_records, c.iterations_capacity)
    recs = records(result)
    assert len(recs) == c.num_iteration_records
    # solves appear in order, a solve's repetition directly after it
    order = [(r.solve_index, r.run) for r in recs]
    assert order == sorted(order), (label, "records out of order")
    by_run = runs(result)
    for (s, run), rr in by_run.items():
        tag = (label, "solve %d run %d" % (s, run))
        assert 0 <= s < c.num_solves and run <= 1, tag
        assert [r.iteration for r in rr] == list(range(len(rr))), (tag, "iterations are not 0, 1, 2, ... without gaps")
        r0 = rr[0]
        assert not r0.valid and not r0.successful and r0.cost_change == 0.0 and r0.step_norm == 0.0, tag
        assert r0.trust_region_radius == opt.initial_trust_region_radius, tag
        x_cost, x_gmax, radius, divisor = r0.cost, r0.gradient_max_norm, r0.trust_region_radius, 2.0
        for i, r in enumerate(rr[1:], 1):
            tag_i = tag + ("iteration %d" % i,)
            assert r.valid or not r.successful, tag_i
            if r.successful:
                # Ceres 1.13 LevenbergMarquardtStrategy::StepAccepted
                rho = r.relative_decrease
                assert rho > opt.min_relative_decrease, tag_i
                want = min(opt.max_trust_region_radius, radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3))
                assert abs(r.trust_region_radius - want) <= 8 * 2.0 ** -52 * want, (tag_i, r.trust_region_radius, want)
                # the sums of the accepted cost may be taken again (with the Jacobian) after the candidate's: rounding only
                assert abs(r.cost_change - (x_cost - r.cost)) <= 1e-12 * x_cost, (tag_i, r.cost_change, x_cost - r.cost)
                assert r.step_norm > 0.0, tag_i
                x_cost, x_gmax, radius, divisor = r.cost, r.gradient_max_norm, r.trust_region_radius, 2.0
                continue
            assert r.gradient_max_norm == x_gmax, (tag_i, "an unsuccessful record carries the gradient of the accepted iterate")
            if _is_tolerance_record(r):
                # the candidate of a firing tolerance test is not applied: cost and radius of x, and the solve ends
                assert i == len(rr) - 1, (tag_i, "a tolerance-terminated record is the last one")
                assert r.cost == x_cost and r.trust_region_radius == radius and r.step_norm > 0.0, tag_i
                assert abs(r.cost_change) <= opt.function_tolerance * x_cost, tag_i
                continue
            # invalid or rejected: StepRejected divides by 2, 4, 8, ... over consecutive failures (powers of two: exact)
            assert r.trust_region_radius == radius / divisor, (tag_i, r.trust_region_radius, radius, divisor)
            radius, divisor = r.trust_region_radius, 2.0 * divisor
            if not r.valid:
                assert r.cost == x_cost and r.cost_change == 0.0 and r.step_norm == 0.0 and r.relative_decrease == 0.0, tag_i
            else:
                assert r.relative_decrease <= opt.min_relative_decrease and r.step_norm > 0.0, tag_i
                if r.cost < 1e300:   # a candidate that failed to evaluate has cost DBL_MAX
                    assert abs(r.cost_change - (x_cost - r.cost)) <= 1e-12 * max(x_cost, abs(r.cost)), tag_i
    for s in range(c.num_solves):
        sm = c.solves[s]
        tag = (label, "solve %d" % s)
        mine = [by_run[k] for k in sorted(by_run) if k[0] == s]
        if sm.initial_cost == -1.0:   # the first evaluation failed: no record of this solve (of its repetition, if it was one)
            assert sm.termination == TERM_FAILURE and sm.final_cost == -1.0 and sm.num_iterations == 0 and len(mine) <= 1, tag
            continue
        assert 1 <= len(mine) <= 2, (tag, "a solve without records")
        if len(mine) == 2:   # repeated because the first run did not decrease the cost
            assert min(r.cost for r in mine[0] if r.successful or r.iteration == 0) >= mine[0][0].cost, tag
        rr = mine[-1]
        # a FAILURE by consecutive invalid steps (or by an accepted iterate that does not evaluate) counts its last iteration
        # and writes no record for it
        last = len(rr) - 1
        assert last == sm.num_iterations or (sm.termination == TERM_FAILURE and last == sm.num_iterations - 1), (tag, last,
                                                                                                                  sm.num_iterations)
        assert sm.num_successful_steps == sum(r.successful for r in rr), tag
        assert sm.initial_cost == rr[0].cost, (tag, sm.initial_cost, rr[0].cost)
        assert sm.final_cost == min(r.cost for r in rr if r.successful or r.iteration == 0), (tag, sm.final_cost)
        if any(_is_tolerance_record(r) for r in rr):
            assert sm.termination == 0, tag
    assert c.initial_cost == c.solves[0].initial_cost and c.final_cost == c.solves[c.num_solves - 1].final_cost, label


def _rel(a, b):
    if a == b:
        return 0.0
    return abs(a - b) / max(abs(a), abs(b))


def _prefix_length(rr):
    """records of a run that the prefix rule compares: up to and including the first one that LEAVES a radius above the limit
    (it was itself computed at a radius below it)"""
    for i, r in enumerate(rr):
        if r.trust_region_radius > RADIUS_PREFIX_LIMIT:
            return i + 1
    return len(rr)


HEAD_ITERATIONS = 2   # "head" of a log: iterations 0 .. 2 of the first inner solve, the length of a trimming-round solve


def log_deviations(gpu, cpu, prefix_rule=False, solves=None, label="", head=False):
    """Align the records of two logs by (solve_index, run, iteration), require equal step_is_valid / step_is_successful, and
    return {field: (worst deviation, key of that record)}.

    Without prefix_rule the two logs must hold the same records.  With it (ground-plane windows: at radii near 1e15 the reduced
    system is numerically singular, and whether a step is invalid is decided by rounding) each run is compared up to the first
    record that leaves a radius above RADIUS_PREFIX_LIMIT in either log; behind it only the accepted steps are compared -- the
    k-th successful record of one log against the k-th of the other, in cost, cost_change and step_norm.
    solves: the solve indices to compare (default: all).  head: only the first HEAD_ITERATIONS iterations of the first inner
    solve -- the records computed from (nearly) the same iterate in both logs, before rounding differences between the two
    iterate sequences have been amplified by the flat directions of the problem."""
    rg, rc = runs(gpu), runs(cpu)
    if head:
        rg = {k: v[:HEAD_ITERATIONS + 1] for k, v in rg.items() if k == (0, 0)}
        rc = {k: v[:HEAD_ITERATIONS + 1] for k, v in rc.items() if k == (0, 0)}
    if solves is not None:
        rg = {k: v for k, v in rg.items() if k[0] in solves}
        rc = {k: v for k, v in rc.items() if k[0] in solves}
    assert sorted(rg) == sorted(rc), (label, "different solves / repetitions", sorted(rg), sorted(rc))
    worst = {f: (0.0, None) for f in FIELDS}

    def note(field, dev, key):
        assert not math.isnan(dev), (label, field, key)
        if dev > worst[field][0]:
            worst[field] = (dev, key)

    def compare(a, b, fields, key):
        assert (a.valid, a.successful) == (b.valid, b.successful), (label, key, "valid / successful", a, b)
        big = abs(b.cost) >= 1e300   # DBL_MAX: the candidate failed to evaluate
        for f in fields:
            x, y = getattr(a, f), getattr(b, f)
            if f == "cost_change":
                if not big:
                    note(f, abs(x - y) / abs(b.cost), key)
            elif f == "relative_decrease":
                if x == 0.0 or y == 0.0:   # the tolerance-terminated record writes 0: both must
                    assert x == y, (label, key, f, x, y)
                elif not big and abs(b.cost_change) >= 1e-4 * abs(b.cost):
                    note(f, _rel(x, y), key)
            else:
                note(f, _rel(x, y), key)

    for k in sorted(rc):
        a, b = rg[k], rc[k]
        n = len(b)
        if prefix_rule:
            n = min(_prefix_length(a), _prefix_length(b))
            assert len(a) >= n and len(b) >= n
            sa, sb = [r for r in a[n:] if r.successful], [r for r in b[n:] if r.successful]
            assert len(sa) == len(sb), (label, k, "accepted steps behind the prefix", len(sa), len(sb))
            for i, (x, y) in enumerate(zip(sa, sb)):
                compare(x, y, ("cost", "cost_change", "step_norm"), k + ("accepted step %d behind the prefix" % i,))
        else:
            assert len(a) == len(b), (label, k, "number of records", len(a), len(b))
        for x, y in zip(a[:n], b[:n]):
            compare(x, y, FIELDS, k + (y.iteration,))
            # the tolerance-terminated record: cost_change is 0 where the parameter tolerance fired
            assert (x.cost_change == 0.0) == (y.cost_change == 0.0) or not _is_tolerance_record(y), (label, k, y.iteration)
    return worst


def compare_logs(gpu, cpu, tol, prefix_rule=False, solves=None, label="", head=False):
    """log_deviations held to one row of TOL; fields the row does not name are not compared"""
    worst = log_deviations(gpu, cpu, prefix_rule, solves, label, head)
    for f, limit in tol.items():
        dev, key = worst[f]
        assert dev <= limit, (label, f, "deviation %.3e > %.1e at (solve, run, iteration) %s" % (dev, limit, key))
    return worst
