"""The quantile trimming of one residual group (kba::trim_select_group, kba_controller.cuh) against an exact-rank reference.

limo's solveTrimmed rejects, in each residual group, the landmarks whose trimming value (largest raw block norm, < 0: the landmark
has no residual of the group) ranks at or above num = (int)(N * quantile) among the N that have one; equal values are ordered by
the caller's landmark index.  One function takes these decisions on the device for every caller: k_trim_select (batch, track and
sharded solves, 512 threads), k_ev_finish (kba_track_evaluate, 512) and k_adjust_pose (adjustPoseOnly, 256).  It keeps 8 keys
per thread in registers and streams past 8 * blockDim items, so the sizes below straddle 256 * 8 and 512 * 8.

Without a GPU: the reference against the CPU oracle's TrimmerQuantile (ties included), the reference's sensitivity to a wrong
tie order and to num off by one, the driver's sm_90a compile, and the quantile rule against the kba_options layout.
On the GPU:
  - tests/cpp/trim_select_driver.cu runs the function in one CTA of 32, 256 and 512 threads on sizes 0 .. 100 000, every value
    family below and quantiles 0 .. 1; every mask must equal the reference exactly;
  - one end-to-end test per caller, on windows whose ties are exact by construction: every third landmark duplicated into
    another slot with the same (constant) position and measurements, so the two trimming values are the same bits;
  - a quantile that is NaN or outside [0, 1] is refused by every entry that takes kba_options, before any launch."""
import math
import os
import re
import struct
import subprocess

import numpy as np
import pytest

from tests.test_adjust_pose import _Frame, _equal_to_general, _opt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "limo_b200", "csrc")
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
NVFLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17"]  # the library's (limo_b200/csrc/Makefile)

SIZES = [0, 1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 4097, 8193, 20000, 100000]
QUANTILES = [0.0, 1e-12, 0.5, 0.7, 0.95, 1.0 - 2.0 ** -53, 1.0, 1.5]
BLOCKS = [32, 256, 512]


# ---- the reference ------------------------------------------------------------------------------------------------------------
def _order(values, oid):
    """indices of the valid items (value >= 0) by (value, oid), -0.0 == +0.0"""
    v = np.asarray(values, np.float64)
    idx = np.nonzero(v >= 0)[0]
    return idx[np.lexsort((np.asarray(oid)[idx], v[idx] + 0.0))]


def _reject_from_order(n, order, quantile, min_groups, off_by=0):
    rej = np.zeros(n, bool)
    N = len(order)
    if N == 0 or N < min_groups:
        return rej
    num = int(float(N) * quantile) + off_by  # the device's IEEE double product, truncated
    if num >= N:
        return rej
    rank = np.arange(N)
    rej[order[rank >= num]] = True
    return rej


def trim_reference(values, oid, quantile, min_groups):
    """TrimmerQuantile of one residual group by exact rank: the valid items (value >= 0; NaN and negative values have no
    residual) ordered by (value, oid) with -0.0 == +0.0; nothing is rejected when N == 0 or N < min_groups or num >= N,
    otherwise the items of rank >= num = (int)(N * quantile)"""
    return _reject_from_order(len(values), _order(values, oid), quantile, min_groups)


# ---- the value families -------------------------------------------------------------------------------------------------------
def _bits(u):
    return np.asarray(u, np.uint64).view(np.float64)


def _family(name, n, rng):
    """n trimming values of one family (deterministic in rng)"""
    if name == "distinct":
        return rng.uniform(0.0, 10.0, n)
    if name == "equal":
        return np.full(n, 0.37)
    if name == "tie_at_pivot":  # a group of 3 .. 50 equal values across the rank each quantile selects, the pivot anywhere in it
        v = np.sort(rng.uniform(0.0, 10.0, n))
        for q in (0.5, 0.7, 0.95, 1.0 - 2.0 ** -53, 0.0) if n else ():
            num = min(int(float(n) * q), n - 1)
            g = int(rng.integers(3, 51))
            a = int(rng.integers(0, g))
            lo, hi = max(num - a, 0), min(num - a + g, n)
            v[lo:hi] = v[lo]
        return rng.permutation(v)
    if name == "many_ties":
        return rng.integers(0, max(n // 4, 1), n) * 0.125
    if name.startswith("sentinel"):  # the -1 "no residual" sentinel on a share of the items, NaN and -inf among them
        share = {"sentinel0": 0.0, "sentinel50": 0.5, "sentinel100": 1.0}[name]
        v = np.where(rng.random(n) < 0.5, rng.integers(0, max(n // 8, 1), n) * 0.25, rng.uniform(0.0, 5.0, n))
        out = rng.random(n) < share
        v[out] = -1.0
        kind = rng.random(n)
        v[out & (kind < 0.1)] = np.nan
        v[out & (kind >= 0.1) & (kind < 0.15)] = -np.inf
        v[out & (kind >= 0.15) & (kind < 0.2)] = -1e-300
        return v
    if name == "signed_zero":  # +0.0 and -0.0 in one tie group among positive values
        v = rng.uniform(0.0, 1.0, n)
        z = rng.random(n) < 1.0 / 32
        v[z] = np.where(rng.random(n) < 0.5, 0.0, -0.0)[z]
        return v
    if name == "subnormal_inf":  # subnormals (some equal), and tie groups of the smallest normal, DBL_MAX and +inf
        pick = rng.choice(6, n, p=[0.2, 0.3, 0.02, 0.02, 0.02, 0.44])
        v = np.empty(n)
        v[pick == 0] = _bits(rng.integers(1, 64, (pick == 0).sum()))
        v[pick == 1] = _bits(rng.integers(1, 1 << 52, (pick == 1).sum(), dtype=np.uint64))
        v[pick == 2] = np.finfo(np.float64).tiny
        v[pick == 3] = np.finfo(np.float64).max
        v[pick == 4] = np.inf
        v[pick == 5] = rng.uniform(0.0, 1e3, (pick == 5).sum())
        return v
    if name == "low_byte":  # the same upper 7 bytes: only the last radix pass separates them
        base = np.float64(3.25).view(np.uint64) & np.uint64(0xFFFFFFFFFFFFFF00)
        return _bits(base | rng.integers(0, 256, n, dtype=np.uint64))
    if name == "top_byte":  # differ only in the top byte (sign bit clear; the low exponent nibble keeps them finite)
        return _bits((rng.integers(0, 128, n, dtype=np.uint64) << np.uint64(56)) | np.uint64(0x000123456789ABCD))
    raise ValueError(name)


FAMILIES = ["distinct", "equal", "tie_at_pivot", "many_ties", "sentinel0", "sentinel50", "sentinel100", "signed_zero",
            "subnormal_inf", "low_byte", "top_byte"]
# families whose pivot sits in a tie group of hundreds to all of the items: at 100 000 items their O(n) index count per tied item
# takes minutes, so they stop at 20 000 (all-equal values at quantile 0.5 only)
HEAVY_TIES = ("equal", "signed_zero", "subnormal_inf", "low_byte", "top_byte")


def _cases(sizes=SIZES, blocks=BLOCKS):
    """[(label, values, oid, [(block, min_groups, quantile)])]: every size x family x tie-break index; up to 8193 items every
    quantile with min_groups N, N + 1 and 0 on every block size; past it every quantile with min_groups 0 and the two boundaries
    at 0.5, 100 000 items on 256 and 512 threads only and without the HEAVY_TIES families"""
    rng = np.random.Generator(np.random.MT19937(20261019))
    out = []
    for n in sizes:
        for fam in FAMILIES:
            v = _family(fam, n, rng)
            N = int((v >= 0).sum())
            for perm in (False, True):
                oid = rng.permutation(n).astype(np.int32) if perm else np.arange(n, dtype=np.int32)
                if n <= 8193:
                    runs = [(b, mg, q) for b in blocks for q in QUANTILES for mg in (N, N + 1, 0)]
                elif fam in HEAVY_TIES:
                    runs = [(b, 0, 0.5) for b in blocks] if fam == "equal" and n <= 20000 else []
                    if fam != "equal" and n <= 20000:
                        runs = [(b, 0, q) for b in blocks for q in QUANTILES] + [(b, mg, 0.5) for b in blocks for mg in (N, N + 1)]
                else:
                    bs = [b for b in blocks if n <= 20000 or b >= 256]
                    runs = [(b, 0, q) for b in bs for q in QUANTILES] + [(b, mg, 0.5) for b in bs for mg in (N, N + 1)]
                if not runs:
                    continue
                out.append(("%s n=%d oid=%s" % (fam, n, "perm" if perm else "id"), v, oid, runs))
    return out


# ---- CPU ------------------------------------------------------------------------------------------------------------------------
def test_reference_matches_oracle(oracle):
    """the reference equals the oracle's TrimmerQuantile (qsort by value, then index) on every case the oracle takes: its input
    is the valid values in tie-break order, and the caller's min_residual_groups rule (robust_solving.cpp:19-21)"""
    checked = ties = 0
    for label, v, oid, runs in _cases(sizes=[n for n in SIZES if n <= 8193], blocks=[512]):
        valid = np.nonzero(v >= 0)[0]
        by_oid = valid[np.argsort(oid[valid], kind="stable")]  # the oracle breaks ties by position
        vals = v[by_oid]
        ties += len(vals) - len(np.unique(vals + 0.0))
        for _, mg, q in runs:
            want = np.zeros(len(v), bool)
            if len(vals) and len(vals) >= mg:
                n_rej, rej = oracle.trimmer_quantile(vals, q)
                want[by_oid] = rej
                assert n_rej == rej.sum()
            got = trim_reference(v, oid, q, mg)
            assert np.array_equal(got, want), (label, mg, q)
            checked += 1
    assert checked == 16 * len(FAMILIES) * 2 * len(QUANTILES) * 3 and ties > 10000, (checked, ties)


def test_reference_edges():
    """the rule's edges on hand-made cases"""
    v = np.array([0.5, -1.0, 0.5, np.nan, 0.25, -0.0, 0.0, 0.5])
    # valid in (value, oid) order: 5 (-0.0), 6 (+0.0), 4, 0, 2, 7
    assert list(np.nonzero(trim_reference(v, np.arange(8), 0.5, 0))[0]) == [0, 2, 7]           # num = 3
    assert list(np.nonzero(trim_reference(v, np.arange(8), 0.2, 0))[0]) == [0, 2, 4, 6, 7]     # num = 1: +0.0 after -0.0
    assert list(np.nonzero(trim_reference(v, np.arange(8)[::-1], 0.2, 0))[0]) == [0, 2, 4, 5, 7]  # ... unless its oid is smaller
    assert not trim_reference(v, np.arange(8), 0.5, 7).any()   # N = 6 < min_groups
    assert trim_reference(v, np.arange(8), 0.5, 6).sum() == 3   # N == min_groups trims
    assert not trim_reference(v, np.arange(8), 1.0, 0).any()    # num = N
    assert trim_reference(v, np.arange(8), 1.0 - 2.0 ** -53, 0).sum() == 1  # 6 * (1 - 2^-53) rounds below 6: num = N - 1
    assert trim_reference(v, np.arange(8), 0.0, 0).sum() == 6   # num = 0: every valid item
    assert trim_reference(v, np.arange(8), -0.1, 0).sum() == 6  # what the device does with a negative quantile
    assert not trim_reference(np.full(5, -1.0), np.arange(5), 0.0, 0).any()


def test_reference_detects_a_wrong_rule():
    """the comparison can fail: ties broken by descending index, and num off by one, disagree with the reference on the tie
    families (the masks differ at the pivot)"""
    diff_desc = diff_off = 0
    for label, v, oid, runs in _cases(sizes=[33, 257, 2049, 4097], blocks=[512]):
        order = _order(v, oid)
        order_desc = _order(v, -oid.astype(np.int64))
        for _, mg, q in runs:
            ref = _reject_from_order(len(v), order, q, mg)
            diff_desc += not np.array_equal(_reject_from_order(len(v), order_desc, q, mg), ref)
            diff_off += not np.array_equal(_reject_from_order(len(v), order, q, mg, off_by=1), ref)
    assert diff_desc > 100 and diff_off > 500, (diff_desc, diff_off)


def _compile_driver(out_dir):
    exe = os.path.join(str(out_dir), "trim_select_driver")
    subprocess.check_call([NVCC] + NVFLAGS + ["-ccbin", "/usr/bin/g++", "-I", CSRC, "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "trim_select_driver.cu"), "-o", exe])
    return exe


def test_driver_compiles_for_sm90a(tmp_path):
    exe = _compile_driver(tmp_path)
    sass = subprocess.run([os.path.join(os.path.dirname(NVCC), "cuobjdump"), "--list-elf", exe], capture_output=True, text=True,
                          check=True).stdout
    assert "sm_90a" in sass


def test_quantile_rule_covers_every_quantile_option():
    """every *_quantile field of kba_options is checked by the one rule (kba_api.cu quantile_check), which solve_options_check
    and the frame path's options_check call"""
    from limo_b200.capi_types import KbaOptions
    fields = [f for f, _ in KbaOptions._fields_ if f.endswith("_quantile")]
    with open(os.path.join(ROOT, "include", "kba_b200.h")) as f:
        header = f.read()
    assert sorted(fields) == sorted(set(re.findall(r"double\s+(\w+_quantile)\s*;", header))) and len(fields) == 3
    with open(os.path.join(CSRC, "kba_api.cu")) as f:
        src = f.read()
    body = src[src.index("static int quantile_check("):]
    body = body[:body.index("\n}\n")]
    assert sorted(re.findall(r'\{"(\w+)", o->(\w+)\}', body)) == sorted((f, f) for f in fields)
    for caller in ("static int solve_options_check(", "static int options_check("):
        fn = src[src.index(caller):]
        assert "quantile_check(o" in fn[:fn.index("\n}\n")], caller


# ---- GPU: the driver ------------------------------------------------------------------------------------------------------------
def _write_cases(path, cases):
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(cases)))
        for _, v, oid, runs in cases:
            f.write(struct.pack("<i", len(v)))
            f.write(np.ascontiguousarray(v, "<f8").tobytes())
            f.write(np.ascontiguousarray(oid, "<i4").tobytes())
            f.write(struct.pack("<i", len(runs)))
            for b, mg, q in runs:
                f.write(struct.pack("<iid", b, mg, q))


@pytest.mark.gpu
def test_driver_matches_reference(tmp_path):
    """every mask of trim_select_group, on 32-, 256- and 512-thread CTAs, equals the exact-rank reference; the all-equal
    20 000-item selection is timed"""
    exe = _compile_driver(tmp_path)
    cases = _cases()
    _write_cases(tmp_path / "cases.bin", cases)
    subprocess.run([exe, str(tmp_path / "cases.bin"), str(tmp_path / "masks.bin")], check=True, timeout=400,
                   env=dict(os.environ, TRIM_DRIVER_PROGRESS="1"))
    data = np.fromfile(tmp_path / "masks.bin", np.uint8)
    pos = n_runs = wrong_desc = wrong_off = 0
    times = {}
    for label, v, oid, runs in cases:
        n = len(v)
        order = _order(v, oid)
        order_desc = _order(v, -oid.astype(np.int64))
        for b, mg, q in runs:
            ms = float(data[pos:pos + 4].view(np.float32)[0])
            got = data[pos + 4:pos + 4 + n].astype(bool)
            pos += 4 + n
            want = _reject_from_order(n, order, q, mg)
            assert np.array_equal(got, want), "%s block %d min_groups %d quantile %r: %d of %d differ" % (
                label, b, mg, q, (got != want).sum(), n)
            wrong_desc += not np.array_equal(got, _reject_from_order(n, order_desc, q, mg))
            wrong_off += not np.array_equal(got, _reject_from_order(n, order, q, mg, off_by=1))
            if label == "equal n=20000 oid=id" and mg == 0:
                times[b] = ms
            n_runs += 1
    assert pos == len(data)
    # the masks tell a wrong tie order and num off by one apart from the rule
    assert wrong_desc > 100 and wrong_off > 1000, (wrong_desc, wrong_off)
    print("trim_select_group: %d selections equal to the reference; all-equal 20 000 items at quantile 0.5: %s" % (
        n_runs, ", ".join("%d threads %.3f ms" % (b, times[b]) for b in sorted(times))))


@pytest.mark.gpu
def test_driver_negative_quantile_rejects_everything(tmp_path):
    """what an unchecked negative quantile did: num < 0, no bin holds rank num, the pivot stays 0 and every landmark with a
    residual is rejected (the reason the options refuse it)"""
    exe = _compile_driver(tmp_path)
    v = np.random.default_rng(5).uniform(0, 1, 3000)
    v[::7] = -1.0
    cases = [("negative quantile", v, np.arange(len(v), dtype=np.int32), [(b, 0, -0.05) for b in BLOCKS])]
    _write_cases(tmp_path / "cases.bin", cases)
    subprocess.check_call([exe, str(tmp_path / "cases.bin"), str(tmp_path / "masks.bin")])
    data = np.fromfile(tmp_path / "masks.bin", np.uint8)
    for i in range(len(BLOCKS)):
        got = data[i * (4 + len(v)) + 4:(i + 1) * (4 + len(v))].astype(bool)
        assert np.array_equal(got, v >= 0)


# ---- GPU: end to end, with ties exact by construction ---------------------------------------------------------------------------
def _split_pairs(rej, pairs):
    """how many duplicate pairs (i, j) the trimming separated: one kept, one rejected -- only a tie at the pivot does that"""
    rej = np.asarray(rej, bool)
    return int(sum(rej[i] != rej[j] for i, j in pairs))


def _duplicated_window(win, every=3):
    """win with every `every`-th landmark followed by a copy of itself (position, weight, observations), landmarks fixed.
    Returns (window, [(original, copy)] in the new indices)."""
    from limo_b200.capi_types import Window
    src, pairs = [], []
    for j in range(win.n_lm):
        src.append(j)
        if j % every == 0:
            src.append(j)
            pairs.append((len(src) - 2, len(src) - 1))
    src = np.array(src)
    ptr = win.lm_obs_ptr
    obs = np.concatenate([np.arange(ptr[j], ptr[j + 1]) for j in src]).astype(np.int64)
    new_ptr = np.concatenate([[0], np.cumsum(np.diff(ptr)[src])]).astype(np.int32)
    w = Window(win.kf_pose, win.kf_fixed, win.cam_intr, win.cam_pose, win.lm_pos[src], win.lm_weight[src], new_ptr, win.obs_kf[obs],
               win.obs_u[obs], win.obs_v[obs], win.obs_d[obs], obs_cam=None if win.obs_cam is None else win.obs_cam[obs],
               landmarks_fixed=True)
    return w, pairs


def _window_case(which):
    from limo_b200 import synth
    if which == "1500":
        win = synth.make_window(2, seed=7102, n_kf=8, n_lm=1130, n_obs=11000)
    else:  # past the 4096 keys a 512-thread CTA holds in registers
        win = synth.make_window(2, seed=7102, n_kf=8, n_lm=3300, n_obs=33000)
    return _duplicated_window(win)


def _window_opt(q_depth, q_repr):
    from limo_b200 import capi
    o = capi.default_options()
    o.depth_quantile, o.reprojection_quantile = q_depth, q_repr
    o.num_trim_rounds = 3
    o.solver_time_sec = 20.0
    return o


WINDOW_QUANTILES = {"1500": (0.5, 0.7), "4400": (0.5, 0.6)}


@pytest.fixture(scope="module")
def handle():
    from limo_b200 import capi
    h = capi.Handle(0)
    yield h
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["1500", "4400"])
def test_trim_select_ties_match_oracle_and_shards(handle, oracle, which):
    """k_trim_select on landmarks_fixed windows with duplicated landmarks: rejections equal to the oracle's, the solve to the
    suite's tolerances; the same window sharded over the in-process exchange: world 1 the plain solve's rejections and counts
    exactly, worlds 2 and 3 the same rejections, with a duplicate pair straddling a shard boundary"""
    from limo_b200 import parallel
    from tests.test_gpu_parity import _compare_solves
    from tests.test_shard_ground import _assert_close, _summary
    win, pairs = _window_case(which)
    opt = _window_opt(*WINDOW_QUANTILES[which])
    res = handle.solve_window(win, opt)
    ref = oracle.solve_window(win, opt)
    assert res.c.num_solves >= 4
    _compare_solves(res, ref, win, "tie window %s" % which)
    split = _split_pairs(res.lm_rejected[:win.n_lm], pairs)
    assert split > 0, "no pivot fell in a tie group"
    straddle = 0
    for world in (2, 3):
        for j0, _ in parallel.landmark_ranges(win.lm_obs_ptr, world)[1:]:
            straddle += any(j0 == b for _, b in pairs)
    assert straddle > 0, "no duplicate pair straddles a shard boundary"
    [(r1, j0, j1)] = parallel.solve_sharded_local(win, 1, opt)
    assert (j0, j1) == (0, win.n_lm)
    # one rank: the same decisions and counts as the plain solve; with constant landmarks the exchanged cost sums can differ
    # from the plain solve's in the last bit (the 1500-landmark window: 399.4415019456064 against ...0626 after three trimming
    # steps), so the costs and poses are held to rounding rather than bits
    assert _summary(r1) == _summary(res)
    assert np.array_equal(r1.lm_rejected[:win.n_lm], res.lm_rejected[:win.n_lm])
    for x, y in zip(r1.solves, res.solves):
        assert x.final_cost == pytest.approx(y.final_cost, rel=1e-13)
    assert np.abs(r1.kf_pose - res.kf_pose).max() <= 1e-12
    for world in (2, 3):
        _assert_close(parallel.solve_sharded_local(win, world, opt), res, win)
    print("window %s: %d landmarks, %d pairs split by the trimming, %d rejected" % (which, win.n_lm, split, res.lm_rejected[:win.n_lm].sum()))


class _DupFrame(_Frame):
    """a tests/test_adjust_pose.py frame whose every third run is duplicated into a new slot (after the window's landmarks) with
    the same position, weight and measurements; pairs: (run, its copy's run)"""

    def __init__(self, seed, **kw):
        super().__init__(seed, **kw)
        n = self.win.n_lm
        slots, starts = self.runs()
        dup = [r for r in range(len(slots)) if slots[r] % 3 == 0]
        rows = np.concatenate([np.arange(starts[r], starts[r + 1]) for r in dup]).astype(np.int64)
        reps = np.diff(starts)[dup]
        self.lm = np.concatenate([self.lm, np.repeat(n + np.arange(len(dup)), reps)]).astype(np.int32)
        self.cam, self.u, self.v, self.d = (np.concatenate([a, a[rows]]) for a in (self.cam, self.u, self.v, self.d))
        self.lm_pos = np.concatenate([self.lm_pos, self.lm_pos[slots[dup]]])
        self.lm_weight = np.concatenate([self.lm_weight, self.lm_weight[slots[dup]]])
        self.pairs = [(r, len(slots) + i) for i, r in enumerate(dup)]
        self.n_slots = n + len(dup)

    def track(self, h):
        from limo_b200 import capi
        t = capi.Track(h, self.cam_intr, self.cam_pose, max_keyframes=3, max_landmarks=self.n_slots, max_measurements=1,
                       win_keyframes=3, win_landmarks=self.n_slots, win_observations=len(self.lm))
        t.set_landmarks(np.arange(self.n_slots, dtype=np.int32), pos=self.lm_pos, weight=self.lm_weight)
        return t


def _adjust_pose_case(h, oracle, fr, opt, label):
    """the frame on the store against kba_solve_window on the equivalent window (bit for bit) and the oracle"""
    from tests.test_gpu_parity import _compare_solves
    t = fr.track(h)
    try:
        a = t.adjust_pose(opt=opt, **fr.args())
    finally:
        t.close()
    win = fr.window()
    b = h.solve_window(win, opt)
    _equal_to_general(a, b, win.n_lm, label)
    a.lm_pos[:win.n_lm] = win.lm_pos  # constant landmarks: the track path does not return them
    _compare_solves(a, oracle.solve_window(win, opt), win, "adjust_pose ties " + label)
    return a.lm_rejected[:win.n_lm].astype(bool)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["mono", "rig", "min_groups"])
def test_adjust_pose_ties(handle, oracle, case):
    """k_adjust_pose (256 threads, 2048 keys in registers) on frames of more than 2048 runs with every third landmark duplicated,
    depth quantile 0.5: rejections bit for bit those of kba_solve_window on the equivalent window, and the oracle's.  min_groups:
    the depth group's landmark count exactly min_residual_groups (its first trimming step trims it) and one below (it does not)"""
    fr = _DupFrame(8101 + ["mono", "rig", "min_groups"].index(case), n_lm=5200, n_obs=52000, rig=case == "rig")
    slots, starts = fr.runs()
    n_runs = len(slots)
    assert n_runs > 2048
    opt = _opt(2, depth_quantile=0.5, reprojection_quantile=0.7, solver_time_sec=20.0)
    n_depth = int(sum((fr.d[starts[r]:starts[r + 1]] > 0).any() for r in range(n_runs)))
    if case != "min_groups":
        rej = _adjust_pose_case(handle, oracle, fr, opt, case)
    else:
        opt.min_residual_groups = n_depth
        rej = _adjust_pose_case(handle, oracle, fr, opt, "depth group at min_residual_groups")
        opt.min_residual_groups = n_depth + 1
        below = _adjust_pose_case(handle, oracle, fr, opt, "depth group one below min_residual_groups")
        assert not np.array_equal(rej, below)
    split = _split_pairs(rej, fr.pairs)
    print("adjust_pose %s: %d runs (%d with depth), %d pairs split, %d rejected" % (case, n_runs, n_depth, split, rej.sum()))
    if case != "rig":  # the rig frame's pivots miss the pairs: its ties are compared, but none decides
        assert split > 0, "no pivot fell in a tie group"


def _dup_track(h, win):
    """a track holding win's keyframes (slot k = keyframe k) and landmarks (slot j = landmark j)"""
    from limo_b200 import capi
    lm_of = np.repeat(np.arange(win.n_lm), np.diff(win.lm_obs_ptr)).astype(np.int32)
    t = capi.Track(h, win.cam_intr, win.cam_pose, max_keyframes=win.n_kf, max_landmarks=win.n_lm, max_measurements=win.n_obs,
                   win_keyframes=win.n_kf, win_landmarks=win.n_lm, win_observations=win.n_obs)
    t.set_landmarks(np.arange(win.n_lm, dtype=np.int32), pos=win.lm_pos, weight=win.lm_weight)
    for k in range(win.n_kf):
        sel = np.nonzero(win.obs_kf == k)[0]  # landmark-major: ascending slot
        t.push_keyframe(k, win.kf_pose[k], lm_of[sel], win.obs_u[sel], win.obs_v[sel], win.obs_d[sel])
    return t


def _quantile_in_tie(vals, pairs):
    """a quantile whose pivot rank lies inside a duplicate pair's tie group"""
    valid = np.nonzero(vals >= 0)[0]
    order = valid[np.lexsort((valid, vals[valid]))]
    rank = np.empty(len(vals), np.int64)
    rank[order] = np.arange(len(order))
    N = len(order)
    for i, j in sorted(pairs, key=lambda p: abs(rank[p[0]] - N // 2) if vals[p[0]] >= 0 else N):
        if vals[i] >= 0 and vals[i] == vals[j] and (vals[order] == vals[i]).sum() == 2:
            r = max(rank[i], rank[j])  # the second of the two: num = r keeps one, rejects the other
            q = (r + 0.5) / N
            assert int(float(N) * q) == r
            return q
    raise AssertionError("no tie group")


@pytest.mark.gpu
def test_evaluate_ties(handle):
    """k_ev_finish (512 threads) on a stored window of more than 4096 landmarks, every third duplicated: per track quantiles
    through the group _opts form, each putting the pivot inside a tie pair; the returned decisions equal the reference applied
    to the returned trimming values"""
    from limo_b200 import capi, synth
    base = synth.make_window(2, seed=7201, n_kf=8, n_lm=3300, n_obs=33000)
    win, pairs = _duplicated_window(base)
    assert win.n_lm > 4096
    tracks = [_dup_track(handle, win) for _ in range(2)]
    req = dict(kf_slots=np.arange(win.n_kf, dtype=np.int32), kf_fixed=win.kf_fixed, lm_slots=np.arange(win.n_lm, dtype=np.int32))
    grp = capi.TrackGroup(handle, tracks)
    try:
        ev0 = tracks[0].evaluate(**req)
        for key in ("trim_repr", "trim_depth"):  # the duplicates' values are the same bits
            v = ev0[key]
            assert all(v[i] == v[j] or (np.isnan(v[i]) and np.isnan(v[j])) for i, j in pairs), key
        q_r, q_d = _quantile_in_tie(ev0["trim_repr"], pairs), _quantile_in_tie(ev0["trim_depth"], pairs)
        opts = []
        for q_repr, q_depth, mg in ((q_r, q_d, 5), (0.5, 0.5, 0)):
            o = capi.default_options()
            o.reprojection_quantile, o.depth_quantile, o.min_residual_groups = q_repr, q_depth, mg
            opts.append(o)
        evs = grp.evaluate([req, req], opt=opts)
        for i, (ev, o) in enumerate(zip(evs, opts)):
            oid = np.arange(win.n_lm)
            for rk, tk, q in (("rejected_repr", "trim_repr", o.reprojection_quantile), ("rejected_depth", "trim_depth", o.depth_quantile)):
                assert np.array_equal(ev[tk], ev0[tk]), (i, tk)
                want = trim_reference(ev[tk], oid, q, o.min_residual_groups)
                assert np.array_equal(ev[rk], want), (i, rk, (ev[rk] != want).sum())
        split = _split_pairs(evs[0]["rejected_repr"], pairs) + _split_pairs(evs[0]["rejected_depth"], pairs)
        assert split >= 2, split
        print("evaluate: %d landmarks, %d pairs split at the chosen quantiles" % (win.n_lm, split))
    finally:
        grp.close()
        for t in tracks:
            t.close()


# ---- GPU: the quantile options are refused before any launch --------------------------------------------------------------------
BAD_QUANTILES = [("depth_quantile", -0.1), ("reprojection_quantile", math.nan), ("gp_quantile", 1.5), ("depth_quantile", -1e-300),
                 ("reprojection_quantile", math.inf)]


@pytest.mark.gpu
def test_bad_quantiles_are_refused_before_any_launch(handle):
    """kba_solve_window, a batch _opts call, Track.solve, Track.adjust_pose, Track.evaluate and a group _opts call refuse a NaN
    quantile or one outside [0, 1] with KBA_ERR_BAD_ARG (1), naming the field and a per-unit option's unit, and launch nothing;
    0 and 1 stay valid"""
    from limo_b200 import capi, synth
    from tests.test_track_group import _Drive
    win = synth.make_window(1)
    fr = _Frame(101, n_lm=400, n_obs=4000)
    ft = fr.track(handle)
    drv = _Drive(7, W=6, n_lm=300, n_obs=2500, steps=1)
    t, t2 = drv.make_track(handle), drv.make_track(handle)
    grp = capi.TrackGroup(handle, [t, t2])
    req = drv.request(0)
    good = capi.default_options()
    calls = [
        ("kba_solve_window", lambda o: handle.solve_window(win, o), ""),
        ("batch _opts", lambda o: handle.solve_batch([win, win], [good, o]), "window 1"),
        ("Track.solve", lambda o: t.solve(**req, opt=o), ""),
        ("Track.adjust_pose", lambda o: ft.adjust_pose(opt=o, **fr.args()), ""),
        ("Track.evaluate", lambda o: t.evaluate(**req, opt=o), ""),
        ("group solve _opts", lambda o: grp.solve([req, req], opt=[good, o]), "track 1"),
        ("group evaluate _opts", lambda o: grp.evaluate([req, req], opt=[good, o]), "track 1"),
    ]
    try:
        for field, value in BAD_QUANTILES:
            o = capi.default_options()
            setattr(o, field, value)
            for name, call, unit in calls:
                before = handle.counters().launches_total
                with pytest.raises(capi.KbaError, match="error 1.*%s.*kba_options\\.%s" % (unit, field)):
                    call(o)
                assert handle.counters().launches_total == before, (name, field, value)
        for q in (0.0, 1.0):  # the bounds stay valid
            o = _opt(1)
            o.depth_quantile = o.reprojection_quantile = o.gp_quantile = q
            handle.solve_window(win, o)
            ft.adjust_pose(opt=o, **fr.args())
            t.evaluate(**req, opt=o)
    finally:
        grp.close(); t.close(); t2.close(); ft.close()
