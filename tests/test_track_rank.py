"""The ranked landmark selection on the device-resident store -- kba_track_rank_landmarks / kba_track_solve_ranked and their group
forms -- against a restatement of the facade's ranking.

The restatement ranks the chain's quantities as LandmarkSelector::select does (chooseNearLmIds, chooseMiddleLmIds, chooseFarLmIds,
the AddDepth scheme's std::partial_sort) with a replay of libstdc++'s heap routines, so that ties fall as on the host.
test_restatement_equals_facade pins it to the facade and libstdc++ without a GPU (tests/cpp/test_facade_rank.cpp, host mode) on
tie-heavy cases; on the GPU the device must equal it, and a solve of the ranking must equal kba_track_solve on the same lists."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.test_track_select import Scene, _candidates, host_select
from tests.test_track_upkeep import cost_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_facade_rank")
NEG = -np.finfo(np.float64).max


# ---- the ranking, restated ----------------------------------------------------------------------------------------------------
def heap_keep(items, cap, less):
    """the elements std::partial_sort_copy (or std::partial_sort's __heap_select) keeps from `items` with comparator `less` and
    cap outputs: libstdc++'s __make_heap over the first cap, then __adjust_heap at the root for each later element that beats it"""
    a = list(items[:cap])
    n = len(a)

    def adjust(hole, value):
        top = second = hole
        while second < (n - 1) // 2:
            second = 2 * (second + 1)
            if less(a[second], a[second - 1]):
                second -= 1
            a[hole] = a[second]
            hole = second
        if (n & 1) == 0 and second == (n - 2) // 2:
            second = 2 * (second + 1)
            a[hole] = a[second - 1]
            hole = second - 1
        parent = (hole - 1) // 2
        while hole > top and less(a[parent], value):
            a[hole] = a[parent]
            hole = parent
            parent = (hole - 1) // 2
        a[hole] = value

    if cap <= 0 or n == 0:
        return []
    if n >= 2:
        for parent in range((n - 2) // 2, -1, -1):
            adjust(parent, a[parent])
    for x in items[cap:]:
        if less(x, a[0]):
            adjust(0, x)
    return a


def rank_quantities(near, flow, middle, far, seen, depth, caps, draws):
    """near: ids in near order; flow: id -> flow (NaN: none); middle / far: ids in candidate order; seen: id -> count; depth: per
    AddDepth entry (wanted, [(id, cost)] in arena order); caps (near, middle, far); draws: the random values.  Returns
    ({id: category}, draws used): 0 near, 1 middle, 2 far, 3 AddDepth only."""
    out = {}
    with_flow = [i for i in near if not np.isnan(flow[i])]
    for i in heap_keep(with_flow, min(caps[0], len(with_flow)), lambda x, y: flow[x] > flow[y]):
        out[i] = 0
    m = list(middle)
    for i in range(1, len(m)):
        j = int(draws[i - 1]) % (i + 1)
        if i != j:
            m[i], m[j] = m[j], m[i]
    for i in m[:caps[1]]:
        out[i] = 1
    for i in heap_keep(list(far), min(caps[2], len(far)), lambda x, y: seen[x] > seen[y]):
        out[i] = 2
    for wanted, pairs in depth:
        for i, _ in heap_keep(pairs, min(wanted, len(pairs)), lambda x, y: x[1] < y[1]):
            out.setdefault(i, 3)
    return out, max(len(middle) - 1, 0)


# ---- CPU: the restatement against the facade -----------------------------------------------------------------------------------
def _tie_cases():
    """all-far windows with 2-3 distinct seen values, repeated flows, repeated and -DBL_MAX costs, bins below, at and above their
    caps, middle bins of 0, 1 and 2 entries"""
    rng = np.random.default_rng(11)
    cases = []
    for k in range(60):
        n = int(rng.integers(1, 120))
        ids = np.sort(rng.choice(100000, n, replace=False)).tolist()
        kind = k % 6
        if kind == 0:  # everything far, few distinct seen values
            near, middle, far = [], [], ids
        else:
            lab = rng.integers(0, 3, n)
            near = [i for i, b in zip(ids, lab) if b == 0]
            rng.shuffle(near)
            middle = [i for i, b in zip(ids, lab) if b == 1][: [0, 1, 2, 1000][kind % 4]]
            far = [i for i, b in zip(ids, lab) if b == 2]
        flow = {i: float(rng.choice([np.nan, 1.0, 2.5, 2.5, 7.0, rng.uniform(0, 9)])) for i in near}
        seen = {i: int(rng.choice([2, 3, 5][: 2 + (k % 2)])) for i in far}
        caps = [int(rng.choice([0, 1, len(near), max(len(near) - 3, 0), 300])), int(rng.choice([0, 1, 2, 40])),
                int(rng.choice([0, 1, len(far), max(len(far) // 2, 1), 300]))]
        depth = []
        for _ in range(int(rng.integers(0, 4))):
            sub = [i for i in ids if rng.random() < 0.5]
            cost = [float(rng.choice([NEG, 3.0, 3.0, 4.5, float(np.float32(rng.uniform(0, 30)))])) for _ in sub]
            depth.append((int(rng.choice([0, 1, 5, 50, len(sub)])), list(zip(sub, cost))))
        cases.append(dict(near=near, flow=flow, middle=middle, far=far, seen=seen, depth=depth, caps=caps, seed=int(rng.integers(1, 2**31))))
    return cases


def _write_cases(cases, path):
    with open(path, "w") as f:
        for c in cases:
            f.write("case %d %d %d %d\n" % (*c["caps"], c["seed"]))
            f.write("near %d %s\n" % (len(c["near"]), " ".join("%d %s" % (i, float(c["flow"][i]).hex()) for i in c["near"])))
            f.write("middle %d %s\n" % (len(c["middle"]), " ".join(str(i) for i in c["middle"])))
            f.write("far %d %s\n" % (len(c["far"]), " ".join("%d %d" % (i, c["seen"][i]) for i in c["far"])))
            f.write("depth %d\n" % len(c["depth"]))
            for wanted, pairs in c["depth"]:
                f.write("entry %d %d %s\n" % (wanted, len(pairs), " ".join("%d %s" % (i, x.hex()) for i, x in pairs)))


def _build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])


def test_heap_keep_is_libstdcpp_partial_sort():
    """the heap keeps libstdc++'s tied elements, not the first ones (the case of test_track_upkeep's partial_sort restatement)"""
    c = list(enumerate([1.0, 2.0, 1.0, 1.0, 1.0, 1.0, 0.0, 1.0, 2.0]))
    assert {i for i, _ in heap_keep(c, 5, lambda x, y: x[1] < y[1])} == {0, 3, 4, 5, 6}


def test_restatement_equals_facade(tmp_path):
    _build()
    cases = _tie_cases()
    path = tmp_path / "cases.txt"
    _write_cases(cases, path)
    r = subprocess.run([EXE, "host", str(path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = {}
    for line in r.stdout.split("\n"):
        if line:
            tag, k, *rest = line.split()
            lines[(tag, int(k))] = rest
    seen = dict(tie_far=0, capped=0, uncapped=0, mid0=0, mid1=0, mid2=0, neg=0)
    for k, c in enumerate(cases):
        n_draws, *draws = [int(x) for x in lines[("R", k)]]
        ref, used = rank_quantities(c["near"], c["flow"], c["middle"], c["far"], c["seen"], c["depth"], c["caps"], draws)
        facade = dict(tuple(int(v) for v in x.split(":")) for x in lines[("C", k)])
        assert facade == ref, k
        assert used == n_draws, k
        far = c["far"]
        seen["tie_far"] += int(len(far) > c["caps"][2] > 0 and len({c["seen"][i] for i in far}) < len(far))
        seen["capped"] += int(len(far) > c["caps"][2])
        seen["uncapped"] += int(len(far) <= c["caps"][2])
        seen["mid%d" % min(len(c["middle"]), 2)] += 1
        seen["neg"] += sum(1 for _, p in c["depth"] for _, x in p if x == NEG)
    assert all(v > 0 for v in seen.values()), seen


def test_rank_struct_sizes_match_header(tmp_path):
    from limo_b200 import capi_types as T
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n",sizeof(kba_depth_entry),'
                    'sizeof(kba_rank_request),sizeof(kba_rank_out),sizeof(kba_ranked_request));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(T.KbaDepthEntry), C.sizeof(T.KbaRankRequest), C.sizeof(T.KbaRankOut), C.sizeof(T.KbaRankedRequest)]


def test_rank_null_arguments_need_no_device():
    _build()
    from limo_b200 import capi
    L = capi.lib()
    q, o = capi.KbaRankRequest(), capi.KbaRankOut()
    assert L.kba_track_rank_landmarks(None, C.byref(q), C.byref(o)) == 1
    assert L.kba_track_group_rank_landmarks(None, C.byref(q), C.byref(o)) == 1
    assert L.kba_track_solve_ranked(None, 0, None, None, None, None, None) == 1


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
CAPS = dict(max_near=40, max_middle=30, max_far=25)
VOX = dict(voxel_size=(0.5, 0.5, 0.3), roi_far=40.0, roi_middle=15.0)


def host_rank(sc, kf_list, cand, elig, depth, caps, draws):
    """the restatement on a Scene: host_select's quantities, limo's AddDepth costs, the ranking; returns (cand indices, categories)"""
    q = host_select(sc, kf_list, cand, VOX["voxel_size"], VOX["roi_far"], VOX["roi_middle"])
    n = len(cand)
    flow = {c: q["flow"][c] for c in range(n)}
    seen = {c: int(q["seen"][c]) for c in range(n)}
    middle = [c for c in range(n) if q["bin"][c] == 1]
    far = [c for c in range(n) if q["bin"][c] == 2]
    index = {lid: c for c, lid in enumerate(cand)}
    ent = []
    for ind, wanted in depth:
        if ind >= len(kf_list):
            continue
        k = kf_list[ind]
        pairs = [(index[lid], cost_of(sc.kf_pose[k], sc.lm_pos[lid])) for lid in sorted(sc.meas[k])
                 if lid in index and q["cheiral"][index[lid]] and elig[index[lid]]]
        ent.append((wanted, pairs))
    out, used = rank_quantities(list(q["near_order"]), flow, middle, far, seen, ent,
                                (caps["max_near"], caps["max_middle"], caps["max_far"]), draws)
    sel = sorted(out)
    return np.array(sel, np.int32), np.array([out[c] for c in sel], np.int8), used, len(middle)


def _track(h, sc, win_rows=0):
    from limo_b200 import capi
    n_meas = sum(len(ms) for d in sc.meas for ms in d.values())
    t = capi.Track(h, sc.cam_intr, sc.cam_pose, max_keyframes=sc.n_kf + 2, max_landmarks=len(sc.lm_pos), max_measurements=n_meas,
                   win_keyframes=sc.n_kf, win_landmarks=len(sc.lm_pos), win_observations=n_meas, win_ground=len(sc.lm_pos) if win_rows else 0,
                   win_rows=win_rows)
    order = np.argsort(sc.slot)
    t.set_landmarks(np.arange(len(sc.lm_pos), dtype=np.int32), pos=np.array(sc.lm_pos)[order], weight=np.ones(len(sc.lm_pos)))
    for k in range(sc.n_kf):
        lm, cam, u, v = [], [], [], []
        for lid in sorted(sc.meas[k]):
            for c, uu, vv in sc.meas[k][lid]:
                lm.append(sc.slot[lid]); cam.append(c); u.append(uu); v.append(vv)
        t.push_keyframe(k, sc.kf_pose[k], lm, u, v, np.full(len(lm), -1.0, np.float32), cam=cam)
    return t


def _request(sc, kf_list, rng):
    cand = _candidates(sc, kf_list)
    elig = (rng.random(len(cand)) < 0.4).astype(np.uint8)
    depth = [(i, 50 if i % 3 else 7) for i in range(len(kf_list) + 1)]  # one entry past the window: skipped
    return cand, elig, depth


def _bound(n, n_mid, caps, depth):
    return min(n, min(caps["max_near"], n) + min(caps["max_middle"], n_mid) + min(caps["max_far"], n) + sum(min(w, n) for _, w in depth))


@pytest.mark.gpu
@pytest.mark.parametrize("n_kf,rig", [(12, False), (12, True), (20, False), (20, True)])
def test_rank_matches_restatement(n_kf, rig):
    from limo_b200 import capi
    sc = Scene(n_kf + (3 if rig else 0), n_kf=n_kf, n_lm=1500, rig=rig)
    h = capi.Handle(0)
    t = _track(h, sc)
    rng = np.random.default_rng(n_kf)
    covered = dict(near=0, middle=0, far=0, depth=0, draws=0)
    for step in range(30):
        lo = step % 4
        kf_list = list(range(lo, n_kf - (step % 3)))
        cand, elig, depth = _request(sc, kf_list, rng)
        draws = rng.integers(0, 2**31 - 1, len(cand))
        caps = dict(max_near=int(rng.choice([0, 5, 40, 300])), max_middle=int(rng.choice([0, 3, 30])), max_far=int(rng.choice([1, 25, 300])))
        dev = t.rank_landmarks(kf_list, sc.slot[cand], elig=elig, draws=draws, depth=depth, **caps, **VOX)
        ref_c, ref_k, used, n_mid = host_rank(sc, kf_list, cand, elig, depth, caps, draws)
        assert np.array_equal(dev["cand"], ref_c), step
        assert np.array_equal(dev["category"], ref_k), step
        assert dev["n_draws"] == used
        assert dev["n_ground"] == int(elig[ref_c].sum())
        h2d, d2h, _ = t.transfer_bytes()
        n = len(cand)
        assert h2d == 4 * (len(kf_list) + n) + n + 8 * len(depth) + 8 + 4 * used
        assert d2h == 4 + 8 + 5 * _bound(n, n_mid, caps, depth)
        for cat in range(4):
            covered[("near", "middle", "far", "depth")[cat]] += int((dev["category"] == cat).sum())
        covered["draws"] += used
    assert all(v > 0 for v in covered.values()), covered
    t.close(); h.close()


@pytest.mark.gpu
def test_rank_transfer_counts_equal_the_formulas():
    from limo_b200 import capi
    sc = Scene(21, n_kf=12, n_lm=1200, rig=True)
    h = capi.Handle(0)
    t = _track(h, sc)
    rng = np.random.default_rng(3)
    kf_list = list(range(1, 12))
    cand, elig, depth = _request(sc, kf_list, rng)
    q = host_select(sc, kf_list, cand, VOX["voxel_size"], VOX["roi_far"], VOX["roi_middle"])
    n_mid = int((q["bin"] == 1).sum())
    assert n_mid > 1
    dev = t.rank_landmarks(kf_list, sc.slot[cand], elig=elig, draws=lambda n: rng.integers(0, 1000, n), depth=depth, **CAPS, **VOX)
    n = len(cand)
    h2d, d2h, _ = t.transfer_bytes()
    assert dev["n_draws"] == n_mid - 1
    assert h2d == 4 * (len(kf_list) + n) + n + 8 * len(depth) + 8 + 4 * (n_mid - 1)
    assert d2h == 4 + 8 + 5 * _bound(n, n_mid, CAPS, depth)
    t.close(); h.close()


@pytest.mark.gpu
def test_group_rank_equals_single_calls():
    from limo_b200 import capi
    h = capi.Handle(0)
    scs = [Scene(30 + i, n_kf=12 if i % 2 else 20, n_lm=800 + 300 * i, rig=bool(i % 2)) for i in range(4)]
    ts = [_track(h, sc) for sc in scs]
    g = capi.TrackGroup(h, ts)
    rng = np.random.default_rng(5)
    R_seen = {}
    for rnd in range(3):
        reqs, draws = [], []
        for i, sc in enumerate(scs):
            if (i + rnd) % 3 == 2:
                reqs.append(None)
                continue
            kf_list = list(range(rnd, sc.n_kf))
            cand, elig, depth = _request(sc, kf_list, rng)
            d = rng.integers(0, 2**31 - 1, len(cand))
            reqs.append(dict(kf_slots=kf_list, lm_slots=sc.slot[cand], elig=elig, depth=depth, draws=d, **CAPS, **VOX))
        out = g.rank_landmarks(reqs)
        # the header's transfer formulas over the W requests that do not sit out; R, one window's argument records, is a
        # constant of the library build: the same in every round
        h2d, d2h = g.transfer_bytes()
        live = [(i, r) for i, r in enumerate(reqs) if r is not None]
        W, up, down = len(live), 8 * len(live), 4 * len(live)
        for i, r in live:
            n, n_kf, nd = len(r["lm_slots"]), len(r["kf_slots"]), len(r["depth"])
            q = host_select(scs[i], r["kf_slots"], list(np.argsort(scs[i].slot)[r["lm_slots"]]), VOX["voxel_size"], VOX["roi_far"],
                            VOX["roi_middle"])
            n_mid = int((q["bin"] == 1).sum())
            assert out[i]["n_draws"] == max(n_mid - 1, 0)
            up += 4 * (n_kf + n) + n + 8 * nd + 4 * max(n_mid - 1, 0)
            down += 8 + 5 * _bound(n, n_mid, CAPS, r["depth"])
        assert d2h == down, rnd
        assert W > 1 and h2d > up and (h2d - up) % (W - 1) == 0, rnd
        R = (h2d - up) // (W - 1)
        assert R_seen.setdefault("R", R) == R, rnd
        for i, r in enumerate(reqs):
            if r is None:
                assert out[i] is None
                continue
            one = ts[i].rank_landmarks(**r)
            for key in ("cand", "category"):
                assert np.array_equal(out[i][key], one[key]), (rnd, i, key)
            assert (out[i]["n_ground"], out[i]["n_draws"]) == (one["n_ground"], one["n_draws"])
    g.close()
    for t in ts:
        t.close()
    h.close()


@pytest.mark.gpu
def test_rank_rejects_bad_requests_and_writes_nothing():
    from limo_b200 import capi
    sc = Scene(9, n_kf=12, n_lm=600, rig=False)
    h = capi.Handle(0)
    t = _track(h, sc)
    kf_list = list(range(12))
    cand = sc.slot[_candidates(sc, kf_list)]
    n = len(cand)
    for kw, msg in ((dict(kf_slots=[], lm_slots=cand), "no keyframes"), (dict(kf_slots=[1, 1], lm_slots=cand), "listed twice"),
                    (dict(kf_slots=kf_list, lm_slots=cand, max_far=-1), "negative"),
                    (dict(kf_slots=kf_list, lm_slots=cand, depth=[(-1, 5)]), "negative"),
                    (dict(kf_slots=kf_list, lm_slots=cand, depth=[(0, 1)] * 1025), "1024"),
                    (dict(kf_slots=kf_list, lm_slots=cand, draws=None), "draw"),
                    (dict(kf_slots=kf_list, lm_slots=cand, draws=np.zeros(1, np.int64)), "draw function failed")):
        q, o, (c, k, *keep), _done = t._rank_request(**kw)
        c[:] = -7
        k[:] = -7
        o.n_sel = o.n_ground = o.n_draws = -7
        with pytest.raises(capi.KbaError, match=msg):
            capi._check(capi.lib().kba_track_rank_landmarks(t._p, C.byref(q), C.byref(o)))
        assert (c == -7).all() and (k == -7).all() and (o.n_sel, o.n_ground, o.n_draws) == (-7, -7, -7)
        with pytest.raises(capi.KbaError, match="no ranking"):  # a failed draw leaves no ranking behind
            t.solve_ranked(kf_list, np.r_[[1], np.zeros(11, np.uint8)])
    assert n > 0
    t.close(); h.close()


@pytest.mark.gpu
def test_group_rank_draw_failure_names_its_track():
    """a group of three whose track 0 sits out and whose track 2's draws are too short: the error names track 2 (not its index
    among the requests that run), nothing is written, and neither running track keeps a ranking"""
    from limo_b200 import capi
    h = capi.Handle(0)
    scs = [Scene(41, n_kf=12, n_lm=900, rig=False), Scene(42, n_kf=12, n_lm=1000, rig=True), Scene(21, n_kf=12, n_lm=1200, rig=True)]
    ts = [_track(h, sc) for sc in scs]
    g = capi.TrackGroup(h, ts)
    kf_list = list(range(1, 12))
    cands = [scs[i].slot[_candidates(scs[i], kf_list)] for i in range(3)]
    q2 = host_select(scs[2], kf_list, _candidates(scs[2], kf_list), VOX["voxel_size"], VOX["roi_far"], VOX["roi_middle"])
    assert (q2["bin"] == 1).sum() > 1  # track 2 needs draws
    rng = np.random.default_rng(11)
    ts[1].rank_landmarks(kf_list, cands[1], draws=rng.integers(0, 2**31 - 1, len(cands[1])), **CAPS, **VOX)  # a ranking to lose
    reqs, outs = (capi.KbaRankRequest * 3)(), (capi.KbaRankOut * 3)()
    keep = []
    for i, draws in ((1, rng.integers(0, 2**31 - 1, len(cands[1]))), (2, np.zeros(0, np.int64))):
        q, o, (c, k, *lists), _done = ts[i]._rank_request(kf_list, cands[i], draws=draws, **CAPS, **VOX)
        c[:] = -7
        k[:] = -7
        o.n_sel = o.n_ground = o.n_draws = -7
        reqs[i], outs[i] = q, o
        keep.append((i, c, k, lists))
    outs[0].n_sel = outs[0].n_ground = outs[0].n_draws = -7
    assert capi.lib().kba_track_group_rank_landmarks(g._p, reqs, outs) == 1  # KBA_ERR_BAD_ARG
    msg = capi.lib().kba_last_error().decode()
    assert "kba_track_group_rank_landmarks" in msg and "track 2: " in msg, msg
    for i in range(3):
        assert (outs[i].n_sel, outs[i].n_ground, outs[i].n_draws) == (-7, -7, -7), i
    for i, c, k, _ in keep:
        assert (c == -7).all() and (k == -7).all(), i
        with pytest.raises(capi.KbaError, match="no ranking"):
            ts[i].solve_ranked(kf_list, np.r_[[1], np.zeros(10, np.uint8)])
    g.close()
    for t in ts:
        t.close()
    h.close()


def _same_result(a, b):
    for key in ("kf_pose", "kf_plane", "lm_pos"):
        assert np.array_equal(getattr(a, key).view(np.int64), getattr(b, key).view(np.int64)), key
    assert np.array_equal(a.lm_rejected, b.lm_rejected)
    assert (a.c.initial_cost, a.c.final_cost, a.c.num_solves, a.c.status) == (b.c.initial_cost, b.c.final_cost, b.c.num_solves, b.c.status)
    for s in range(a.c.num_solves):
        x, y = a.c.solves[s], b.c.solves[s]
        assert (x.initial_cost, x.final_cost, x.num_iterations, x.num_residual_blocks) == (y.initial_cost, y.final_cost, y.num_iterations,
                                                                                         y.num_residual_blocks)


@pytest.mark.gpu
@pytest.mark.parametrize("n_kf,win_rows,ground", [(12, 0, False), (20, 201, True)])
def test_solve_ranked_equals_solve(n_kf, win_rows, ground):
    """kba_track_solve_ranked equals kba_track_solve on the same ranked list (and its ground candidates), alone and in a group; a
    solve makes the ranking stale"""
    from limo_b200 import capi
    h = capi.Handle(0)
    scs = [Scene(50 + i, n_kf=n_kf, n_lm=900, rig=False) for i in range(2)]
    a = [_track(h, sc, win_rows) for sc in scs]
    b = [_track(h, sc, win_rows) for sc in scs]
    g = capi.TrackGroup(h, a)
    rng = np.random.default_rng(n_kf)
    kf_list = list(range(n_kf))
    fixed = np.r_[[1, 1], np.zeros(n_kf - 2)].astype(np.uint8)
    opt = capi.default_options()
    opt.solver_time_sec = 20.0
    scal = dict(plane_reg_weight=-1.0) if ground else {}
    ranks = []
    for sc, ta in zip(scs, a):
        cand, elig, depth = _request(sc, kf_list, rng)
        d = rng.integers(0, 2**31 - 1, len(cand))
        r = ta.rank_landmarks(kf_list, sc.slot[cand], elig=elig, depth=depth, draws=d, **CAPS, **VOX)
        ranks.append((np.asarray(cand)[r["cand"]], elig[r["cand"]], r))
    res_a = g.solve_ranked([dict(kf_slots=kf_list, kf_fixed=fixed, ground=ground, **scal) for _ in ranks], opt=opt)
    for (lids, el, r), sc, tb, ra in zip(ranks, scs, b, res_a):
        extra = dict(gp_lm=np.flatnonzero(el).astype(np.int32)) if ground and el.any() else {}
        rb = tb.solve(kf_list, fixed, sc.slot[lids], opt=opt, **extra, **scal)
        assert ra.c.status == 0 and rb.c.status == 0
        _same_result(ra, rb)
    with pytest.raises(capi.KbaError, match="stale"):
        a[0].solve_ranked(kf_list, fixed)
    # alone: rank again (the store moved) on both, then the single ranked solve against the single solve
    sc, ta, tb = scs[0], a[0], b[0]
    cand, elig, depth = _request(sc, kf_list, rng)
    d = rng.integers(0, 2**31 - 1, len(cand))
    r = ta.rank_landmarks(kf_list, sc.slot[cand], elig=elig, depth=depth, draws=d, **CAPS, **VOX)
    lids, el = np.asarray(cand)[r["cand"]], elig[r["cand"]]
    with pytest.raises(capi.KbaError, match="differ"):
        ta.solve_ranked(kf_list[1:], fixed[1:])
    ra = ta.solve_ranked(kf_list, fixed, opt=opt, ground=ground, **scal)
    extra = dict(gp_lm=np.flatnonzero(el).astype(np.int32)) if ground and el.any() else {}
    rb = tb.solve(kf_list, fixed, sc.slot[lids], opt=opt, **extra, **scal)
    _same_result(ra, rb)
    ta.rank_landmarks(kf_list, sc.slot[cand], elig=elig, depth=depth, draws=d, **CAPS, **VOX)
    ta.set_landmarks([0], pos=[[0.0, 0.0, 5.0]])
    with pytest.raises(capi.KbaError, match="stale"):
        ta.solve_ranked(kf_list, fixed)
    g.close()
    for t in a + b:
        t.close()
    h.close()


@pytest.mark.gpu
def test_facade_drive_rank_equals_host_select():
    """tests/cpp/test_facade_rank in device mode: limo's chain over 12- and 20-keyframe facade drives mirrored into a track; at
    every step kba_track_rank_landmarks with a std::rand draw function equals the host select() seeded the same way, categories
    included, and leaves std::rand() where select() leaves it"""
    assert os.path.exists(EXE), "build it with make -C limo_b200/csrc facade"
    r = subprocess.run([EXE, "device"], capture_output=True, text=True, timeout=1200)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
