"""The Python binding of the track calls, without a GPU: capi.lib is replaced by a stub that records what each C call receives.

For every store call, Track.X(**r) and TrackGroup.X([None, r]) must hand the C library the same request: the structs field by
field and the arrays behind their pointers by content.  The group's entry 0 must carry the ABI's sit-out encoding, and a
request that the group call would read as a sit-out, or that has a key the single call does not take, must fail before any C
call."""
import ctypes as C

import numpy as np
import pytest

from limo_b200 import capi
from limo_b200.capi_types import (KbaCreateRequest, KbaDeactivateRequest, KbaDepthRequest, KbaFlowRequest, KbaLandmarkWrite,
                                  KbaPoseWrite, KbaPushRequest, KbaRankedRequest, KbaRankRequest, KbaReclaimRequest, KbaSelectRequest,
                                  KbaTrackFrame, KbaTrackRequest, KbaWindow)

KBA_WINDOW = "window"
N = "n_meas"
# pointer fields of each request: (bytes per element, element count: a field of the request or a number); KBA_WINDOW: a kba_window
POINTERS = {
    KbaPushRequest: dict(pose7=(8, 7), plane4=(8, 4), lm_slot=(4, N), cam=(4, N), u=(4, N), v=(4, N), d=(4, N)),
    KbaLandmarkWrite: dict(lm_slot=(4, "n"), pos3=(24, "n"), weight=(8, "n")),
    KbaPoseWrite: dict(kf_slot=(4, "n"), pose7s=(56, "n"), plane4s=(32, "n")),
    KbaSelectRequest: dict(kf_slot=(4, "n_kf"), lm_slot=(4, "n_cand"), params=(40, 1)),
    KbaCreateRequest: dict(kf_slot=(4, "n_kf"), lm_slot=(4, "n_new")),
    KbaDeactivateRequest: dict(kf_slot=(4, "n_kf"), lm_slot=(4, "n_lm")),
    KbaDepthRequest: dict(kf_slot=(4, "n_kf"), lm_slot=(4, "n_elig")),
    KbaFlowRequest: dict(lm_slot=(4, N), cam=(4, N), u=(4, N), v=(4, N)),
    KbaReclaimRequest: dict(),
    KbaRankRequest: dict(kf_slot=(4, "n_kf"), lm_slot=(4, "n_cand"), elig=(1, "n_cand"), params=(40, 1), depth=(8, "n_depth")),
    KbaTrackRequest: dict(kf_slot=(4, "n_kf"), kf_fixed=(1, "n_kf"), lm_slot=(4, "n_lm"), sel=KBA_WINDOW),
    KbaRankedRequest: dict(kf_slot=(4, "n_kf"), kf_fixed=(1, "n_kf"), sel=KBA_WINDOW),
    KbaTrackFrame: dict(pose7=(8, 7), lm_slot=(4, N), cam=(4, N), u=(4, N), v=(4, N), d=(4, N)),
    KbaWindow: dict(kf_fixed=(1, "n_kf"), lm_weight=(8, "n_lm"), gp_lm=(4, "n_gp"), gp_kf=(4, "n_gp"), gp_weight=(8, "n_gp")),
}


def _address(v):
    if v is None or isinstance(v, int):
        return v or None
    return C.cast(v, C.c_void_p).value


def _decode(struct, get):
    """the request of type struct whose field f is get(f), its pointers replaced by the bytes they point to (None: NULL)"""
    d = {}
    for f, t in struct._fields_:
        v = get(f)
        if f in POINTERS[struct]:
            a = _address(v)
            if a is None:
                d[f] = None
            elif POINTERS[struct][f] == KBA_WINDOW:
                w = KbaWindow.from_address(a)
                d[f] = _decode(KbaWindow, lambda g: getattr(w, g))
            else:
                size, count = POINTERS[struct][f]
                d[f] = C.string_at(a, size * (count if isinstance(count, int) else d[count]))
        elif issubclass(t, (C._Pointer, C.c_void_p)):
            d[f] = _address(v) is not None
        elif issubclass(t, C._CFuncPtr):
            d[f] = bool(v)
        elif issubclass(t, C.Array):
            d[f] = list(v)
        else:
            d[f] = v
    return d


def _out(o):
    """an output struct: its counts and capacities, and which of its pointers are set"""
    return {f: (_address(getattr(o, f)) is not None) if issubclass(t, (C._Pointer, C.c_void_p)) else
            (list(getattr(o, f)) if issubclass(t, C.Array) else getattr(o, f)) for f, t in o._fields_ if f != "solves"}


# call -> (group method, request struct, the single call's arguments after the track: flat request fields, or None: a request
# struct by reference; where its output is among them, or None)
CALLS = {
    "push_keyframe": ("push_keyframes", KbaPushRequest, ["kf_slot", "pose7", "plane4", "n_meas", "lm_slot", "cam", "u", "v", "d"], None),
    "set_landmarks": ("set_landmarks", KbaLandmarkWrite, ["n", "lm_slot", "pos3", "weight"], None),
    "set_keyframe_poses": ("set_keyframe_poses", KbaPoseWrite, ["n", "kf_slot", "pose7s", "plane4s"], None),
    "select_landmarks": ("select_landmarks", KbaSelectRequest, ["n_kf", "kf_slot", "n_cand", "lm_slot", "params"], 6),
    "create_landmarks": ("create_landmarks", KbaCreateRequest, None, 2),
    "deactivate_keyframes": ("deactivate_keyframes", KbaDeactivateRequest, None, 2),
    "depth_costs": ("depth_costs", KbaDepthRequest, None, 2),
    "frame_flow": ("frame_flow", KbaFlowRequest, None, 2),
    "reclaim_landmarks": ("reclaim_landmarks", KbaReclaimRequest, None, 2),
    "rank_landmarks": ("rank_landmarks", KbaRankRequest, None, 2),
    "solve": ("solve", KbaTrackRequest, ["n_kf", "kf_slot", "kf_fixed", "n_lm", "lm_slot", "sel"], 8),
    "solve_ranked": ("solve_ranked", KbaRankedRequest, ["n_kf", "kf_slot", "kf_fixed", "sel"], 6),
    "adjust_pose": ("adjust_pose", KbaTrackFrame, None, 3),
}


def _requests():
    rng = np.random.default_rng(5)
    f = lambda n: rng.random(n).astype(np.float32)  # noqa: E731
    lm = np.array([2, 3, 5, 8, 9])
    return {
        "push_keyframe": dict(slot=3, pose7=rng.random(7), lm_slot=lm, u=f(5), v=f(5), d=f(5), cam=[0, 1, 0, 0, 1], plane4=rng.random(4)),
        "set_landmarks": dict(lm_slot=lm, pos=rng.random((5, 3)), weight=rng.random(5)),
        "set_keyframe_poses": dict(kf_slots=[1, 4], pose7s=rng.random((2, 7))),
        "select_landmarks": dict(kf_slots=[0, 1, 2], lm_slots=lm, voxel_size=(0.5, 0.5, 0.3), roi_far=40.0),
        "create_landmarks": dict(kf_slots=[0, 1, 2], kf_new=2, lm_slots=[4, 7]),
        "deactivate_keyframes": dict(kf_slots=[0, 1, 2], lm_slots=[1, 2, 3], min_window=3),
        "depth_costs": dict(kf_slots=[0, 1], lm_slots=[1, 2, 3], cap=4),
        "frame_flow": dict(kf_last=2, lm_slot=[1, 1, 2], u=f(3), v=f(3), cam=[0, 1, 0], min_median_flow=3.0),
        "reclaim_landmarks": dict(lo=3, hi=9, evict=True),
        "rank_landmarks": dict(kf_slots=[0, 1, 2], lm_slots=lm, elig=[1, 0, 1, 0, 1], depth=[(0, 3)], draws=np.arange(4), max_far=7),
        "solve": dict(kf_slots=[0, 1, 2], kf_fixed=[1, 0, 0], lm_slots=lm, scale_kf1=2, scale_weight=1.5, gp_lm=[0, 2]),
        "solve_ranked": dict(kf_slots=[0, 1, 2], kf_fixed=[1, 0, 0], ground=True, plane_reg_weight=-1.0),
        "adjust_pose": dict(pose7=rng.random(7), lm_slot=[1, 1, 2], u=f(3), v=f(3), d=f(3), cam=[0, 1, 0],
                            speed=dict(weight=2.0, dt=0.1, v_before=(1, 2, 3), T_origin_before=rng.random(7))),
    }


# a request the group call would read as a sit-out: a KbaError of the binding (reclaim: an empty result, see below)
SITS_OUT = {"push_keyframe": dict(slot=-1), "select_landmarks": dict(kf_slots=[]), "create_landmarks": dict(kf_slots=[]),
            "deactivate_keyframes": dict(kf_slots=[]), "depth_costs": dict(kf_slots=[]), "frame_flow": dict(kf_last=-1),
            "rank_landmarks": dict(kf_slots=[])}


class _Stub:
    """capi.lib(): every C function records its name and what it received, decoded during the call, and succeeds"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, self._decode(name, args)))
            return 0
        fn.__name__ = name
        return fn

    @staticmethod
    def _decode(name, args):
        if name == "kba_track_group_drop_keyframes":
            return args[0], [args[1][0], args[1][1]]
        if name.startswith("kba_track_group_"):
            call = next((c for c, g in CALLS.items() if "kba_track_group_" + g[0] == name), None)
            if call is None:
                return args
            Req, at_out = CALLS[call][1], CALLS[call][3]
            return ([_decode(Req, lambda f, i=i: getattr(args[1][i], f)) for i in range(2)],
                    None if at_out is None else [_out(args[-1][i]) for i in range(2)])
        call = name[len("kba_track_"):]
        if call not in CALLS:
            return args
        _, Req, flat, at_out = CALLS[call]
        if flat is None:  # the request and output structs by reference
            q = args[1]._obj
            return _decode(Req, lambda f: getattr(q, f)), _out(args[at_out]._obj)
        vals = dict(zip(flat, args[1:]))  # the request's fields as arguments; its reserved_ fields are zero
        o = None if at_out is None else args[at_out]
        o = None if o is None else (o._obj if hasattr(o, "_obj") else o[0])
        return _decode(Req, lambda f: vals.get(f, 0)), None if o is None else _out(o)


@pytest.fixture
def stub(monkeypatch):
    s = _Stub()
    monkeypatch.setattr(capi, "_lib", s)
    t0, t1 = capi.Track.__new__(capi.Track), capi.Track.__new__(capi.Track)
    for t in (t0, t1):
        t._p, t._n_sel = C.c_void_p(0x10), 4
    g = capi.TrackGroup.__new__(capi.TrackGroup)
    g.tracks, g._p = [t0, t1], C.c_void_p(0x20)
    return s, t1, g


def _recorded(s, prefix):
    calls = [c for c in s.calls if c[0].startswith(prefix)]
    assert len(calls) == 1, s.calls
    return calls[0][1]


@pytest.mark.parametrize("call", sorted(CALLS))
def test_group_request_equals_single_request(stub, call):
    s, t, g = stub
    r = _requests()[call]
    getattr(t, call)(**r)
    q1, o1 = _recorded(s, "kba_track_" + call)
    s.calls.clear()
    res = getattr(g, CALLS[call][0])([None, r])
    qs, os_ = _recorded(s, "kba_track_group_" + CALLS[call][0])
    assert qs[1] == q1
    assert (os_ and os_[1]) == o1
    sat_out = qs[0]  # the ABI's sit-out encoding
    if call == "push_keyframe":
        assert sat_out["kf_slot"] == -1
    elif call == "frame_flow":
        assert sat_out["kf_last"] == -1
    elif call == "reclaim_landmarks":
        assert sat_out["lo"] == sat_out["hi"]
    elif call == "adjust_pose":
        assert sat_out["n_meas"] == 0
    elif call.startswith("set_"):
        assert sat_out["n"] == 0
    else:
        assert sat_out["n_kf"] == 0
    if call in ("solve", "solve_ranked", "adjust_pose"):  # an idle Result, kf_pose [0 or 1, 7]
        assert os_[0]["iterations_capacity"] == 1 and res[0].kf_pose.shape == ((1, 7) if call == "adjust_pose" else (0, 7))
    elif res is not None:
        assert res[0] is None


def test_drop_request(stub):
    s, t, g = stub
    t.drop_keyframe(6)
    assert _recorded(s, "kba_track_drop_keyframe")[1] == 6
    s.calls.clear()
    g.drop_keyframes([None, 6])
    arr = _recorded(s, "kba_track_group_drop_keyframes")[1]
    assert (arr[0], arr[1]) == (-1, 6)


@pytest.mark.parametrize("call", sorted(SITS_OUT))
def test_sit_out_request_fails_before_the_call(stub, call):
    s, t, g = stub
    with pytest.raises(capi.KbaError, match="kba_track_group_%s: track 1: " % CALLS[call][0]):
        getattr(g, CALLS[call][0])([None, dict(_requests()[call], **SITS_OUT[call])])
    assert s.calls == []


def test_empty_reclaim_range_is_an_empty_result(stub):
    s, t, g = stub
    for evict in (False, True):
        s.calls.clear()
        res = g.reclaim_landmarks([None, dict(lo=5, hi=5, evict=evict)])
        qs, _ = _recorded(s, "kba_track_group_reclaim_landmarks")
        assert qs[1]["lo"] == qs[1]["hi"]  # the track sits the call out
        assert res[0] is None
        if evict:
            assert [a.shape for a in res[1]] == [(0,), (0, 3), (0,)]
        else:
            assert res[1].shape == (0,) and res[1].dtype == np.int32


@pytest.mark.parametrize("call", sorted(CALLS))
def test_unexpected_key_fails_before_the_call(stub, call):
    s, t, g = stub
    with pytest.raises(TypeError, match="request 1"):
        getattr(g, CALLS[call][0])([None, dict(_requests()[call], no_such_key=1)])
    assert [c for c in s.calls if c[0] != "kba_default_options"] == []
