"""The Python binding of the keyframe solve without a GPU: capi.lib is replaced by a stub that records what each C call receives.
Track.keyframe_solve(**r) and TrackGroup.keyframe_solve([None, r]) must hand the C library the same request -- the struct field by
field, the arrays behind its pointers by content, tracklets and class table in the ABI's layout -- the group's entry 0 the sit-out
encoding, and a request without keyframes or with an unknown key must fail before any C call."""
import ctypes as C
import struct

import numpy as np
import pytest

from limo_b200 import capi
from limo_b200.capi_types import KbaKfsolveOut, KbaKfsolveRequest, KbaWindow

# pointer fields: (bytes per element, element count: a field of the request or a number)
POINTERS = dict(kf_slot=(4, "n_kf"), lm_slot=(4, "n_lm"), lm_ground=(1, "n_lm"), trk=(12, "n_trk"), classes=(8, "n_class"),
                outlier_slot=(4, "n_outlier"), params=(40, 1), depth=(8, "n_depth"))
WINDOW = ("n_kf", "n_lm", "n_gp", "scale_kf0", "scale_kf1", "scale_weight", "scale_value", "plane_reg_weight")


def _addr(v):
    if v is None or isinstance(v, int):
        return v or None
    return C.cast(v, C.c_void_p).value


def _decode(q):
    d = {}
    for f, _t in KbaKfsolveRequest._fields_:
        v = getattr(q, f)
        if f in POINTERS:
            a = _addr(v)
            size, count = POINTERS[f]
            d[f] = None if a is None else C.string_at(a, size * (count if isinstance(count, int) else getattr(q, count)))
        elif f == "sel":
            d[f] = None if v is None else {g: getattr(KbaWindow.from_address(v), g) for g in WINDOW}
        elif f == "draw":
            d[f] = bool(v)
        elif f == "draw_ctx":
            d[f] = _addr(v)
        else:
            d[f] = v
    return d


def _out(o):
    return {f: _addr(getattr(o, f)) is not None for f, _t in KbaKfsolveOut._fields_ if f != "rank"}


class _Stub:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            if name == "kba_track_keyframe_solve":
                self.calls.append((name, [_decode(args[1]._obj)], [_out(args[3]._obj)]))
            elif name.startswith("kba_track_group_keyframe_solve"):
                self.calls.append((name, [_decode(args[1][i]) for i in range(2)], [_out(args[3][i]) for i in range(2)]))
            return 0
        fn.__name__ = name
        return fn


@pytest.fixture
def stub(monkeypatch):
    s = _Stub()
    monkeypatch.setattr(capi, "_lib", s)
    t0, t1 = capi.Track.__new__(capi.Track), capi.Track.__new__(capi.Track)
    for t in (t0, t1):
        t._p, t._n_sel = C.c_void_p(0x10), None
    g = capi.TrackGroup.__new__(capi.TrackGroup)
    g.tracks, g._p = [t0, t1], C.c_void_p(0x20)
    return s, t1, g


def _request():
    return dict(kf_slots=[4, 5, 6, 7], lm_slots=[1, 3, 8, 9, 12], min_window=3, max_window=9, lm_ground=[1, 0, 0, 1, 0],
                tracklets=[(3, 2, 0), (-1, 1, 1), (12, 3, 0)], label_classes={3: 4, 1: 1, 2: 2}, outliers=[9, 1],
                shrubbery_weight=0.5, voxel_size=(0.5, 0.5, 0.3), max_far=7, depth=[(0, 3), (2, 1)], draws=np.arange(6),
                ground=True, plane_reg_weight=-1.0, scale_weight=-1.0, scale_value=1.25)


def test_request_layout(stub):
    s, t, _g = stub
    t.keyframe_solve(**_request())
    (name, (q,), (o,)), = s.calls
    assert name == "kba_track_keyframe_solve"
    assert (q["n_kf"], q["n_lm"], q["min_connecting"], q["min_window"], q["max_window"], q["n_trk"]) == (4, 5, 3, 3, 9, 3)
    assert np.frombuffer(q["kf_slot"], np.int32).tolist() == [4, 5, 6, 7]
    assert np.frombuffer(q["lm_ground"], np.uint8).tolist() == [1, 0, 0, 1, 0]
    assert [struct.unpack("<iiB3x", q["trk"][12 * i:12 * i + 12]) for i in range(3)] == [(3, 2, 0), (-1, 1, 1), (12, 3, 0)]
    assert struct.unpack("<6i", q["classes"]) == (1, 1, 2, 2, 3, 4)
    assert np.frombuffer(q["outlier_slot"], np.int32).tolist() == [9, 1]
    assert struct.unpack("<5d", q["params"]) == (0.5, 0.5, 0.3, capi.SELECT_DEFAULTS["roi_far"], capi.SELECT_DEFAULTS["roi_middle"])
    assert np.frombuffer(q["depth"], np.int32).tolist() == [0, 3, 2, 1]
    assert (q["shrubbery_weight"], q["max_near"], q["max_middle"], q["max_far"], q["draw"]) == (0.5, 300, 300, 7, True)
    assert q["sel"] == dict(n_kf=4, n_lm=5, n_gp=1, scale_kf0=0, scale_kf1=1, scale_weight=-1.0, scale_value=1.25, plane_reg_weight=-1.0)
    assert all(o.values()), o


def test_group_request_equals_single_request(stub):
    s, t, g = stub
    t.keyframe_solve(**_request())
    (_n, (q1,), (o1,)), = s.calls
    s.calls.clear()
    res = g.keyframe_solve([None, _request()])
    (name, qs, os_), = s.calls
    assert name == "kba_track_group_keyframe_solve"
    assert qs[1] == q1 and os_[1] == o1
    assert qs[0]["n_kf"] == 0 and res[0] is None
    s.calls.clear()
    g.keyframe_solve([None, _request()], opt=[None, capi.KbaOptions()])
    assert s.calls[0][0] == "kba_track_group_keyframe_solve_opts"


@pytest.mark.parametrize("bad, err", [(dict(kf_slots=[]), capi.KbaError), (dict(no_such_key=1), TypeError),
                                      (dict(tracklets=[(1, 0, 2)]), ValueError)])
def test_bad_group_request_fails_before_the_call(stub, bad, err):
    s, _t, g = stub
    with pytest.raises(err, match="track 1|request 1"):
        g.keyframe_solve([None, dict(_request(), **bad)])
    assert s.calls == []
