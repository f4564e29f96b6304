"""kba_lidar_depth_batch: many clouds and cameras in one call.  Each view must return exactly what kba_lidar_depth returns for
it, and so what the CPU oracle returns, bit for bit.  The binding is checked without a GPU against a stub library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from limo_b200 import capi, synth
from limo_b200 import geometry as g
from limo_b200.capi_types import KbaLidarCloud, KbaLidarOptions, KbaLidarView

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_struct_sizes_match_header(tmp_path):
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "kba_b200.h"\nint main(){printf("%zu %zu\\n",sizeof(kba_lidar_cloud),'
                    'sizeof(kba_lidar_view));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    assert [int(x) for x in subprocess.check_output([str(exe)]).split()] == [C.sizeof(KbaLidarCloud), C.sizeof(KbaLidarView)]


# ---- the binding against a stub library ---------------------------------------------------------------------------------
class _Stub:
    """capi.lib(): every C function records its name and its arguments decoded during the call, and succeeds"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, self._decode(name, args)))
            return 0
        return fn

    @staticmethod
    def _decode(name, args):
        if not name.startswith("kba_lidar_depth_batch"):
            return args
        _, n_clouds, clouds, n_views, views, opt, _ms = args
        cl = [(C.string_at(c.points, 4 * c.n_points * c.stride), c.n_points, c.stride) for c in clouds[:n_clouds]]
        vs = []
        for v in views[:n_views]:
            n = v.n_features
            vs.append((v.cloud, n, C.string_at(v.T_cam_lidar, 56), C.string_at(v.intr, 24), C.string_at(v.features_uv, 8 * n),
                       bool(v.depth_out)))
        opts = [opt[i] for i in range(n_views)] if name.endswith("_opts") else [opt._obj]
        return cl, vs, [(o.image_width, o.rect_width) for o in opts]


@pytest.fixture
def stub(monkeypatch):
    s = _Stub()
    monkeypatch.setattr(capi, "_lib", s)
    h = capi.Handle.__new__(capi.Handle)
    h._p = C.c_void_p(0x10)
    yield s, h
    h._p = C.c_void_p()  # no kba_destroy of the fake handle once the real library is back


def _small_request(rng):
    clouds = [rng.random((50, 4)).astype(np.float32), rng.random((30, 3)).astype(np.float32)]
    views = [(1, rng.random(7), rng.random(3), rng.random((5, 2)).astype(np.float32)),
             (0, rng.random(7), rng.random(3), np.zeros((0, 2), np.float32)),
             (1, rng.random(7), rng.random(3), rng.random((3, 2)))]
    return clouds, views


def _opt(width, rect):
    o = KbaLidarOptions()
    o.image_width, o.rect_width = width, rect
    return o


def test_binding_passes_the_arrays_by_content(stub):
    s, h = stub
    clouds, views = _small_request(np.random.default_rng(1))
    for opt, fn, opts in ((_opt(640, 6.0), "kba_lidar_depth_batch", [(640, 6.0)]),
                          ([_opt(640, 6.0), _opt(1242, 24.0), _opt(320, 3.0)], "kba_lidar_depth_batch_opts",
                           [(640, 6.0), (1242, 24.0), (320, 3.0)])):
        s.calls.clear()
        depths, _ = h.lidar_depth_batch(clouds, views, opt)
        (name, (cl, vs, os_)), = s.calls
        assert name == fn and os_ == opts
        assert cl == [(c.tobytes(), c.shape[0], c.shape[1]) for c in clouds]
        for v, (ci, T, K, uv) in zip(vs, views):
            uv = np.asarray(uv, dtype=np.float32)
            assert v == (ci, len(uv), np.asarray(T, np.float64).tobytes(), np.asarray(K, np.float64).tobytes(), uv.tobytes(),
                         len(uv) > 0)  # a view without features passes no depth_out
        assert [d.shape for d in depths] == [(5,), (0,), (3,)] and all(d.dtype == np.float32 for d in depths)


def test_bad_request_fails_before_the_call(stub):
    s, h = stub
    clouds, views = _small_request(np.random.default_rng(2))
    with pytest.raises(ValueError, match="2 option sets for 3 views"):
        h.lidar_depth_batch(clouds, views, [_opt(640, 6.0), None])
    bad = list(views)
    bad[2] = (2,) + tuple(views[2][1:])
    with pytest.raises(IndexError, match="view 2 names cloud 2"):
        h.lidar_depth_batch(clouds, bad)
    bad[2] = (-1,) + tuple(views[2][1:])
    with pytest.raises(IndexError, match="view 2 names cloud -1"):
        h.lidar_depth_batch(clouds, bad)
    assert s.calls == []


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    clouds, views = _small_request(np.random.default_rng(3))
    with pytest.raises(capi.KbaError):
        h = capi.Handle(0)
        h.lidar_depth_batch(clouds, views)


# ---- on the device --------------------------------------------------------------------------------------------------------
def _wall(depth=12.0, tilt=0.2):
    xs, ys = np.meshgrid(np.linspace(-6, 6, 500), np.linspace(-2, 2, 160))
    return np.stack([xs.ravel(), ys.ravel(), (depth + tilt * xs).ravel(), np.zeros(xs.size)], axis=1).astype(np.float32)


def _options(lib_opts, **mod):
    o = lib_opts()
    for k, v in mod.items():
        setattr(o, k, v)
    return o


def _yawed(T, angle):
    """the camera of T turned about the lidar's vertical axis"""
    return g.iso_to_pose(g.pose_to_iso(T) @ g.iso(g.angle_axis(angle, [0.0, 0.0, 1.0])))


def _baseline(T, b=0.54):
    """a second camera b metres to the right of T's (a stereo rig)"""
    return g.iso_to_pose(g.iso(t=[-b, 0.0, 0.0]) @ g.pose_to_iso(T))


def _features(rng, n, w=synth.IMG_W, h=synth.IMG_H):
    return np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], axis=1).astype(np.float32)


@pytest.mark.gpu
def test_mixed_batch_matches_oracle_and_single_call(oracle):
    rng = np.random.default_rng(11)
    K0 = np.array([synth.F, synth.CX, synth.CY])
    K640 = np.array([synth.F * 0.6, 320.0, 240.0])
    mods = [dict(), dict(rect_width=24.0, rect_height=30.0), dict(local_rel_tolerance=-1.0),
            dict(image_width=640, image_height=480), dict(rect_width=24.0, rect_height=30.0, hist_bin_width=0.5)]
    clouds, T0 = [], None
    for i in range(8):  # strides 4 and 3, and smaller scans
        c, T0, _, _ = synth.make_lidar_scene(seed=100 + i, n_azimuth=1875 if i < 4 else 700)
        clouds.append(c if i % 2 == 0 else np.ascontiguousarray(c[:, :3]))
    clouds.append(np.zeros((0, 4), np.float32))  # 8: empty
    clouds.append(_wall())                       # 9: a plane in front of the camera
    clouds.append(_wall(30.0, 0.0))              # 10: named by no view
    wall_T = np.array([1.0, 0, 0, 0, 0, 0, 0])
    views, mod_of = [], []
    for i in range(8):
        for j in range(4 if i != 3 else 1):
            m = (i + j) % len(mods)
            K = K640 if "image_width" in mods[m] else K0
            w, h = (640, 480) if "image_width" in mods[m] else (synth.IMG_W, synth.IMG_H)
            n = 2000 if (i, j) == (0, 0) else 300
            views.append((i, _yawed(T0, 0.4 * j), K, _features(rng, n, w, h)))
            mod_of.append(1 if (i, j) == (0, 0) else m)
    for j, T in enumerate((_yawed(T0, -0.7), _baseline(T0), _yawed(_baseline(T0), 0.3))):  # cloud 3 shared by three more views
        views.append((3, T, K0 if j != 1 else K0 * [1.1, 1, 1], _features(rng, 300)))
        mod_of.append(j)
    views.append((8, T0, K0, _features(rng, 100))); mod_of.append(0)
    views.append((9, wall_T, K0, np.stack([np.linspace(300, 900, 64), np.full(64, 180.0)], axis=1))); mod_of.append(0)
    for i in (1, 9):  # views that sit out
        views.insert(i, (i % 8, T0, K0, np.zeros((0, 2), np.float32))); mod_of.insert(i, 0)
    assert 35 <= len(views) <= 45
    h = capi.Handle(0)
    og = [_options(capi.lidar_default_options, **mods[m]) for m in mod_of]
    depths, ms = h.lidar_depth_batch(clouds, views, og)
    assert ms > 0
    best = 0
    for (ci, T, K, uv), d, m in zip(views, depths, mod_of):
        assert d.shape == (len(uv),)
        if len(uv) == 0:
            continue
        dc = oracle.lidar_depth(clouds[ci], T, K, uv, _options(oracle.lidar_default_options, **mods[m]))
        ds, _ = h.lidar_depth(clouds[ci], T, K, uv, _options(capi.lidar_default_options, **mods[m]))
        assert np.array_equal(d, dc) and np.array_equal(d, ds), (ci, m)
        best = max(best, int((d > 0).sum()))
        if ci == 8:
            assert (d == -1).all()
    assert best > 400
    h.close()


def _config4_views(n, scenes, rng):
    views = []
    for v in range(n):
        c = v % len(scenes)
        T = scenes[c][1] if v % 3 else _baseline(scenes[c][1])
        views.append((c, T, scenes[c][2], _features(rng, 2000)))
    return views


@pytest.mark.gpu
def test_264_views_and_workspace_growth():
    scenes = [synth.make_lidar_scene(seed=200 + i) for i in range(16)]
    clouds = [s[0] for s in scenes]
    h = capi.Handle(0)
    views = _config4_views(264, scenes, np.random.default_rng(21))
    single = [h.lidar_depth(clouds[c], T, K, uv)[0] for c, T, K, uv in views]
    for sel in (slice(None), slice(40, 48), slice(None)):
        depths, ms = h.lidar_depth_batch(clouds, views[sel])
        assert ms > 0
        assert all(np.array_equal(d, s) for d, s in zip(depths, single[sel]))
    assert sum(int((s > 0).sum()) for s in single) > 264 * 20
    h.close()


KBA_ERR_BAD_ARG = 1


@pytest.mark.gpu
def test_validation_names_the_index_and_writes_nothing():
    cloud, T, K, _ = synth.make_lidar_scene(seed=7)
    rng = np.random.default_rng(31)
    clouds = [cloud, np.ascontiguousarray(cloud[::2, :3])]
    views = [(0, T, K, _features(rng, 500)), (1, _baseline(T), K, _features(rng, 400)), (1, T, K, _features(rng, 300))]
    h = capi.Handle(0)
    L = capi.lib()
    sentinel = np.float32(-7.5)
    cases = [("view 1", lambda cs, vs: setattr(vs[1], "cloud", 2)),
             ("view 2", lambda cs, vs: setattr(vs[2], "n_features", -1)),
             ("cloud 1", lambda cs, vs: setattr(cs[1], "n_points", -1)),
             ("cloud 1", lambda cs, vs: setattr(cs[1], "stride", 2)),
             ("view 0", lambda cs, vs: setattr(vs[0], "features_uv", None))]
    for where, spoil in cases:
        fn, cs, vs, o, outs, keep = capi._lidar_batch_request(clouds, views, None)
        for d in outs:
            d[:] = sentinel
        spoil(cs, vs)
        ms = C.c_float(-1.0)
        assert fn(h._p, len(cs), cs, len(vs), vs, o, C.byref(ms)) == KBA_ERR_BAD_ARG, where
        assert ("kba_lidar_depth_batch: %s: " % where) in L.kba_last_error().decode()
        assert all((d == sentinel).all() for d in outs)
    fn, cs, vs, o, outs, keep = capi._lidar_batch_request(clouds, views, None)
    assert fn(h._p, -1, cs, len(vs), vs, o, None) == KBA_ERR_BAD_ARG
    depths, _ = h.lidar_depth_batch(clouds, views)
    for (c, Tv, Kv, uv), d in zip(views, depths):
        assert np.array_equal(d, h.lidar_depth(clouds[c], Tv, Kv, uv)[0])
    assert (depths[0] > 0).sum() > 20
    h.close()


@pytest.mark.gpu
def test_every_view_sits_out():
    h = capi.Handle(0)
    L = capi.lib()
    vs = (KbaLidarView * 3)()
    for i, v in enumerate(vs):
        v.cloud, v.n_features = 5, 0  # not read: a view without features names no cloud
    ms = C.c_float(-1.0)
    assert L.kba_lidar_depth_batch(h._p, 0, None, 3, vs, None, C.byref(ms)) == 0 and ms.value == 0.0
    ms = C.c_float(-1.0)
    assert L.kba_lidar_depth_batch_opts(h._p, 0, None, 0, None, None, C.byref(ms)) == 0 and ms.value == 0.0
    cloud, T, K, _ = synth.make_lidar_scene(seed=9)
    depths, ms = h.lidar_depth_batch([cloud], [(0, T, K, np.zeros((0, 2), np.float32))] * 4)
    assert ms == 0.0 and [d.shape for d in depths] == [(0,)] * 4
    h.close()
