#!/usr/bin/env python
"""Lidar depth for many views in one call (kba_lidar_depth_batch) against a loop of single kba_lidar_depth calls, on the
120k-point, 2000-feature scene of bench.py's config 4.  16 seeded clouds (synth.make_lidar_scene) are cycled over the views;
each view gets its own cloud entry, so a batch of N views uploads N clouds, as N sequences of a track group would.
  - mono: 1, 8, 32, 132 and 264 views, one per cloud;
  - rig: two views per cloud, the second camera offset by a 0.54 m stereo baseline (the cloud is uploaded once).
Per size: device ms per call and device clouds/s (CUDA events around the kernels), end-to-end views/s over host buffers
(clouds, features and depths in pageable host memory), the same views through single calls in the same process, the
algorithmic bytes over the device time as a share of the data sheet's HBM bandwidth, the H2D / D2H bytes per call, and
whether every batch output equals the single-call output bit for bit.  Prints one JSON line; the card's name, power limit and
maximum SM clock are read in the same call."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from limo_b200 import capi, synth  # noqa: E402
from limo_b200 import geometry as g  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
PARAM_BYTES = 152 + 8      # per view in the packed upload: sizeof(LidarParams) and two prefix entries


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), [x.strip() for x in out.strip().splitlines()[0].split(",")])) if out.strip() else {}


def baseline(T, b=0.54):
    return g.iso_to_pose(g.iso(t=[-b, 0.0, 0.0]) @ g.pose_to_iso(T))


def case(scenes, n_views, rig):
    """(clouds, views): one cloud entry per view (mono) or per pair of views (rig)"""
    n_clouds = n_views // 2 if rig else n_views
    clouds = [scenes[c % len(scenes)][0] for c in range(n_clouds)]
    views = []
    for c in range(n_clouds):
        _, T, K, uv = scenes[c % len(scenes)]
        views.append((c, T, K, uv))
        if rig:
            views.append((c, baseline(T), K, uv))
    return clouds, views


def measure(h, clouds, views, reps):
    batch = lambda: h.lidar_depth_batch(clouds, views)  # noqa: E731
    single = lambda: [h.lidar_depth(clouds[c], T, K, uv) for c, T, K, uv in views]  # noqa: E731
    ref = [d for d, _ in single()]
    out, _ = batch()
    exact = all(np.array_equal(a, b) for a, b in zip(out, ref))
    dev, t0 = [], time.perf_counter()
    for _ in range(reps):
        dev.append(batch()[1])
    wall_b = (time.perf_counter() - t0) / reps
    dev_s, t0 = [], time.perf_counter()
    for _ in range(reps):
        dev_s.append(sum(ms for _, ms in single()))
    wall_s = (time.perf_counter() - t0) / reps
    nv, nc = len(views), len(clouds)
    pairs = sum(len(clouds[c]) for c, *_ in views)
    feats = sum(len(uv) for *_, uv in views)
    ms_b, ms_s = float(np.median(dev)), float(np.median(dev_s))
    alg = 56.0 * pairs  # two projection passes of 16 B per point, 24 B per sorted point record
    return {"views": nv, "clouds": nc,
            "batch": {"device_ms_per_call": ms_b, "device_us_per_view": 1e3 * ms_b / nv, "clouds_per_s_device": nc / (ms_b * 1e-3),
                      "views_per_s_e2e": nv / wall_b, "e2e_ms_per_call": 1e3 * wall_b},
            "single_calls": {"device_ms_per_loop": ms_s, "device_us_per_view": 1e3 * ms_s / nv, "views_per_s_e2e": nv / wall_s},
            "device_speedup_vs_single": ms_s / ms_b, "e2e_speedup_vs_single": wall_s / wall_b,
            "algorithmic": {"bytes_per_call": alg, "GB_per_s": alg / (ms_b * 1e-3) / 1e9,
                            "share_of_datasheet_hbm": alg / (ms_b * 1e-3) / HBM_BYTES_PER_S},
            "h2d_bytes_per_call": int(sum(c.nbytes for c in clouds) + 8 * feats + PARAM_BYTES * nv),
            "d2h_bytes_per_call": 4 * feats, "bit_exact_vs_single": bool(exact)}


def main():
    scenes = [synth.make_lidar_scene(seed=0xBA5E0004 + i) for i in range(16)]
    h = capi.Handle(0)
    shapes = [(n, False) for n in (1, 8, 32, 132, 264)] + [(n, True) for n in (8, 32, 132, 264)]
    for n, rig in shapes:  # warm every shape; the workspace grows to the largest
        clouds, views = case(scenes, n, rig)
        h.lidar_depth_batch(clouds, views)
        h.lidar_depth(clouds[0], *views[0][1:])
    res = {"workload": "config 4 scene: %d-point clouds -> 1242x375, 2000 features per view" % len(scenes[0][0]), "gpu": gpu_info(),
           "hbm_datasheet_bytes_per_s": HBM_BYTES_PER_S, "mono": [], "rig": []}
    for n, rig in shapes:
        clouds, views = case(scenes, n, rig)
        res["rig" if rig else "mono"].append(measure(h, clouds, views, reps=max(5, 200 // n)))
    res["bit_exact_vs_single_all"] = all(r["bit_exact_vs_single"] for k in ("mono", "rig") for r in res[k])
    h.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
