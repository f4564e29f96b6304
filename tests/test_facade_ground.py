"""The facade with ground-plane landmarks on the persistent window (tests/cpp/test_facade_ground.cpp): a mono-lidar drive whose
ground points are attached on the device, against a twin that rebuilds every window."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_facade_ground_points_on_the_store():
    """labelled ground tracklets, the AddDepth ground scheme and a 12-keyframe window: every solve() runs on the device-resident
    window and leaves poses, planes and landmarks bit-identical to the rebuild path's, with under 10 % of its upload; every
    adjustPoseOnly() runs on the store with a frame-sized upload"""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])
    out = subprocess.run([os.path.join(ROOT, "tests", "cpp", "test_facade_ground")], capture_output=True, text=True)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
