"""The facade past its store's landmark capacity (tests/cpp/test_facade_reclaim.cpp): a 4096-slot store reclaims landmark slots
through a drive of several times as many landmarks and stays bit-identical to the rebuild path, on the device at every solve."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_facade_reclaims_landmark_slots():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all", "facade"])
    out = subprocess.run([os.path.join(ROOT, "tests", "cpp", "test_facade_reclaim")], capture_output=True, text=True)
    print(out.stdout[-4000:], out.stderr[-2000:])
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    assert "0 failed checks" in out.stdout
