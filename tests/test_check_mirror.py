"""Runs the C++ host-mirror test of the object check (tests/cpp/test_check_mirror.cpp): RemoteSegmentChecker checks uploaded
segments from their manifest through a ranged-GET fetcher and returns the CRC-32C of the object and of the segment."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_remote_segment_checker_under_emulation():
    target = "tests/cpp/test_check_mirror_simt"
    subprocess.check_call(["make", "-s", "-C", ROOT, target])
    out = subprocess.run([os.path.join(ROOT, target)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr
