"""Runs the C++ host-mirror test of the object rewrite (tests/cpp/test_rewrite_mirror.cpp): RemoteSegmentRewriter rewrites an
uploaded segment and its indexes to Zstd+AES under a new key from the manifest through a ranged-GET fetcher; the new object and
indexes read back with the new key and not with the old one."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_remote_segment_rewriter_under_emulation():
    target = "tests/cpp/test_rewrite_mirror_simt"
    subprocess.check_call(["make", "-s", "-C", ROOT, target])
    out = subprocess.run([os.path.join(ROOT, target)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr
