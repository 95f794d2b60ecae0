"""Runs the C++ host-mirror test of key rotation (tests/cpp/test_rekey_mirror.cpp): RemoteSegmentRekeyer re-encrypts an
oracle-written Zstd+AES `.log` object and its `.indexes` object under a new key; both decrypt under the new key only, the chunk
index and SegmentIndexesV1 are unchanged and the manifest changes only in its encryption fields."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_remote_segment_rekeyer_under_emulation():
    target = "tests/cpp/test_rekey_mirror_simt"
    subprocess.check_call(["make", "-s", "-C", ROOT, target])
    out = subprocess.run([os.path.join(ROOT, target)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr
