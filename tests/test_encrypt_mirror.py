"""Runs the C++ host-mirror test of encryption after the fact (tests/cpp/test_encrypt_mirror.cpp): RemoteSegmentEncryptor encrypts
an oracle-written Zstd-only `.log` object, a plain one, and their `.indexes` object; the new chunk index is TransformFinisher's
with encryption on, the SegmentIndexesV1 positions follow the new sizes, and a manifest that already has encryption is refused."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_remote_segment_encryptor_under_emulation():
    target = "tests/cpp/test_encrypt_mirror_simt"
    subprocess.check_call(["make", "-s", "-C", ROOT, target])
    out = subprocess.run([os.path.join(ROOT, target)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr
