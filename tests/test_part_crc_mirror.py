"""Runs the C++ host-mirror test of the upload-part checksums (tests/cpp/test_part_crc_mirror.cpp): SegmentLogUploader with
partChecksums hands every part to the sink with the CRC-32C of its bytes, and the upload carries the object's."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_part_checksums_reach_the_sink_under_emulation():
    target = "tests/cpp/test_part_crc_mirror_simt"
    subprocess.check_call(["make", "-s", "-C", ROOT, target])
    out = subprocess.run([os.path.join(ROOT, target)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr
