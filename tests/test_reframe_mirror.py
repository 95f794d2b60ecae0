"""Runs the C++ host-mirror test of TSGPU_FLAG_REFRAME (tests/cpp/test_reframe_mirror.cpp): RemoteSegmentRewriter with
addChecksums and denseFrames seals and re-encodes an oracle-written Zstd+AES object from its manifest through a ranged-GET fetcher;
the new ChunkIndex, part CRCs and the check of the new object agree."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_remote_segment_rewriter_reframes_under_emulation():
    target = "tests/cpp/test_reframe_mirror_simt"
    subprocess.check_call(["make", "-s", "-C", ROOT, target])
    out = subprocess.run([os.path.join(ROOT, target)], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr
