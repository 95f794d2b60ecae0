"""Speed-mode frames (TSGPU_FLAG_ZSTD) written by the emulated kernels are the committed ones in
tests/golden/speed_frames.json (made by tests/golden/make_speed_golden.py), and every one of them reads back through the
oracle's libzstd.  Under the emulator lanes run in a fixed order, so the frames are a function of the input there: a change
to the entropy stage that alters a Huffman code length, a code or an FSE table shows up as a different digest."""
import json
import os
import subprocess
import sys

import numpy as np

from oracle import oracle as ora
import tsgpu
from tsgpu import corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
SPEED = json.load(open(os.path.join(GOLD, "speed_frames.json")))["cases"]
sys.path.insert(0, GOLD)
from make_speed_golden import SPEED_CASES, speed_digests  # noqa: E402


def test_fixture_lists_every_case():
    assert [(c["kind"], c["seed"], c["n"], c["chunk_size"]) for c in SPEED] == [tuple(c) for c in SPEED_CASES]


def test_emulated_speed_frames_are_the_committed_ones():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    ctx = tsgpu.Context(max_chunk_bytes=1 << 17, max_batch=4, lib_path=SIMT_LIB)
    try:
        got = speed_digests(ctx)
        for c in SPEED:                                  # the frames read back, whatever their bytes
            src = corpus.gen_segment(c["kind"], c["seed"], c["n"], c["chunk_size"])
            out, sizes = ctx.transform(tsgpu.FLAG_ZSTD, src, c["chunk_size"])
            back, _ = ora.detransform_chunks(ora.FLAG_ZSTD, out, sizes, c["n"])
            assert np.array_equal(back, src), c
    finally:
        ctx.close()
    assert [(g["sizes"], g["sha256"]) for g in got] == [(c["sizes"], c["sha256"]) for c in SPEED]
