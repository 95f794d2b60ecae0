"""The zstd decoder's serial kernel (`zstd_dec_frames_kernel`) under the test-only SIMT emulator.  Frames of every writer reach it
when they carry more blocks than the index walks (serial_frames.py); nothing else in the suite does."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as ora
import tsgpu
from tsgpu import binding
from serial_frames import serial_kernel_frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z = tsgpu.FLAG_ZSTD


def test_simt_serial_kernel_frames():
    # libzstd frames, both own modes and a Content_Checksum, right and wrong; only the serial counter moves
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    c = tsgpu.Context(max_chunk_bytes=1 << 20, max_batch=4, lib_path=SIMT_LIB)
    try:
        frames = serial_kernel_frames(c)
        for name, src, f in frames:
            assert ora.zstd_decompress_chunk(f) == src.tobytes(), name
            st0 = c.decode_path_stats()
            back, osz = c.detransform(Z, f, [f.size], src.size)
            assert osz == [src.size] and np.array_equal(back, src), name
            assert c.decode_path_stats() == dict(st0, serial_frames=st0["serial_frames"] + 1), name
        name, src, f = frames[-1]
        assert name == "checksum" and f[4] & 4
        bad = f.copy()
        bad[-2] ^= 0x21
        with pytest.raises(Exception):
            ora.zstd_decompress_chunk(bad)
        with pytest.raises(tsgpu.TsgpuError) as e:
            c.detransform(Z, bad, [bad.size], src.size)
        assert e.value.code == binding.E_CORRUPT
        name, src, f = frames[1]
        rng = np.random.default_rng(8)
        for trial in range(40):
            bad = f.copy()
            bad[int(rng.integers(0, bad.size))] ^= 1 << int(rng.integers(0, 8))
            try:
                out, _ = c.detransform(Z, bad, [bad.size], src.size)
            except tsgpu.TsgpuError as e:
                assert e.code == binding.E_CORRUPT
            else:
                assert len(out) == src.size
    finally:
        c.close()


def test_serial_kernel_mutated_frames_never_overrun_under_asan():
    # bit flips, stomps, truncations, appended bytes on serial-routed libzstd frames: any answer but an out-of-bounds access
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so"])
    env = dict(os.environ, LD_PRELOAD=runtime, ASAN_OPTIONS="detect_leaks=0")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_serial.py"), "libtsgpu_simt_asan.so", "24", "11"],
                         env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "serial-kernel sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]
