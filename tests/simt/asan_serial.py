"""Run with libasan preloaded (tests/test_simt_serial_kernel.py): mutated libzstd frames that the decoder hands to its serial kernel
(serial_frames.serial_routed) — bit flips, byte stomps, truncations, appended bytes — go through the emulated decoder.  Any answer
is fine (an error, or bytes if the mutation left a valid frame) except an out-of-bounds access, which aborts under ASan.
argv[1] = library, argv[2] = mutations per frame (default 60), argv[3] = seed."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
from oracle import oracle as ora  # noqa: E402
from serial_frames import serial_routed  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
per = int(sys.argv[2]) if len(sys.argv) > 2 else 60
rng = np.random.default_rng(int(sys.argv[3]) if len(sys.argv) > 3 else 5)
CAP = 1 << 17
c = tsgpu.Context(max_chunk_bytes=CAP, max_batch=4, lib_path=lib)
src = corpus.gen_segment("K", 3, 70000, 70000)
frames = [serial_routed(ora.zstd_compress_level(src, level)) for level in (1, 3, 19)]
ok = err = 0
for frame in frames:
    for _ in range(per):
        f = frame.copy()
        how = int(rng.integers(0, 5))
        if how == 0:                                   # flip 1-3 bits
            for _ in range(int(rng.integers(1, 4))):
                f[int(rng.integers(0, f.size))] ^= 1 << int(rng.integers(0, 8))
        elif how == 1:                                 # stomp a short stretch
            a = int(rng.integers(0, f.size)); k = int(rng.integers(1, 9))
            f[a:a + k] = rng.integers(0, 256, min(k, f.size - a), dtype=np.uint8)
        elif how == 2:                                 # truncate
            f = f[:int(rng.integers(1, f.size))].copy()
        elif how == 3:                                 # the block headers after the frame header (empty ones, then the first real one)
            f[int(rng.integers(0, min(24 + 600, f.size)))] = int(rng.integers(0, 256))
        else:                                          # append garbage
            f = np.concatenate([f, rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8)])
        try:
            c.detransform(1, f, [f.size], CAP)
            ok += 1
            assert how != 4, "bytes after the frame were accepted (zstd-jni refuses them: Src size is incorrect)"
        except tsgpu.TsgpuError:
            err += 1
c.close()
print("serial-kernel sweep ok: %d frames x %d mutations, %d still decoded, %d refused" % (len(frames), per, ok, err))
